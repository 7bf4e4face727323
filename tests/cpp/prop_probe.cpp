// prop_probe.cpp — test helper for ovb_cov_propagate_imu: runs Propagator::propagate_and_clone (include/ovb200_vio.hpp) over
// `steps` IMU steps of seeded readings and dumps what it hands to CovBackend::propagate_imu, and the Phi / Q that the base
// (host) implementation then passes to CovBackend::propagate.
//   prop_probe METHOD CALIB STEPS SEED OUT
//     METHOD discrete | rk4 | analytical; CALIB 0: no IMU intrinsics (n = 15), 1: intrinsics without g-sensitivity (n = 30),
//     2: with g-sensitivity (n = 39)
// OUT: one text line "PROPIMU1 n=.. steps=.. nold=.. new_off=.. clone_off=.. clone_size=.. dt_off=.. N=.." followed by
// little-endian arrays: old_off, old_sz (int32 [nold]), F [steps][n][n], G [steps][n][12], qc [steps][4], dnc_dt [clone_size],
// Phi [n][n], Q [n][n] (float64).
#include "../../include/ovb200_vio.hpp"
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
using namespace ovb200;

namespace {
struct Recorder : CovBackend {
  int N = 0;
  int n = 0, steps = 0, new_off = 0, clone_off = 0, clone_size = 0, dt_off = -1;
  std::vector<double> F, G, qc, dnc, Phi, Q;
  std::vector<int> old_off, old_sz;
  int dim() override { return N; }
  void set(const std::vector<double> &, int N_) override { N = N_; }
  std::vector<double> get() override { return {}; }
  std::vector<double> get_marginal(const std::vector<int> &, const std::vector<int> &) override { return {}; }
  void clone(int, int size, const double *, int) override { N += size; }
  void marginalize(int, int size) override { N -= size; }
  void propagate(int, int, const std::vector<int> &, const std::vector<int> &, const std::vector<double> &Phi_, const std::vector<double> &Q_) override {
    Phi = Phi_, Q = Q_;
  }
  int msckf_update(const ovb_frame *, const ovb_feat_batch *, const ovb_opts *, ovb_feat_out *, double *, ovb_stats *) override { return 0; }
  void propagate_imu(int n_, int steps_, const std::vector<double> &F_, const std::vector<double> &G_, const std::vector<double> &qc_, int new_off_,
                     const std::vector<int> &old_off_, const std::vector<int> &old_sz_, int clone_off_, int clone_size_, const double *dnc_dt, int dt_off_) override {
    n = n_, steps = steps_, F = F_, G = G_, qc = qc_, new_off = new_off_, old_off = old_off_, old_sz = old_sz_;
    clone_off = clone_off_, clone_size = clone_size_, dt_off = dt_off_;
    dnc.assign(dnc_dt, dnc_dt ? dnc_dt + clone_size_ : dnc_dt);
    CovBackend::propagate_imu(n_, steps_, F_, G_, qc_, new_off_, old_off_, old_sz_, clone_off_, clone_size_, dnc_dt, dt_off_); // the host path
  }
};
} // namespace

int main(int argc, char **argv) {
  if (argc < 6)
    return 2;
  const std::string m = argv[1];
  const int calib = std::atoi(argv[2]), steps = std::atoi(argv[3]), seed = std::atoi(argv[4]);
  SimParams sp;
  rpng_sim_cameras(1, sp);
  sp.calib_camimu_dt = 0.0;
  VioOptions vo;
  vo.num_cameras = 1;
  vo.integration_method = m == "discrete" ? INTEGRATION_DISCRETE : (m == "analytical" ? INTEGRATION_ANALYTICAL : INTEGRATION_RK4);
  vo.do_calib_imu_intrinsics = calib >= 1;
  vo.do_calib_imu_g_sensitivity = calib >= 2;
  auto rec = std::make_shared<Recorder>();
  VioManager sys(vo, sp, rec);
  VioState st = sys.state;
  rec->N = st.base_size;
  std::mt19937 rng((unsigned)seed);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  st.timestamp = 0.0;
  st.q = st.q_fej = quatnorm({0.1 + 0.05 * U(rng), -0.2 + 0.05 * U(rng), 0.3 + 0.05 * U(rng), 0.9});
  st.p = st.p_fej = {U(rng), U(rng), U(rng)};
  st.v = st.v_fej = {U(rng), U(rng), U(rng)};
  st.bg = {0.01 * U(rng), 0.01 * U(rng), 0.01 * U(rng)};
  st.ba = {0.05 * U(rng), 0.05 * U(rng), 0.05 * U(rng)};
  for (int k = 0; k < 6; k++)
    st.dw[k] += 0.01 * U(rng), st.da[k] += 0.01 * U(rng);
  for (int k = 0; k < 9; k++)
    st.tg[k] = 1e-3 * U(rng);
  st.q_GYROtoIMU = quatnorm({0.01 * U(rng), 0.01 * U(rng), 0.01 * U(rng), 1.0});
  st.q_ACCtoIMU = quatnorm({0.01 * U(rng), 0.01 * U(rng), 0.01 * U(rng), 1.0});
  Propagator prop(vo.gravity_mag);
  const double dt = 0.0025; // rpng_sim's 400 Hz IMU
  for (int k = 0; k <= steps && steps > 0; k++) {
    ImuData d;
    d.timestamp = k * dt;
    d.wm = {0.3 + 0.2 * U(rng), -0.2 + 0.2 * U(rng), 0.5 + 0.2 * U(rng)};
    d.am = {0.5 + 0.5 * U(rng), 9.6 + 0.5 * U(rng), 1.0 + 0.5 * U(rng)};
    prop.imu_data.push_back(d);
  }
  prop.propagate_and_clone(st, *rec, steps > 0 ? steps * dt : 0.01);
  if (rec->steps != steps)
    return 3;
  FILE *f = std::fopen(argv[5], "wb");
  if (!f)
    return 4;
  const int N = rec->N - rec->clone_size; // P's dimension before the clone
  std::fprintf(f, "PROPIMU1 n=%d steps=%d nold=%d new_off=%d clone_off=%d clone_size=%d dt_off=%d N=%d\n", rec->n, rec->steps, (int)rec->old_off.size(),
               rec->new_off, rec->clone_off, rec->clone_size, rec->dt_off, N);
  std::fwrite(rec->old_off.data(), sizeof(int), rec->old_off.size(), f);
  std::fwrite(rec->old_sz.data(), sizeof(int), rec->old_sz.size(), f);
  for (const std::vector<double> *v : {&rec->F, &rec->G, &rec->qc})
    std::fwrite(v->data(), sizeof(double), v->size(), f);
  std::vector<double> dnc = rec->dnc;
  dnc.resize((size_t)rec->clone_size, 0.0); // without a time offset in the state: zeros, unused
  std::fwrite(dnc.data(), sizeof(double), dnc.size(), f);
  std::fwrite(rec->Phi.data(), sizeof(double), rec->Phi.size(), f);
  std::fwrite(rec->Q.data(), sizeof(double), rec->Q.size(), f);
  std::fclose(f);
  return 0;
}
