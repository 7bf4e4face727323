// perturb_probe.cpp — test helper for tests/test_sim_perturb_cpu.py: the simulator's calibration perturbation
// (Simulator::perturb_parameters in include/ovb200_sim.hpp).
//   perturb_probe TRAJ CAMS SEED_PERTURB FRAMES
// Builds the rpng_sim simulator twice with the same seeds, without and with sim_do_perturbation, steps both through FRAMES
// camera frames and prints
//   draws N d...         the perturbation's draws in draw order
//   init_err N e...      the estimator's initial calibration error in the consistency file's convention (truth - estimate,
//                        orientations -log(R_true R_est')), in the same order
//   true_params 0|1      1 when the perturbed simulator's true parameters and the unperturbed one's estimator parameters
//                        are the configured ones, bit for bit
//   map N 0|1            map points, and 1 when both maps are the same points in the same iteration order, bit for bit
//   streams I C F 0|1    IMU readings, camera messages, pixels, and 1 when both simulators produced the same ones, bit for bit
#include "../../include/ovb200_vio.hpp"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
using namespace ovb200;

static bool same_params(const SimParams &a, const SimParams &b) {
  bool ok = a.calib_camimu_dt == b.calib_camimu_dt && a.q_GYROtoIMU == b.q_GYROtoIMU && a.q_ACCtoIMU == b.q_ACCtoIMU &&
            !std::memcmp(a.vec_dw, b.vec_dw, sizeof(a.vec_dw)) && !std::memcmp(a.vec_da, b.vec_da, sizeof(a.vec_da)) &&
            !std::memcmp(a.vec_tg, b.vec_tg, sizeof(a.vec_tg)) && a.camera_extrinsics == b.camera_extrinsics;
  for (size_t i = 0; ok && i < a.camera_intrinsics.size(); i++)
    ok = !std::memcmp(a.camera_intrinsics[i].d, b.camera_intrinsics[i].d, sizeof(a.camera_intrinsics[i].d));
  return ok;
}

int main(int argc, char **argv) {
  if (argc < 5)
    return 2;
  const std::string traj = argv[1];
  const int cams = std::atoi(argv[2]), frames = std::atoi(argv[4]);
  const auto data = traj.substr(traj.size() - 4) == ".bin" ? load_trajectory_bin(traj) : load_simulated_trajectory(traj);
  SimParams sp;
  rpng_sim_cameras(cams, sp);
  sp.use_stereo = cams > 1;
  sp.num_pts = 200;
  sp.seed_preturb = std::atoi(argv[3]);
  SimParams spp = sp;
  spp.sim_do_perturbation = true;
  Simulator a(sp, data), b(spp, data);

  const SimParams &tru = b.get_true_parameters(), &est = b.get_estimator_parameters();
  std::vector<double> e;
  auto add = [&](const double *t, const double *x, int n) {
    for (int k = 0; k < n; k++)
      e.push_back(t[k] - x[k]);
  };
  auto add_ori = [&](const Vec4 &qt, const Vec4 &qe) {
    for (double x : ori_error(qt, qe))
      e.push_back(x);
  };
  add(&tru.calib_camimu_dt, &est.calib_camimu_dt, 1);
  for (int i = 0; i < cams; i++) {
    add(tru.camera_intrinsics[(size_t)i].d, est.camera_intrinsics[(size_t)i].d, 8);
    add_ori(tru.camera_extrinsics[(size_t)i].first, est.camera_extrinsics[(size_t)i].first);
    add(tru.camera_extrinsics[(size_t)i].second.data(), est.camera_extrinsics[(size_t)i].second.data(), 3);
  }
  for (int j = 0; j < 6; j++) {
    add(tru.vec_dw + j, est.vec_dw + j, 1);
    add(tru.vec_da + j, est.vec_da + j, 1);
  }
  add_ori(tru.q_GYROtoIMU, est.q_GYROtoIMU);
  add(tru.vec_tg, est.vec_tg, 9);
  std::printf("draws %zu", b.perturbation.size());
  for (double x : b.perturbation)
    std::printf(" %.17g", x);
  std::printf("\ninit_err %zu", e.size());
  for (double x : e)
    std::printf(" %.17g", x);
  std::printf("\ntrue_params %d\n", (int)(same_params(tru, sp) && same_params(a.get_estimator_parameters(), sp) && a.perturbation.empty()));

  bool map_same = a.featmap.size() == b.featmap.size();
  for (auto ia = a.featmap.begin(), ib = b.featmap.begin(); map_same && ia != a.featmap.end(); ++ia, ++ib)
    map_same = ia->first == ib->first && ia->second == ib->second;
  std::printf("map %zu %d\n", a.featmap.size(), (int)map_same);

  long n_imu = 0, n_cam = 0, n_pix = 0;
  bool same = true;
  while (a.ok() && n_cam < frames) {
    double ta = 0, tb = 0;
    Vec3 wa, aa, wb, ab;
    const bool ia = a.get_next_imu(ta, wa, aa), ib = b.get_next_imu(tb, wb, ab);
    same = same && ia == ib && (!ia || (ta == tb && wa == wb && aa == ab));
    n_imu += ia;
    std::vector<int> ca, cb;
    std::vector<std::vector<SimFeat>> fa, fb;
    const bool ka = a.get_next_cam(ta, ca, fa), kb = b.get_next_cam(tb, cb, fb);
    same = same && ka == kb && (!ka || (ta == tb && ca == cb && fa.size() == fb.size()));
    for (size_t c = 0; same && ka && c < fa.size(); c++) {
      same = fa[c].size() == fb[c].size();
      for (size_t k = 0; same && k < fa[c].size(); k++)
        same = fa[c][k].id == fb[c][k].id && fa[c][k].u == fb[c][k].u && fa[c][k].v == fb[c][k].v;
      n_pix += (long)fa[c].size();
    }
    n_cam += ka;
  }
  std::printf("streams %ld %ld %ld %d\n", n_imu, n_cam, n_pix, (int)same);
  return 0;
}
