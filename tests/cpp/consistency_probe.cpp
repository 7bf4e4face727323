// consistency_probe.cpp — test helper for tests/test_consistency_cpu.py: the error convention and the NEES of
// consistency_sample (include/ovb200_vio.hpp) on a hand-built state whose truth is a known perturbation of the estimate.
//   consistency_probe  -> four lines of numbers:
//     imu   dtheta(3) err_theta(3) other_frame(3) dp(3) err_p(3) nees_ori nees_pos P_thth(9) P_pp(9)
//     cam   dtheta(3) err_theta(3) other_frame(3)
//     gyro  dtheta(3) err_theta(3)
//     sigma max_k |sigma_k - sqrt(P_kk)|  n
// The truth is q_true = dq(dtheta) ⊗ q_est with the exact quaternion exponential dq = [sin(|d|/2) d/|d|, cos(|d|/2)]
// (JPLQuat::update's first-order [d/2, 1] normalised has the same axis and agrees with it to O(|d|^3)), so err_theta must
// equal dtheta to rounding. other_frame = -log(R_est' R_true), the error taken in the other frame, for the test to reject.
#include "../../include/ovb200_vio.hpp"
#include <cstdio>
using namespace ovb200;

struct NullCov : CovBackend {
  int dim() override { return 0; }
  void set(const std::vector<double> &, int) override {}
  std::vector<double> get() override { return {}; }
  std::vector<double> get_marginal(const std::vector<int> &, const std::vector<int> &) override { return {}; }
  void clone(int, int, const double *, int) override {}
  void marginalize(int, int) override {}
  void propagate(int, int, const std::vector<int> &, const std::vector<int> &, const std::vector<double> &, const std::vector<double> &) override {}
  int msckf_update(const ovb_frame *, const ovb_feat_batch *, const ovb_opts *, ovb_feat_out *, double *, ovb_stats *) override { return 0; }
};

static Vec4 dq_exact(const Vec3 &d) {
  const double a = norm(d), s = std::sin(0.5 * a) / a;
  return {s * d[0], s * d[1], s * d[2], std::cos(0.5 * a)};
}

static void print3(const Vec3 &v) { std::printf(" %.17g %.17g %.17g", v[0], v[1], v[2]); }

int main() {
  SimParams sp;
  rpng_sim_cameras(1, sp);
  VioOptions vo;
  vo.num_cameras = 1;
  VioManager sys(vo, sp, std::make_shared<NullCov>());
  VioState st = sys.state;
  const int n = st.base_size;
  // estimate far from identity; truth = a known perturbation of it
  st.q = quatnorm({0.6, -0.3, 0.5, 0.4});
  st.p = {1.5, -2.0, 0.7};
  const Vec3 dth{0.031, -0.052, 0.017}, dp{0.04, -0.013, 0.021};
  const Vec4 q_true = quat_multiply(dq_exact(dth), st.q);
  const Vec3 p_true = st.p + dp;
  std::array<double, 17> gt{};
  gt[0] = st.timestamp;
  for (int k = 0; k < 4; k++)
    gt[(size_t)(1 + k)] = q_true[(size_t)k];
  for (int k = 0; k < 3; k++) {
    gt[(size_t)(5 + k)] = p_true[(size_t)k];
    gt[(size_t)(8 + k)] = st.v[(size_t)k];
    gt[(size_t)(11 + k)] = st.bg[(size_t)k];
    gt[(size_t)(14 + k)] = st.ba[(size_t)k];
  }
  // camera extrinsic and gyroscope rotation: estimate far from identity, configured truth = its perturbation
  auto &cam = st.cams[0];
  cam.q_ItoC = quatnorm({-0.45, 0.35, 0.6, 0.55});
  const Vec3 dth_c{-0.024, 0.011, 0.047};
  sp.camera_extrinsics[0].first = quat_multiply(dq_exact(dth_c), cam.q_ItoC);
  sp.camera_extrinsics[0].second = cam.p_IinC;
  st.q_GYROtoIMU = quatnorm({0.2, 0.1, -0.3, 0.9});
  const Vec3 dth_g{0.013, 0.008, -0.021};
  sp.q_GYROtoIMU = quat_multiply(dq_exact(dth_g), st.q_GYROtoIMU);
  // a symmetric positive definite P with non-diagonal blocks: A A' / n + diag, A from a fixed linear congruential sequence
  std::vector<double> A((size_t)n * n), P((size_t)n * n);
  unsigned long long x = 12345;
  for (auto &a : A) {
    x = x * 6364136223846793005ULL + 1442695040888963407ULL;
    a = ((double)(x >> 11) / 9007199254740992.0 - 0.5) * 1e-2;
  }
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++) {
      double s = 0;
      for (int k = 0; k < n; k++)
        s += A[(size_t)i * n + k] * A[(size_t)j * n + k];
      P[(size_t)i * n + j] = s + (i == j ? 1e-5 * (1 + i % 7) : 0.0);
    }
  const ConsistencySample s = consistency_sample(st, sp, gt, P);
  const int ti = st.imu_id, ci = cam.ext_id, gi = st.gyro_id;
  auto err3 = [&](int id) { return Vec3{s.err[(size_t)id], s.err[(size_t)id + 1], s.err[(size_t)id + 2]}; };
  std::printf("imu");
  print3(dth), print3(err3(ti)), print3(-log_so3(transpose(quat_2_Rot(st.q)) * quat_2_Rot(q_true))), print3(dp), print3(err3(ti + 3));
  std::printf(" %.17g %.17g", s.nees_ori, s.nees_pos);
  for (int b : {ti, ti + 3})
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        std::printf(" %.17g", P[(size_t)(b + i) * n + b + j]);
  std::printf("\ncam");
  print3(dth_c), print3(err3(ci)), print3(-log_so3(transpose(quat_2_Rot(cam.q_ItoC)) * quat_2_Rot(sp.camera_extrinsics[0].first)));
  std::printf("\ngyro");
  print3(dth_g), print3(err3(gi));
  double dsig = 0;
  for (int k = 0; k < n; k++)
    dsig = std::max(dsig, std::abs(s.sigma[(size_t)k] - std::sqrt(P[(size_t)k * n + k])));
  std::printf("\nsigma %.17g %d\n", dsig, n);
  return 0;
}
