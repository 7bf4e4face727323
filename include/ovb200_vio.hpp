// ovb200_vio.hpp — the host-side callers either side of the MSCKF update (SURVEY.md §8f rows 2-4), header-only C++17:
//   ov_msckf::Propagator                 state/Propagator.cpp:33-138 (propagate_and_clone), :269-393 (select_imu_readings),
//                                        :395-480 (predict_and_compute), :482-598 (mean: discrete / RK4), :600-681 (Xi sums,
//                                        analytic mean), :683-828 (analytic F, G), :830-950 (discrete F, G), :952-1015 (H_Dw/Da/Tg)
//   ov_msckf::State (mean + ids)         state/State.cpp:28-166, state/State.h:66-135
//   StateHelper::augment_clone           state/StateHelper.cpp:579-616; marginalize_old_clone :618-629; EKFUpdate's mean update :185-196
//   ov_core::FeatureDatabase             feat/FeatureDatabase.cpp:59-321        ov_core::TrackSIM   track/TrackSIM.cpp:30-79
//   VioManager                           core/VioManager.cpp:166-254 (feed_*), :323-644 (do_feature_propagate_update: feature
//                                        selection, sort, cap, update, cleanup, marginalize, timing CSV), VioManagerHelper.cpp:40-76
//   run_simulation                       ov_msckf/src/run_simulation.cpp:117-176 (init from ground truth, 1-frame delay buffer)
//   ov_eval ATE                          ov_eval/src/calc/ResultTrajectory.cpp:82-109 (alignment "none": the filter starts from truth)
// The covariance is behind CovBackend: the product backend is the CUDA engine (EngineCov, libovb200.so through the C ABI);
// tests plug the CPU oracle behind the same interface (tests/cpp/oracle_backend.hpp, its SLAM calls in
// tests/cpp/oracle_slam_backend.hpp), so the two runs consume byte-identical inputs. Scope: MSCKF features and SLAM landmarks (max_slam >= 0; every landmark in feat_rep_slam), no ZUPT, no ArUco,
// radtan and equidistant (fisheye) cameras, mixed rigs included, KALIBR IMU model.
//   UpdaterSLAM                          update/UpdaterSLAM.cpp:61-251 (delayed_init), :253-479 (update), :481-647 (change_anchors)
//   ov_type::Landmark                    types/Landmark.cpp (set_from_xyz, get_xyz), types/Vec.h (update)
//   StateHelper::marginalize_slam        state/StateHelper.cpp (the should_marg landmarks)
#ifndef OVB200_VIO_HPP
#define OVB200_VIO_HPP

#include "ovb200_host.hpp"
#include "ovb200_sim.hpp"

#include <algorithm>
#include <chrono>
#include <cstring>
#include <functional>
#include <limits>
#include <memory>

namespace ovb200 {

struct ImuData {
  double timestamp = 0;
  Vec3 wm{0, 0, 0}, am{0, 0, 0};
};

// ---------------------------------------------------------------------------------------------------------------------
// the covariance arithmetic of Propagator::propagate_and_clone on the host, in the reference's order: every entry is one
// dot product over ascending k from 0, with separate multiply and add (ovb_cov_propagate_imu reproduces these bits)

// Qd = sym(G diag(qc[k/3]) G') of one IMU step, G n x 12 row-major (Propagator.cpp:453-464; sym(X) = 0.5 (X + X'))
inline void imu_discrete_noise(int n, const double *G, const double *qc, std::vector<double> &Qd) {
  std::vector<double> Qt((size_t)n * n, 0.0);
  for (int a = 0; a < n; a++)
    for (int b = 0; b < n; b++) {
      double s = 0;
      for (int k = 0; k < 12; k++)
        s += G[(size_t)a * 12 + k] * qc[k / 3] * G[(size_t)b * 12 + k];
      Qt[(size_t)a * n + b] = s;
    }
  Qd.assign((size_t)n * n, 0.0);
  for (int a = 0; a < n; a++)
    for (int b = 0; b < n; b++)
      Qd[(size_t)a * n + b] = 0.5 * (Qt[(size_t)a * n + b] + Qt[(size_t)b * n + a]);
}

// Phi_summed, Qd_summed over the IMU steps between two clone times (Propagator.cpp:83-99). F: [steps][n][n],
// G: [steps][n][12], qc: [steps][4], row-major; steps = 0 leaves Phi = I, Q = 0.
inline void imu_accumulate(int n, int steps, const double *F, const double *G, const double *qc, std::vector<double> &Phi_summed,
                           std::vector<double> &Qd_summed) {
  auto matmul = [n](const double *A, const double *B, double *C) { // C = A B
    for (int i = 0; i < n; i++)
      for (int j = 0; j < n; j++) {
        double s = 0;
        for (int k = 0; k < n; k++)
          s += A[(size_t)i * n + k] * B[(size_t)k * n + j];
        C[(size_t)i * n + j] = s;
      }
  };
  auto matmul_bt = [n](const double *A, const double *B, double *C) { // C = A B'
    for (int i = 0; i < n; i++)
      for (int j = 0; j < n; j++) {
        double s = 0;
        for (int k = 0; k < n; k++)
          s += A[(size_t)i * n + k] * B[(size_t)j * n + k];
        C[(size_t)i * n + j] = s;
      }
  };
  Phi_summed.assign((size_t)n * n, 0.0);
  Qd_summed.assign((size_t)n * n, 0.0);
  std::vector<double> tmp((size_t)n * n), tmp2((size_t)n * n), Qdi;
  for (int i = 0; i < n; i++)
    Phi_summed[(size_t)i * n + i] = 1.0;
  for (int s = 0; s < steps; s++) {
    const double *Fs = F + (size_t)s * n * n;
    imu_discrete_noise(n, G + (size_t)s * n * 12, qc + (size_t)s * 4, Qdi);
    // Phi_summed = F * Phi_summed; Qd_summed = F * Qd_summed * F' + Qdi, symmetrised (:91-99)
    matmul(Fs, Phi_summed.data(), tmp.data());
    Phi_summed = tmp;
    matmul(Fs, Qd_summed.data(), tmp.data());
    matmul_bt(tmp.data(), Fs, tmp2.data());
    for (int a = 0; a < n * n; a++)
      tmp2[(size_t)a] += Qdi[(size_t)a];
    for (int a = 0; a < n; a++)
      for (int b = 0; b < n; b++)
        Qd_summed[(size_t)a * n + b] = 0.5 * (tmp2[(size_t)a * n + b] + tmp2[(size_t)b * n + a]);
  }
}

// JPLQuat::update (types/JPLQuat.h:114-126): q <- quatnorm([dθ/2; 1]) ⊗ q. The engine's ovb_slam_delayed_init_batch moves
// its frame with the same source on the device.
inline void jpl_update(Vec4 &q, const double *d) {
  const Vec4 dq = quatnorm({.5 * d[0], .5 * d[1], .5 * d[2], 1.0});
  q = quat_multiply(dq, q);
}

// PoseJPL::update (types/PoseJPL.h:74-91) of a pose marshalled as ovb_frame reads it: q and R = quat_2_Rot(q), p
inline void pose_update(Vec4 &q, double *R, double *p, const double *d) {
  jpl_update(q, d);
  const Mat3 Rn = quat_2_Rot(q);
  std::copy(Rn.begin(), Rn.end(), R);
  for (int j = 0; j < 3; j++)
    p[j] += d[3 + j];
}

// covariance residency + the update arithmetic, i.e. everything the reference does on State::_Cov
struct CovBackend {
  virtual ~CovBackend() {}
  virtual int dim() = 0;
  virtual void set(const std::vector<double> &P, int N) = 0;                                              // StateHelper::set_initial_covariance
  virtual std::vector<double> get() = 0;                                                                  // get_full_covariance
  virtual std::vector<double> get_marginal(const std::vector<int> &off, const std::vector<int> &sz) = 0;  // get_marginal_covariance
  virtual void clone(int old_off, int size, const double *dnc_dt, int dt_off) = 0;                        // clone + augment_clone's dt term
  virtual void marginalize(int off, int size) = 0;                                                        // marginalize
  virtual void propagate(int new_off, int p, const std::vector<int> &old_off, const std::vector<int> &old_sz, const std::vector<double> &Phi,
                         const std::vector<double> &Q) = 0;                                               // EKFPropagation
  virtual int msckf_update(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, ovb_feat_out *out, double *dx,
                           ovb_stats *stats) = 0;                                                         // UpdaterMSCKF::update steps 2-6
  // UpdaterSLAM::update steps 4-5 on one batch, landmark f in representation reps[f] (ovb_slam_update_reps)
  virtual int slam_update(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_landmarks *landmarks, const int32_t *reps, const ovb_opts *opts,
                          ovb_feat_out *out, double *dx, ovb_stats *stats) {
    return unsupported("slam_update");
  }
  // UpdaterSLAM::delayed_init after the measurement cleaning (ovb_slam_delayed_init_reps): on_init runs after every accepted
  // feature and refreshes the arrays `frame` points to
  virtual void slam_delayed_init(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, const int32_t *reps, const double *sigma_pix,
                                 const double *chi2_multipler, ovb_init_callback on_init, void *user, ovb_feat_out *out, int32_t *lm_off) {
    unsupported("slam_delayed_init");
  }
  // UpdaterSLAM::delayed_init without a callback (ovb_slam_delayed_init_batch): the backend moves the frame between the
  // features itself and returns every initialised feature's records (lm_off, dx_new [F][3], dx [F][ld_dx]), which the caller
  // replays in feature order. This default runs slam_delayed_init with a callback that moves a copy of the frame with the
  // reference's mean update (clone poses; extrinsics and intrinsics when they are calibrated) and collects the records.
  virtual void slam_delayed_init_batch(const ovb_frame *frame, const ovb_frame_quat *quat, const ovb_feat_batch *feats, const ovb_opts *opts,
                                       const int32_t *reps, const double *sigma_pix, const double *chi2_multipler, ovb_feat_out *out,
                                       int32_t *lm_off, double *dx_new, double *dx, int ld_dx) {
    struct Moved {
      std::vector<double> cR, cp, kR, kp, kin;
      std::vector<Vec4> cq, kq;
      ovb_frame fr;
      const ovb_opts *opts;
      double *dx_new, *dx;
      int ld_dx, short_dx;
    } mv;
    const int C = frame->n_clones, K = frame->n_cams;
    mv.cR.assign(frame->clone_R, frame->clone_R + 9 * C), mv.cp.assign(frame->clone_p, frame->clone_p + 3 * C);
    mv.kR.assign(frame->cam_R, frame->cam_R + 9 * K), mv.kp.assign(frame->cam_p, frame->cam_p + 3 * K);
    mv.kin.assign(frame->cam_intr, frame->cam_intr + 8 * K);
    for (int c = 0; c < C; c++)
      mv.cq.push_back({quat->clone_q[4 * c], quat->clone_q[4 * c + 1], quat->clone_q[4 * c + 2], quat->clone_q[4 * c + 3]});
    for (int k = 0; k < K; k++)
      mv.kq.push_back({quat->cam_q[4 * k], quat->cam_q[4 * k + 1], quat->cam_q[4 * k + 2], quat->cam_q[4 * k + 3]});
    mv.fr = *frame; // the FEJ arrays are the caller's: they never move
    mv.fr.clone_R = mv.cR.data(), mv.fr.clone_p = mv.cp.data(), mv.fr.cam_R = mv.kR.data(), mv.fr.cam_p = mv.kp.data(), mv.fr.cam_intr = mv.kin.data();
    mv.opts = opts, mv.dx_new = dx_new, mv.dx = dx, mv.ld_dx = ld_dx, mv.short_dx = 0;
    ovb_init_callback on_init = [](void *user, int f, int lm_off_f, int lm_size, const double *dxn, const double *d, int n_dx) {
      (void)lm_off_f;
      Moved &m = *(Moved *)user;
      std::copy(dxn, dxn + lm_size, m.dx_new + 3 * (size_t)f);
      if (n_dx > m.ld_dx)
        m.short_dx = 1;
      else
        std::copy(d, d + n_dx, m.dx + (size_t)f * m.ld_dx);
      for (int c = 0; c < m.fr.n_clones; c++)
        pose_update(m.cq[(size_t)c], &m.cR[(size_t)9 * c], &m.cp[(size_t)3 * c], d + m.fr.clone_off[c]);
      for (int k = 0; k < m.fr.n_cams; k++) {
        if (m.opts->do_calib_camera_pose)
          pose_update(m.kq[(size_t)k], &m.kR[(size_t)9 * k], &m.kp[(size_t)3 * k], d + m.fr.cam_ext_off[k]);
        if (m.opts->do_calib_camera_intrinsics)
          for (int j = 0; j < 8; j++)
            m.kin[(size_t)8 * k + j] += d[m.fr.cam_intr_off[k] + j];
      }
    };
    slam_delayed_init(&mv.fr, feats, opts, reps, sigma_pix, chi2_multipler, on_init, &mv, out, lm_off);
    if (mv.short_dx)
      throw Error(OVB_ERR_ARG, "slam_delayed_init_batch: ld_dx is shorter than a landmark's correction");
  }
  // StateHelper::marginalize_slam / UpdaterSLAM::change_anchors / StateHelper::marginalize_old_clone (ovb_marginalize_window):
  // the anchor changes in the order given, then the ranges removed, offsets as before the call
  virtual void marginalize_window(const ovb_frame *frame, const ovb_opts *opts, const int32_t *marg_off, const int32_t *marg_sz, int n_marg,
                                  const ovb_anchor_changes *anchors) {
    unsupported("marginalize_window");
  }
  // a backend without the SLAM calls (or the window shift) cannot run a frame that needs them
  [[noreturn]] static int unsupported(const char *what) { throw Error(OVB_ERR_ARG, std::string(what) + ": not provided by this covariance backend"); }
  // Propagator::propagate_and_clone's covariance side (Propagator.cpp:83-137): Phi and Qd accumulated over the IMU steps
  // (F: [steps][n][n], G: [steps][n][12], qc: [steps][4]), EKFPropagation of [new_off, new_off+n) from (old_off, old_sz),
  // then augment_clone. This is the reference's host arithmetic; a backend that runs it elsewhere must keep its bits.
  virtual void propagate_imu(int n, int steps, const std::vector<double> &F, const std::vector<double> &G, const std::vector<double> &qc, int new_off,
                             const std::vector<int> &old_off, const std::vector<int> &old_sz, int clone_off, int clone_size, const double *dnc_dt,
                             int dt_off) {
    std::vector<double> Phi, Q;
    imu_accumulate(n, steps, F.data(), G.data(), qc.data(), Phi, Q);
    propagate(new_off, n, old_off, old_sz, Phi, Q);
    clone(clone_off, clone_size, dnc_dt, dt_off);
  }
};

// product backend: the device-resident covariance of the CUDA engine
class EngineCov : public CovBackend {
public:
  explicit EngineCov(const ovb_config &cfg) {
    const ovb_status st = ovb_create(&cfg, &ctx_);
    if (st != OVB_OK)
      throw Error(st, std::string("ovb_create: ") + (ctx_ ? ovb_last_error(ctx_) : "no context (is a CUDA GPU visible?)"));
    check(ovb_set_slam_unbounded(ctx_, 1), "set_slam_unbounded"); // one call per max_slam_in_update batch, whatever its width
  }
  ~EngineCov() override {
    if (ctx_)
      ovb_destroy(ctx_);
  }
  ovb_ctx *ctx() const { return ctx_; }
  int dim() override { return ovb_cov_dim(ctx_); }
  void set(const std::vector<double> &P, int N) override { check(ovb_cov_set(ctx_, P.data(), N), "cov_set"); }
  std::vector<double> get() override {
    const int N = dim();
    std::vector<double> P((size_t)N * N);
    check(ovb_cov_get(ctx_, P.data(), N), "cov_get");
    return P;
  }
  std::vector<double> get_marginal(const std::vector<int> &off, const std::vector<int> &sz) override {
    int n = 0;
    for (int s : sz)
      n += s;
    std::vector<double> out((size_t)n * n);
    check(ovb_cov_get_marginal(ctx_, off.data(), sz.data(), (int)off.size(), out.data()), "cov_get_marginal");
    return out;
  }
  void clone(int old_off, int size, const double *dnc_dt, int dt_off) override { check(ovb_cov_clone(ctx_, old_off, size, dnc_dt, dt_off), "cov_clone"); }
  void marginalize(int off, int size) override { check(ovb_cov_marginalize(ctx_, off, size), "cov_marginalize"); }
  void propagate(int new_off, int p, const std::vector<int> &old_off, const std::vector<int> &old_sz, const std::vector<double> &Phi,
                 const std::vector<double> &Q) override {
    check(ovb_cov_propagate(ctx_, new_off, p, old_off.data(), old_sz.data(), (int)old_off.size(), Phi.data(), Q.data()), "cov_propagate");
  }
  int msckf_update(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, ovb_feat_out *out, double *dx, ovb_stats *stats) override {
    const ovb_status st = ovb_msckf_update(ctx_, frame, feats, opts, out, dx, stats);
    check(st, "msckf_update");
    return st;
  }
  int slam_update(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_landmarks *landmarks, const int32_t *reps, const ovb_opts *opts,
                  ovb_feat_out *out, double *dx, ovb_stats *stats) override {
    const ovb_status st = ovb_slam_update_reps(ctx_, frame, feats, landmarks, reps, opts, out, dx, stats);
    check(st, "slam_update");
    return st;
  }
  void slam_delayed_init(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, const int32_t *reps, const double *sigma_pix,
                         const double *chi2_multipler, ovb_init_callback on_init, void *user, ovb_feat_out *out, int32_t *lm_off) override {
    check(ovb_slam_delayed_init_reps(ctx_, frame, feats, opts, reps, sigma_pix, chi2_multipler, on_init, user, out, lm_off), "slam_delayed_init");
  }
  void slam_delayed_init_batch(const ovb_frame *frame, const ovb_frame_quat *quat, const ovb_feat_batch *feats, const ovb_opts *opts,
                               const int32_t *reps, const double *sigma_pix, const double *chi2_multipler, ovb_feat_out *out, int32_t *lm_off,
                               double *dx_new, double *dx, int ld_dx) override {
    check(ovb_slam_delayed_init_batch(ctx_, frame, quat, feats, opts, reps, sigma_pix, chi2_multipler, out, lm_off, dx_new, dx, ld_dx),
          "slam_delayed_init_batch");
  }
  void marginalize_window(const ovb_frame *frame, const ovb_opts *opts, const int32_t *marg_off, const int32_t *marg_sz, int n_marg,
                          const ovb_anchor_changes *anchors) override {
    check(ovb_marginalize_window(ctx_, frame, opts, marg_off, marg_sz, n_marg, anchors), "marginalize_window");
  }
  // the accumulation, EKFPropagation and clone as one device call (one stream synchronisation)
  void propagate_imu(int n, int steps, const std::vector<double> &F, const std::vector<double> &G, const std::vector<double> &qc, int new_off,
                     const std::vector<int> &old_off, const std::vector<int> &old_sz, int clone_off, int clone_size, const double *dnc_dt, int dt_off) override {
    check(ovb_cov_propagate_imu(ctx_, n, steps, F.data(), G.data(), qc.data(), new_off, old_off.data(), old_sz.data(), (int)old_off.size(), clone_off,
                                clone_size, dnc_dt, dt_off, nullptr, nullptr),
          "cov_propagate_imu");
  }

private:
  ovb_ctx *ctx_ = nullptr;
  void check(ovb_status st, const char *where) const {
    if (st != OVB_OK)
      throw Error(st, std::string(where) + ": " + ovb_last_error(ctx_));
  }
};

// ---------------------------------------------------------------------------------------------------------------------
enum IntegrationMethod { INTEGRATION_DISCRETE = 0, INTEGRATION_RK4 = 1, INTEGRATION_ANALYTICAL = 2 }; // StateOptions::IntegrationMethod

// StateOptions (state/StateOptions.h:35-176) + the estimator options of VioManagerOptions the runner reads; defaults =
// config/rpng_sim/estimator_config.yaml
struct VioOptions {
  bool do_fej = true;
  int integration_method = INTEGRATION_RK4;
  bool do_calib_camera_pose = true, do_calib_camera_intrinsics = true, do_calib_camera_timeoffset = true;
  bool do_calib_imu_intrinsics = true, do_calib_imu_g_sensitivity = true;
  int max_clone_size = 11;
  int max_msckf_in_update = 10;
  int num_cameras = 2;
  int feat_rep_msckf = OVB_REP_GLOBAL_3D;
  double gravity_mag = 9.81;
  double sigma_w = 1.6968e-04, sigma_wb = 1.9393e-05, sigma_a = 2.0000e-3, sigma_ab = 3.0000e-3; // NoiseManager (utils/NoiseManager.h)
  UpdaterOptions msckf_options{1.0, 1.0}; // up_msckf_chi2_multipler 1, up_msckf_sigma_px 1
  // SLAM landmarks (StateOptions::max_slam_features, max_slam_in_update, feat_rep_slam; VioManagerOptions::dt_slam_delay).
  // max_slam_features = 0 runs the MSCKF alone; 25 and GLOBAL_3D are the rpng_sim values (SURVEY.md §8d); dt_slam_delay:
  // INTEGRATION.md §8
  int max_slam_features = 0;
  int max_slam_in_update = 25;
  double dt_slam_delay = 1.0;
  int feat_rep_slam = OVB_REP_GLOBAL_3D;
  UpdaterOptions slam_options{1.0, 1.0}; // up_slam_chi2_multipler 1, up_slam_sigma_px 1
  FeatureInitializerOptions featinit_options;
  int col_order = OVB_COLS_CANONICAL;
  int compress = OVB_COMPRESS_CHOLQR2;
  bool record_timing_information = false;
  std::string record_timing_filepath = "/tmp/traj_timing.txt";
};

struct ClonePose { // ov_type::PoseJPL of a clone: value + FEJ
  int id = -1;
  Vec4 q{0, 0, 0, 1}, q_fej{0, 0, 0, 1};
  Vec3 p{0, 0, 0}, p_fej{0, 0, 0};
};

// ov_type::Landmark (types/Landmark.h, Landmark.cpp): a SLAM feature in the state. value / fej hold the representation's own
// parameters (size() of them), as ov_type::Vec keeps them:
//   GLOBAL_3D, ANCHORED_3D                              p (global / anchor frame)
//   GLOBAL_FULL_INVERSE_DEPTH, ANCHORED_FULL_INVERSE_DEPTH  (theta, phi, rho) with p = (1/rho) (cos theta sin phi, sin theta sin phi, cos phi)
//   ANCHORED_MSCKF_INVERSE_DEPTH                        (x/z, y/z, 1/z) of p in the anchor frame
//   ANCHORED_INVERSE_DEPTH_SINGLE                       1/z, with the bearing uv_norm_zero = (x/z, y/z, 1) kept beside it
struct SlamLandmark {
  size_t featid = 0;
  int id = -1; // first row/column of the landmark's block in the covariance
  int rep = OVB_REP_GLOBAL_3D;
  int unique_camera_id = -1; // the camera that triangulated it (should_marg when that camera sees it no longer)
  int anchor_cam_id = -1;
  double anchor_clone_timestamp = -1;
  int update_fail_count = 0;
  bool should_marg = false;
  double value[3] = {0, 0, 0}, fej[3] = {0, 0, 0};
  Vec3 uv_norm_zero{0, 0, 1}, uv_norm_zero_fej{0, 0, 1};

  int size() const { return rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3; }
  static bool anchored(int rep) { return rep != OVB_REP_GLOBAL_3D && rep != OVB_REP_GLOBAL_FULL_INVERSE_DEPTH; }
  // Landmark::set_from_xyz: p is p_FinG for the global representations, p_FinA for the anchored ones
  void set_from_xyz(const Vec3 &p, bool isfej) {
    double *v = isfej ? fej : value;
    if (rep == OVB_REP_GLOBAL_3D || rep == OVB_REP_ANCHORED_3D) {
      v[0] = p[0], v[1] = p[1], v[2] = p[2];
    } else if (rep == OVB_REP_GLOBAL_FULL_INVERSE_DEPTH || rep == OVB_REP_ANCHORED_FULL_INVERSE_DEPTH) {
      const double rho = 1 / norm(p);
      v[0] = std::atan2(p[1], p[0]);
      v[1] = std::acos(rho * p[2]);
      v[2] = rho;
    } else if (rep == OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH) {
      v[0] = p[0] / p[2], v[1] = p[1] / p[2], v[2] = 1 / p[2];
    } else { // ANCHORED_INVERSE_DEPTH_SINGLE
      v[0] = 1.0 / p[2];
      (isfej ? uv_norm_zero_fej : uv_norm_zero) = Vec3{p[0] / p[2], p[1] / p[2], 1.0};
    }
  }
  // Landmark::get_xyz. As in the reference, the two MSCKF-style inverse-depth representations read the value whatever
  // getfej says (Landmark.cpp leaves their FEJ branch out)
  Vec3 get_xyz(bool getfej) const {
    const double *v = getfej ? fej : value;
    if (rep == OVB_REP_GLOBAL_3D || rep == OVB_REP_ANCHORED_3D)
      return {v[0], v[1], v[2]};
    if (rep == OVB_REP_GLOBAL_FULL_INVERSE_DEPTH || rep == OVB_REP_ANCHORED_FULL_INVERSE_DEPTH)
      return {(1 / v[2]) * std::cos(v[0]) * std::sin(v[1]), (1 / v[2]) * std::sin(v[0]) * std::sin(v[1]), (1 / v[2]) * std::cos(v[1])};
    if (rep == OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH)
      return {(1 / value[2]) * value[0], (1 / value[2]) * value[1], 1 / value[2]};
    return (1.0 / value[0]) * uv_norm_zero; // ANCHORED_INVERSE_DEPTH_SINGLE
  }
  // Landmark::update (ov_type::Vec::update): the parameters move by dx, the FEJ stays
  void update(const double *dx) {
    for (int k = 0; k < size(); k++)
      value[k] += dx[k];
  }
};

// ov_msckf::State: the mean of every variable and its covariance id (state/State.cpp:28-131 fixes the order:
// IMU 15 | dw 6 | da 6 | tg 9 | R_GYROtoIMU 3 | dt 1 | per camera: extrinsics 6, intrinsics 8 | clones 6 ...)
struct VioState {
  VioOptions opt;
  double timestamp = -1;
  // ov_type::IMU (types/IMU.h): value and fej, [q(4) p(3) v(3) bg(3) ba(3)]
  Vec4 q{0, 0, 0, 1}, q_fej{0, 0, 0, 1};
  Vec3 p{0, 0, 0}, v{0, 0, 0}, bg{0, 0, 0}, ba{0, 0, 0}, p_fej{0, 0, 0}, v_fej{0, 0, 0};
  int imu_id = 0;
  double dw[6] = {1, 0, 0, 1, 0, 1}, da[6] = {1, 0, 0, 1, 0, 1}, tg[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  Vec4 q_GYROtoIMU{0, 0, 0, 1}, q_ACCtoIMU{0, 0, 0, 1};
  int dw_id = -1, da_id = -1, tg_id = -1, gyro_id = -1;
  double dt_CAMtoIMU = 0;
  int dt_id = -1;
  struct Cam {
    Vec4 q_ItoC{0, 0, 0, 1};
    Vec3 p_IinC{0, 0, 0};
    double intr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int ext_id = -1, intr_id = -1;
    SimCamera model; // State::_cam_intrinsics_cameras: refreshed from intr after every update (StateHelper.cpp:192-196)
  };
  std::vector<Cam> cams;
  std::map<double, ClonePose> clones; // State::_clones_IMU
  std::unordered_map<size_t, SlamLandmark> features_SLAM; // State::_features_SLAM, keyed by feature id
  int base_size = 0;

  int imu_intrinsic_size() const { // State.h:126-135
    int sz = 0;
    if (opt.do_calib_imu_intrinsics) {
      sz += 15;
      if (opt.do_calib_imu_g_sensitivity)
        sz += 9;
    }
    return sz;
  }
  double margtimestep() const { // State.h:66-75
    double time = std::numeric_limits<double>::infinity();
    for (const auto &c : clones)
      if (c.first < time)
        time = c.first;
    return time;
  }
  Mat3 Rot() const { return quat_2_Rot(q); }
  Mat3 Rot_fej() const { return quat_2_Rot(q_fej); }
};

// ---------------------------------------------------------------------------------------------------------------------
// ov_core::FeatureDatabase (feat/FeatureDatabase.cpp); iteration order of the unordered_map is part of the behaviour
class FeatureDatabase {
public:
  std::unordered_map<size_t, std::shared_ptr<Feature>> features_idlookup;

  std::shared_ptr<Feature> get_feature(size_t id) {
    auto it = features_idlookup.find(id);
    return it == features_idlookup.end() ? nullptr : it->second;
  }
  void update_feature(size_t id, double timestamp, size_t cam_id, float u, float v, float u_n, float v_n) { // :59-85
    auto it = features_idlookup.find(id);
    std::shared_ptr<Feature> feat;
    if (it != features_idlookup.end()) {
      feat = it->second;
    } else {
      feat = std::make_shared<Feature>();
      feat->featid = id;
    }
    feat->uvs[cam_id].push_back({u, v});
    feat->uvs_norm[cam_id].push_back({u_n, v_n});
    feat->timestamps[cam_id].push_back(timestamp);
    if (it == features_idlookup.end())
      features_idlookup[id] = feat;
  }
  std::vector<std::shared_ptr<Feature>> features_not_containing_newer(double timestamp, bool remove = false, bool skip_deleted = false) { // :87-125
    std::vector<std::shared_ptr<Feature>> feats_old;
    for (auto it = features_idlookup.begin(); it != features_idlookup.end();) {
      if (skip_deleted && it->second->to_delete) {
        ++it;
        continue;
      }
      bool has_newer_measurement = false;
      for (auto const &pair : it->second->timestamps) {
        has_newer_measurement = (!pair.second.empty() && pair.second.at(pair.second.size() - 1) >= timestamp);
        if (has_newer_measurement)
          break;
      }
      if (!has_newer_measurement) {
        feats_old.push_back(it->second);
        if (remove)
          it = features_idlookup.erase(it);
        else
          ++it;
      } else {
        ++it;
      }
    }
    return feats_old;
  }
  std::vector<std::shared_ptr<Feature>> features_containing(double timestamp, bool remove = false, bool skip_deleted = false) { // :169-207
    std::vector<std::shared_ptr<Feature>> feats_has_timestamp;
    for (auto it = features_idlookup.begin(); it != features_idlookup.end();) {
      if (skip_deleted && it->second->to_delete) {
        ++it;
        continue;
      }
      bool has_timestamp = false;
      for (auto const &pair : it->second->timestamps) {
        has_timestamp = (std::find(pair.second.begin(), pair.second.end(), timestamp) != pair.second.end());
        if (has_timestamp)
          break;
      }
      if (has_timestamp) {
        feats_has_timestamp.push_back(it->second);
        if (remove)
          it = features_idlookup.erase(it);
        else
          ++it;
      } else {
        ++it;
      }
    }
    return feats_has_timestamp;
  }
  void cleanup() { // :211-221
    for (auto it = features_idlookup.begin(); it != features_idlookup.end();) {
      if (it->second->to_delete)
        it = features_idlookup.erase(it);
      else
        ++it;
    }
  }
  // cleanup_measurements (:223-240) with Feature::clean_older_measurements (feat/Feature.cpp:81-110): drop measurements
  // strictly older than `timestamp`, then features without any
  void cleanup_measurements(double timestamp) {
    for (auto it = features_idlookup.begin(); it != features_idlookup.end();) {
      Feature &f = *it->second;
      int ct_meas = 0;
      for (auto &pair : f.timestamps) {
        auto &ts = pair.second;
        auto &uv = f.uvs[pair.first];
        auto &uvn = f.uvs_norm[pair.first];
        size_t w = 0;
        for (size_t i = 0; i < ts.size(); i++) {
          if (!(ts[i] < timestamp)) {
            ts[w] = ts[i];
            uv[w] = uv[i];
            uvn[w] = uvn[i];
            w++;
          }
        }
        ts.resize(w);
        uv.resize(w);
        uvn.resize(w);
        ct_meas += (int)w;
      }
      if (ct_meas < 1)
        it = features_idlookup.erase(it);
      else
        ++it;
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// ov_msckf::Propagator: IMU buffer, mean propagation and the state-transition / noise matrices; the covariance step
// (accumulation over the IMU steps, StateHelper::EKFPropagation and augment_clone) goes through CovBackend::propagate_imu.
class Propagator {
public:
  explicit Propagator(double gravity_mag) : gravity_{0.0, 0.0, gravity_mag} {}

  void feed_imu(const ImuData &message, double oldest_time = -1) { // Propagator.h:65-74
    imu_data.push_back(message);
    clean_old_imu_measurements(oldest_time - 0.10);
  }
  void clean_old_imu_measurements(double oldest_time) { // Propagator.h:80-92
    if (oldest_time < 0)
      return;
    auto it0 = imu_data.begin();
    while (it0 != imu_data.end()) {
      if (it0->timestamp < oldest_time)
        it0 = imu_data.erase(it0);
      else
        ++it0;
    }
  }

  static ImuData interpolate_data(const ImuData &imu_1, const ImuData &imu_2, double timestamp) { // Propagator.h:154-164
    const double lambda = (timestamp - imu_1.timestamp) / (imu_2.timestamp - imu_1.timestamp);
    ImuData data;
    data.timestamp = timestamp;
    data.am = (1 - lambda) * imu_1.am + lambda * imu_2.am;
    data.wm = (1 - lambda) * imu_1.wm + lambda * imu_2.wm;
    return data;
  }

  static std::vector<ImuData> select_imu_readings(const std::vector<ImuData> &imu_data, double time0, double time1) { // Propagator.cpp:269-393
    std::vector<ImuData> prop_data;
    if (imu_data.empty())
      return prop_data;
    for (size_t i = 0; i + 1 < imu_data.size(); i++) {
      if (imu_data[i + 1].timestamp > time0 && imu_data[i].timestamp < time0) {
        prop_data.push_back(interpolate_data(imu_data[i], imu_data[i + 1], time0));
        continue;
      }
      if (imu_data[i].timestamp >= time0 && imu_data[i + 1].timestamp <= time1) {
        prop_data.push_back(imu_data[i]);
        continue;
      }
      if (imu_data[i + 1].timestamp > time1) {
        if (imu_data[i].timestamp > time1 && i == 0) {
          break;
        } else if (imu_data[i].timestamp > time1) {
          prop_data.push_back(interpolate_data(imu_data[i - 1], imu_data[i], time1));
        } else {
          prop_data.push_back(imu_data[i]);
        }
        if (prop_data.back().timestamp != time1)
          prop_data.push_back(interpolate_data(imu_data[i], imu_data[i + 1], time1));
        break;
      }
    }
    if (prop_data.empty())
      return prop_data;
    if (prop_data.back().timestamp != time1)
      prop_data.push_back(interpolate_data(imu_data[imu_data.size() - 2], imu_data[imu_data.size() - 1], time1));
    for (size_t i = 0; i + 1 < prop_data.size(); i++) {
      if (std::abs(prop_data[i + 1].timestamp - prop_data[i].timestamp) < 1e-12) {
        prop_data.erase(prop_data.begin() + (long)i);
        i--;
      }
    }
    if (prop_data.size() < 2)
      prop_data.clear();
    return prop_data;
  }

  // Propagator::propagate_and_clone (Propagator.cpp:33-138)
  void propagate_and_clone(VioState &state, CovBackend &cov, double timestamp) {
    if (state.timestamp == timestamp)
      throw Error(OVB_ERR_ARG, "Propagator::propagate_and_clone(): propagation called again at the same timestep");
    if (state.timestamp > timestamp)
      throw Error(OVB_ERR_ARG, "Propagator::propagate_and_clone(): propagation called trying to propagate backwards in time");
    if (!have_last_prop_time_offset) {
      last_prop_time_offset = state.dt_CAMtoIMU;
      have_last_prop_time_offset = true;
    }
    const double t_off_new = state.dt_CAMtoIMU;
    const double time0 = state.timestamp + last_prop_time_offset;
    const double time1 = timestamp + t_off_new;
    const std::vector<ImuData> prop_data = select_imu_readings(imu_data, time0, time1);
    const int n = state.imu_intrinsic_size() + 15;
    // per-step F, G and noise densities (the mean moves step by step meanwhile); the covariance backend accumulates them
    const int steps = prop_data.size() > 1 ? (int)prop_data.size() - 1 : 0;
    std::vector<double> F_all((size_t)steps * n * n), G_all((size_t)steps * n * 12), qc_all((size_t)steps * 4), F, G;
    for (int i = 0; i < steps; i++) {
      predict_and_compute(state, prop_data[(size_t)i], prop_data[(size_t)i + 1], F, G, &qc_all[(size_t)i * 4]);
      std::copy(F.begin(), F.end(), F_all.begin() + (size_t)i * n * n);
      std::copy(G.begin(), G.end(), G_all.begin() + (size_t)i * n * 12);
    }
    // last angular velocity for the clone's time-offset Jacobian (:104-113)
    Vec3 last_w{0, 0, 0};
    if (!prop_data.empty()) {
      const Mat3 Dw = Simulator::Dm(state.dw), Da = Simulator::Dm(state.da), Tg = Simulator::Tgm(state.tg);
      const Vec3 last_a = quat_2_Rot(state.q_ACCtoIMU) * (Da * (prop_data.back().am - state.ba));
      last_w = quat_2_Rot(state.q_GYROtoIMU) * (Dw * (prop_data.back().wm - state.bg - Tg * last_a));
    }
    // covariance: EKFPropagation over [imu | dw | da | tg | R_GYROtoIMU] (:115-130); all contiguous from the IMU id
    std::vector<int> off{state.imu_id}, sz{15};
    if (state.opt.do_calib_imu_intrinsics) {
      off.push_back(state.dw_id), sz.push_back(6);
      off.push_back(state.da_id), sz.push_back(6);
      if (state.opt.do_calib_imu_g_sensitivity)
        off.push_back(state.tg_id), sz.push_back(9);
      off.push_back(state.gyro_id), sz.push_back(3);
    }
    // StateHelper::augment_clone (StateHelper.cpp:579-616): clone the IMU pose (value and fej), dt Jacobian [last_w; v]
    ClonePose c;
    c.id = cov.dim();
    c.q = state.q, c.p = state.p, c.q_fej = state.q_fej, c.p_fej = state.p_fej;
    if (state.clones.count(timestamp))
      throw Error(OVB_ERR_ARG, "augment_clone: tried to insert a clone at the time of an existing clone");
    double dnc_dt[6] = {last_w[0], last_w[1], last_w[2], state.v[0], state.v[1], state.v[2]};
    cov.propagate_imu(n, steps, F_all, G_all, qc_all, state.imu_id, off, sz, state.imu_id, 6, state.opt.do_calib_camera_timeoffset ? dnc_dt : nullptr,
                      state.dt_id);
    state.timestamp = timestamp;
    last_prop_time_offset = t_off_new;
    state.clones[state.timestamp] = c;
  }

  // Propagator::predict_and_compute (Propagator.cpp:395-480) with the discrete noise Qd = sym(G Qc G'). F, Qd are n x n
  // row-major, n = 15 + imu intrinsics.
  void predict_and_compute(VioState &state, const ImuData &data_minus, const ImuData &data_plus, std::vector<double> &F, std::vector<double> &Qd) {
    std::vector<double> G;
    double qc[4];
    predict_and_compute(state, data_minus, data_plus, F, G, qc);
    imu_discrete_noise(state.imu_intrinsic_size() + 15, G.data(), qc, Qd);
  }
  // ... returning the noise Jacobian G (n x 12, columns [n_w | n_a | n_wb | n_ab]) and the continuous noise
  // Qc = diag(qc[k/3]), qc = sigma^2 / dt (:453-464), of which Qd is made
  void predict_and_compute(VioState &state, const ImuData &data_minus, const ImuData &data_plus, std::vector<double> &F, std::vector<double> &G,
                           double qc[4]) {
    const double dt = data_plus.timestamp - data_minus.timestamp;
    const Mat3 Dw = Simulator::Dm(state.dw), Da = Simulator::Dm(state.da), Tg = Simulator::Tgm(state.tg);
    Vec3 a_hat1 = data_minus.am - state.ba, a_hat2 = data_plus.am - state.ba;
    Vec3 a_hat_avg = .5 * (a_hat1 + a_hat2);
    const Vec3 a_uncorrected = a_hat_avg;
    const Mat3 R_ACCtoIMU = quat_2_Rot(state.q_ACCtoIMU);
    a_hat1 = R_ACCtoIMU * (Da * a_hat1);
    a_hat2 = R_ACCtoIMU * (Da * a_hat2);
    a_hat_avg = R_ACCtoIMU * (Da * a_hat_avg);
    Vec3 w_hat1 = data_minus.wm - state.bg - Tg * a_hat1, w_hat2 = data_plus.wm - state.bg - Tg * a_hat2;
    Vec3 w_hat_avg = .5 * (w_hat1 + w_hat2);
    const Vec3 w_uncorrected = w_hat_avg;
    const Mat3 R_GYROtoIMU = quat_2_Rot(state.q_GYROtoIMU);
    w_hat1 = R_GYROtoIMU * (Dw * w_hat1);
    w_hat2 = R_GYROtoIMU * (Dw * w_hat2);
    w_hat_avg = R_GYROtoIMU * (Dw * w_hat_avg);
    XiSum Xi;
    const bool analytic = state.opt.integration_method == INTEGRATION_RK4 || state.opt.integration_method == INTEGRATION_ANALYTICAL;
    if (analytic)
      compute_Xi_sum(dt, w_hat_avg, a_hat_avg, Xi);
    Vec4 new_q;
    Vec3 new_v, new_p;
    if (state.opt.integration_method == INTEGRATION_ANALYTICAL)
      predict_mean_analytic(state, dt, a_hat_avg, new_q, new_v, new_p, Xi);
    else if (state.opt.integration_method == INTEGRATION_RK4)
      predict_mean_rk4(state, dt, w_hat1, a_hat1, w_hat2, a_hat2, new_q, new_v, new_p);
    else
      predict_mean_discrete(state, dt, w_hat_avg, a_hat_avg, new_q, new_v, new_p);
    const int n = state.imu_intrinsic_size() + 15;
    F.assign((size_t)n * n, 0.0);
    G.assign((size_t)n * 12, 0.0);
    compute_F_and_G(state, analytic, dt, w_uncorrected, a_uncorrected, new_q, new_v, new_p, Xi, F, G, n);
    // Qc = diag(sigma^2 / dt) (:453-464)
    qc[0] = state.opt.sigma_w * state.opt.sigma_w / dt, qc[1] = state.opt.sigma_a * state.opt.sigma_a / dt;
    qc[2] = state.opt.sigma_wb * state.opt.sigma_wb / dt, qc[3] = state.opt.sigma_ab * state.opt.sigma_ab / dt;
    // replace the IMU estimate and its FEJ with the propagated values (:471-479)
    state.q = state.q_fej = new_q;
    state.p = state.p_fej = new_p;
    state.v = state.v_fej = new_v;
  }

  std::vector<ImuData> imu_data;

private:
  Vec3 gravity_;
  bool have_last_prop_time_offset = false;
  double last_prop_time_offset = 0;
  struct XiSum {
    Mat3 R_ktok1 = eye3(), Xi_1 = zero3(), Xi_2 = zero3(), Jr_ktok1 = eye3(), Xi_3 = zero3(), Xi_4 = zero3();
  };

  static void put3(std::vector<double> &M, int ld, int r, int c, const Mat3 &B) {
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        M[(size_t)(r + i) * ld + c + j] = B[(size_t)i * 3 + j];
  }

  void predict_mean_discrete(const VioState &state, double dt, const Vec3 &w_hat, const Vec3 &a_hat, Vec4 &new_q, Vec3 &new_v, Vec3 &new_p) const { // :482-508
    const double w_norm = norm(w_hat);
    const Mat3 R_Gtoi = state.Rot();
    Vec4 bq;
    const Vec4 Oq = Omega_times(w_hat, state.q);
    if (w_norm > 1e-12) {
      const double c = std::cos(0.5 * w_norm * dt), s = 1 / w_norm * std::sin(0.5 * w_norm * dt);
      for (int i = 0; i < 4; i++)
        bq[(size_t)i] = c * state.q[(size_t)i] + s * Oq[(size_t)i];
    } else {
      for (int i = 0; i < 4; i++)
        bq[(size_t)i] = state.q[(size_t)i] + 0.5 * dt * Oq[(size_t)i];
    }
    new_q = quatnorm(bq);
    new_v = state.v + transpose(R_Gtoi) * a_hat * dt - gravity_ * dt;
    new_p = state.p + state.v * dt + 0.5 * (transpose(R_Gtoi) * a_hat) * dt * dt - 0.5 * gravity_ * dt * dt;
  }

  void predict_mean_rk4(const VioState &state, double dt, const Vec3 &w_hat1, const Vec3 &a_hat1, const Vec3 &w_hat2, const Vec3 &a_hat2, Vec4 &new_q,
                        Vec3 &new_v, Vec3 &new_p) const { // :510-598
    Vec3 w_hat = w_hat1, a_hat = a_hat1;
    const Vec3 w_alpha = (1.0 / dt) * (w_hat2 - w_hat1), a_jerk = (1.0 / dt) * (a_hat2 - a_hat1);
    const Vec4 q_0 = state.q;
    const Vec3 p_0 = state.p, v_0 = state.v;
    auto scale4 = [](double s, const Vec4 &a) { return Vec4{s * a[0], s * a[1], s * a[2], s * a[3]}; };
    auto add4 = [](const Vec4 &a, const Vec4 &b) { return Vec4{a[0] + b[0], a[1] + b[1], a[2] + b[2], a[3] + b[3]}; };
    // k1
    const Vec4 dq_0{0, 0, 0, 1};
    const Vec4 q0_dot = scale4(0.5, Omega_times(w_hat, dq_0));
    const Vec3 p0_dot = v_0;
    const Mat3 R_Gto0 = quat_2_Rot(quat_multiply(dq_0, q_0));
    const Vec3 v0_dot = transpose(R_Gto0) * a_hat - gravity_;
    const Vec4 k1_q = scale4(dt, q0_dot);
    const Vec3 k1_p = p0_dot * dt, k1_v = v0_dot * dt;
    // k2
    w_hat += 0.5 * w_alpha * dt;
    a_hat += 0.5 * a_jerk * dt;
    const Vec4 dq_1 = quatnorm(add4(dq_0, scale4(0.5, k1_q)));
    const Vec3 v_1 = v_0 + 0.5 * k1_v;
    const Vec4 q1_dot = scale4(0.5, Omega_times(w_hat, dq_1));
    const Vec3 p1_dot = v_1;
    const Mat3 R_Gto1 = quat_2_Rot(quat_multiply(dq_1, q_0));
    const Vec3 v1_dot = transpose(R_Gto1) * a_hat - gravity_;
    const Vec4 k2_q = scale4(dt, q1_dot);
    const Vec3 k2_p = p1_dot * dt, k2_v = v1_dot * dt;
    // k3
    const Vec4 dq_2 = quatnorm(add4(dq_0, scale4(0.5, k2_q)));
    const Vec3 v_2 = v_0 + 0.5 * k2_v;
    const Vec4 q2_dot = scale4(0.5, Omega_times(w_hat, dq_2));
    const Vec3 p2_dot = v_2;
    const Mat3 R_Gto2 = quat_2_Rot(quat_multiply(dq_2, q_0));
    const Vec3 v2_dot = transpose(R_Gto2) * a_hat - gravity_;
    const Vec4 k3_q = scale4(dt, q2_dot);
    const Vec3 k3_p = p2_dot * dt, k3_v = v2_dot * dt;
    // k4
    w_hat += 0.5 * w_alpha * dt;
    a_hat += 0.5 * a_jerk * dt;
    const Vec4 dq_3 = quatnorm(add4(dq_0, k3_q));
    const Vec3 v_3 = v_0 + k3_v;
    const Vec4 q3_dot = scale4(0.5, Omega_times(w_hat, dq_3));
    const Vec3 p3_dot = v_3;
    const Mat3 R_Gto3 = quat_2_Rot(quat_multiply(dq_3, q_0));
    const Vec3 v3_dot = transpose(R_Gto3) * a_hat - gravity_;
    const Vec4 k4_q = scale4(dt, q3_dot);
    const Vec3 k4_p = p3_dot * dt, k4_v = v3_dot * dt;
    // y+dt
    const Vec4 dq = quatnorm(add4(add4(add4(add4(dq_0, scale4(1.0 / 6.0, k1_q)), scale4(1.0 / 3.0, k2_q)), scale4(1.0 / 3.0, k3_q)), scale4(1.0 / 6.0, k4_q)));
    new_q = quat_multiply(dq, q_0);
    new_p = p_0 + (1.0 / 6.0) * k1_p + (1.0 / 3.0) * k2_p + (1.0 / 3.0) * k3_p + (1.0 / 6.0) * k4_p;
    new_v = v_0 + (1.0 / 6.0) * k1_v + (1.0 / 3.0) * k2_v + (1.0 / 3.0) * k3_v + (1.0 / 6.0) * k4_v;
  }

  static void compute_Xi_sum(double dt, const Vec3 &w_hat, const Vec3 &a_hat, XiSum &X) { // :600-667
    const double w_norm = norm(w_hat), d_th = w_norm * dt;
    Vec3 k_hat{0, 0, 0};
    if (w_norm > 1e-12)
      k_hat = (1.0 / w_norm) * w_hat;
    const Mat3 I = eye3();
    const double d_t2 = std::pow(dt, 2), d_t3 = std::pow(dt, 3), w_norm2 = std::pow(w_norm, 2), w_norm3 = std::pow(w_norm, 3);
    const double cos_dth = std::cos(d_th), sin_dth = std::sin(d_th), d_th2 = std::pow(d_th, 2), d_th3 = std::pow(d_th, 3);
    const Mat3 sK = skew_x(k_hat), sK2 = sK * sK, sA = skew_x(a_hat);
    X.R_ktok1 = exp_so3(-(w_hat * dt));
    X.Jr_ktok1 = Jr_so3(-(w_hat * dt));
    const bool small_w = (w_norm < 1.0 / 180 * M_PI / 2);
    const double ka = dot(k_hat, a_hat);
    if (!small_w) {
      X.Xi_1 = dt * I + ((1.0 - cos_dth) / w_norm) * sK + (dt - sin_dth / w_norm) * sK2;
      X.Xi_2 = (1.0 / 2 * d_t2) * I + ((d_th - sin_dth) / w_norm2) * sK + (1.0 / 2 * d_t2 - (1.0 - cos_dth) / w_norm2) * sK2;
      X.Xi_3 = (1.0 / 2 * d_t2) * sA + ((sin_dth - d_th) / w_norm2) * (sA * sK) + ((sin_dth - d_th * cos_dth) / w_norm2) * (sK * sA) +
               (1.0 / 2 * d_t2 - (1.0 - cos_dth) / w_norm2) * (sA * sK2) +
               (1.0 / 2 * d_t2 + (1.0 - cos_dth - d_th * sin_dth) / w_norm2) * (sK2 * sA + ka * sK) -
               ((3 * sin_dth - 2 * d_th - d_th * cos_dth) / w_norm2 * ka) * sK2;
      X.Xi_4 = (1.0 / 6 * d_t3) * sA + ((2 * (1.0 - cos_dth) - d_th2) / (2 * w_norm3)) * (sA * sK) +
               ((2 * (1.0 - cos_dth) - d_th * sin_dth) / w_norm3) * (sK * sA) + ((sin_dth - d_th) / w_norm3 + d_t3 / 6) * (sA * sK2) +
               ((d_th - 2 * sin_dth + 1.0 / 6 * d_th3 + d_th * cos_dth) / w_norm3) * (sK2 * sA + ka * sK) +
               ((4 * cos_dth - 4 + d_th2 + d_th * sin_dth) / w_norm3 * ka) * sK2;
    } else {
      X.Xi_1 = dt * (I + sin_dth * sK + (1.0 - cos_dth) * sK2);
      X.Xi_2 = (1.0 / 2 * dt) * X.Xi_1;
      X.Xi_3 = (1.0 / 2 * d_t2) * (sA + sin_dth * (-(sA * sK) + sK * sA + ka * sK2) + (1.0 - cos_dth) * (sA * sK2 + sK2 * sA + ka * sK));
      X.Xi_4 = (1.0 / 3 * dt) * X.Xi_3;
    }
  }

  void predict_mean_analytic(const VioState &state, double dt, const Vec3 &a_hat, Vec4 &new_q, Vec3 &new_v, Vec3 &new_p, const XiSum &X) const { // :669-681
    const Mat3 R_Gtok = state.Rot();
    const Vec4 q_ktok1 = rot_2_quat(X.R_ktok1);
    new_q = quat_multiply(q_ktok1, state.q);
    new_v = state.v + transpose(R_Gtok) * (X.Xi_1 * a_hat) - gravity_ * dt;
    new_p = state.p + state.v * dt + transpose(R_Gtok) * (X.Xi_2 * a_hat) - 0.5 * gravity_ * dt * dt;
  }

  // compute_F_and_G_analytic (:683-828) / compute_F_and_G_discrete (:830-950); KALIBR model (th_wtoI block present)
  void compute_F_and_G(const VioState &state, bool analytic, double dt, const Vec3 &w_uncorrected, const Vec3 &a_uncorrected, const Vec4 &new_q,
                       const Vec3 &new_v, const Vec3 &new_p, const XiSum &X, std::vector<double> &F, std::vector<double> &G, int n) const {
    const int th_id = 0, p_id = 3, v_id = 6, bg_id = 9, ba_id = 12;
    int Dw_id = -1, Da_id = -1, Tg_id = -1, th_wtoI_id = -1, local = 15;
    if (state.opt.do_calib_imu_intrinsics) {
      Dw_id = local, local += 6;
      Da_id = local, local += 6;
      if (state.opt.do_calib_imu_g_sensitivity)
        Tg_id = local, local += 9;
      th_wtoI_id = local, local += 3;
    }
    Mat3 R_k = state.Rot();
    Vec3 v_k = state.v, p_k = state.p;
    if (state.opt.do_fej) {
      R_k = state.Rot_fej();
      v_k = state.v_fej;
      p_k = state.p_fej;
    }
    const Mat3 dR_ktok1 = quat_2_Rot(new_q) * transpose(R_k);
    const Mat3 Dw = Simulator::Dm(state.dw), Da = Simulator::Dm(state.da), Tg = Simulator::Tgm(state.tg);
    const Mat3 R_atoI = quat_2_Rot(state.q_ACCtoIMU), R_wtoI = quat_2_Rot(state.q_GYROtoIMU);
    const Vec3 a_k = R_atoI * (Da * a_uncorrected);
    const Vec3 w_k = R_wtoI * (Dw * w_uncorrected);
    const Mat3 Rkt = transpose(R_k);
    const Mat3 Jr = analytic ? X.Jr_ktok1 : Jr_so3(log_so3(dR_ktok1));
    const Mat3 dRJdt = dt * (dR_ktok1 * Jr);
    const Mat3 RwDw = R_wtoI * Dw, RaDa = R_atoI * Da;
    put3(F, n, th_id, th_id, dR_ktok1);
    put3(F, n, p_id, th_id, -(skew_x(new_p - p_k - v_k * dt + 0.5 * gravity_ * dt * dt) * Rkt));
    put3(F, n, v_id, th_id, -(skew_x(new_v - v_k + gravity_ * dt) * Rkt));
    put3(F, n, p_id, p_id, eye3());
    put3(F, n, p_id, v_id, dt * eye3());
    put3(F, n, v_id, v_id, eye3());
    put3(F, n, bg_id, bg_id, eye3());
    put3(F, n, ba_id, ba_id, eye3());
    put3(F, n, th_id, bg_id, -(dRJdt * RwDw));
    put3(F, n, th_id, ba_id, dRJdt * RwDw * Tg * RaDa);
    Mat3 P_a, V_a, P_w, V_w; // position / velocity sensitivities to (corrected) acceleration and angular-rate perturbations
    if (analytic) {
      P_w = Rkt * X.Xi_4, V_w = Rkt * X.Xi_3;
      P_a = Rkt * (X.Xi_2 + X.Xi_4 * RwDw * Tg), V_a = Rkt * (X.Xi_1 + X.Xi_3 * RwDw * Tg);
      put3(F, n, p_id, bg_id, P_w * RwDw);
      put3(F, n, v_id, bg_id, V_w * RwDw);
    } else {
      P_w = zero3(), V_w = zero3();
      P_a = (0.5 * dt * dt) * Rkt, V_a = dt * Rkt;
    }
    put3(F, n, p_id, ba_id, -(P_a * RaDa));
    put3(F, n, v_id, ba_id, -(V_a * RaDa));
    auto put3xk = [&](int r, int c, const Mat3 &L, const double *H, int k, double sign) { // F[r.., c..] = sign * L (3x3) * H (3 x k)
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < k; j++)
          F[(size_t)(r + i) * n + c + j] = sign * (L[(size_t)i * 3] * H[j] + L[(size_t)i * 3 + 1] * H[k + j] + L[(size_t)i * 3 + 2] * H[2 * k + j]);
    };
    if (Dw_id != -1) { // compute_H_Dw (:952-971), KALIBR: [w1 I, w2 e2, w2 e3, w3 e3]
      const double w1 = w_uncorrected[0], w2 = w_uncorrected[1], w3 = w_uncorrected[2];
      const double H[18] = {w1, 0, 0, 0, 0, 0, 0, w1, 0, w2, 0, 0, 0, 0, w1, 0, w2, w3};
      put3xk(th_id, Dw_id, dRJdt * R_wtoI, H, 6, 1.0);
      if (analytic) {
        put3xk(p_id, Dw_id, P_w * R_wtoI, H, 6, -1.0);
        put3xk(v_id, Dw_id, V_w * R_wtoI, H, 6, -1.0);
      }
      for (int i = 0; i < 6; i++)
        F[(size_t)(Dw_id + i) * n + Dw_id + i] = 1.0;
    }
    if (Da_id != -1) { // compute_H_Da (:973-992)
      const double a1 = a_uncorrected[0], a2 = a_uncorrected[1], a3 = a_uncorrected[2];
      const double H[18] = {a1, 0, 0, 0, 0, 0, 0, a1, 0, a2, 0, 0, 0, 0, a1, 0, a2, a3};
      // the discrete variant omits Dw in the orientation block (:905): -dR Jr dt R_wtoI Tg R_atoI H_Da
      put3xk(th_id, Da_id, analytic ? dRJdt * RwDw * Tg * R_atoI : dRJdt * R_wtoI * Tg * R_atoI, H, 6, -1.0);
      put3xk(p_id, Da_id, P_a * R_atoI, H, 6, 1.0);
      put3xk(v_id, Da_id, V_a * R_atoI, H, 6, 1.0);
      for (int i = 0; i < 6; i++)
        F[(size_t)(Da_id + i) * n + Da_id + i] = 1.0;
    }
    if (Tg_id != -1) { // compute_H_Tg (:994-1015): [a1 I, a2 I, a3 I]
      const double H[27] = {a_k[0], 0, 0, a_k[1], 0, 0, a_k[2], 0, 0, 0, a_k[0], 0, 0, a_k[1], 0, 0, a_k[2], 0, 0, 0, a_k[0], 0, 0, a_k[1], 0, 0, a_k[2]};
      put3xk(th_id, Tg_id, dRJdt * RwDw, H, 9, -1.0);
      if (analytic) {
        put3xk(p_id, Tg_id, P_w * RwDw, H, 9, 1.0);
        put3xk(v_id, Tg_id, V_w * RwDw, H, 9, 1.0);
      }
      for (int i = 0; i < 9; i++)
        F[(size_t)(Tg_id + i) * n + Tg_id + i] = 1.0;
    }
    if (th_wtoI_id != -1) {
      put3(F, n, th_id, th_wtoI_id, dRJdt * skew_x(w_k));
      if (analytic) {
        put3(F, n, p_id, th_wtoI_id, -(P_w * skew_x(w_k)));
        put3(F, n, v_id, th_wtoI_id, -(V_w * skew_x(w_k)));
      }
      put3(F, n, th_wtoI_id, th_wtoI_id, eye3());
    }
    // G: columns [n_w | n_a | n_wb | n_ab]
    put3(G, 12, th_id, 0, -(dRJdt * RwDw));
    put3(G, 12, th_id, 3, dRJdt * RwDw * Tg * RaDa);
    if (analytic) {
      put3(G, 12, p_id, 0, P_w * RwDw);
      put3(G, 12, v_id, 0, V_w * RwDw);
    }
    put3(G, 12, p_id, 3, -(P_a * RaDa));
    put3(G, 12, v_id, 3, -(V_a * RaDa));
    put3(G, 12, bg_id, 6, dt * eye3());
    put3(G, 12, ba_id, 9, dt * eye3());
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// timing row of VioManager (core/VioManager.cpp:604-644) and trajectory sample for the evaluation
struct FrameTiming {
  double timestamp_inI = 0, time_track = 0, time_prop = 0, time_msckf = 0, time_slam_update = 0, time_slam_delayed = 0, time_marg = 0, time_total = 0;
  int feats_in = 0, feats_used = 0, rows = 0, cols = 0;
  int slam_live = 0; // landmarks in the state at the end of the frame
};
// what one frame did with the SLAM landmarks (VioManager::record_slam_frames; feature ids throughout)
struct SlamFrameRecord {
  double t = 0, since_start = 0; // the frame's time, and the time since the filter started (what dt_slam_delay is checked against)
  int N = 0, n_clones = 0;
  std::vector<size_t> msckf, slam_update, delayed, marginalized, initialized;
  std::vector<size_t> promoted; // from feats_maxtracks
  // the landmarks at the end of the frame: featid, covariance id, size, anchor clone in the window (1/0; -1 = global)
  std::vector<std::array<long, 4>> landmarks;
  std::vector<std::pair<size_t, int>> marg_fail_count; // update_fail_count of each landmark marginalize_slam removed
};
struct TrajSample {
  double t = 0;
  Vec4 q{0, 0, 0, 1};
  Vec3 p{0, 0, 0};
};

// VioManager reduced to the rpng_sim path (TrackSIM front-end, ground-truth initialisation, MSCKF updates)
class VioManager {
public:
  VioState state;
  std::shared_ptr<CovBackend> cov;
  Propagator propagator;
  FeatureDatabase database;
  std::vector<FrameTiming> timing;
  std::vector<TrajSample> trajectory_est;
  ovb_stats last_stats{};
  // optional hook: called with the marshalled inputs of every MSCKF update before it runs (capture of update cases)
  std::function<void(const ovb_frame &, const ovb_feat_batch &, const ovb_opts &, int frame_index)> on_update;
  int frames_done = 0;
  long status_hist[16] = {0}; // ovb_feat_status histogram over all updates (diagnostics)
  long slam_status_hist[16] = {0}, init_status_hist[16] = {0}; // the same over the SLAM updates / the delayed initialisations
  long slam_initialized = 0, slam_marginalized = 0, anchor_changes = 0;
  bool record_slam_frames = false; // keep one SlamFrameRecord per frame in slam_frames (tests)
  std::vector<SlamFrameRecord> slam_frames;

  VioManager(const VioOptions &opt, const SimParams &calib, std::shared_ptr<CovBackend> backend)
      : cov(std::move(backend)), propagator(opt.gravity_mag) {
    // State::State (state/State.cpp:28-131): variable order and ids
    state.opt = opt;
    int id = 0;
    state.imu_id = id, id += 15;
    if (opt.do_calib_imu_intrinsics) {
      state.dw_id = id, id += 6;
      state.da_id = id, id += 6;
      if (opt.do_calib_imu_g_sensitivity)
        state.tg_id = id, id += 9;
      state.gyro_id = id, id += 3; // KALIBR: R_GYROtoIMU
    }
    if (opt.do_calib_camera_timeoffset)
      state.dt_id = id, id += 1;
    state.cams.resize((size_t)opt.num_cameras);
    for (int i = 0; i < opt.num_cameras; i++) {
      auto &c = state.cams[(size_t)i];
      if (opt.do_calib_camera_pose)
        c.ext_id = id, id += 6;
      if (opt.do_calib_camera_intrinsics)
        c.intr_id = id, id += 8;
      // VioManager::VioManager loads the calibration into the state (core/VioManager.cpp:69-90)
      c.q_ItoC = calib.camera_extrinsics[(size_t)i].first;
      c.p_IinC = calib.camera_extrinsics[(size_t)i].second;
      std::memcpy(c.intr, calib.camera_intrinsics[(size_t)i].d, sizeof(c.intr));
      c.model = calib.camera_intrinsics[(size_t)i];
    }
    state.dt_CAMtoIMU = calib.calib_camimu_dt;
    std::memcpy(state.dw, calib.vec_dw, sizeof(state.dw));
    std::memcpy(state.da, calib.vec_da, sizeof(state.da));
    std::memcpy(state.tg, calib.vec_tg, sizeof(state.tg));
    state.q_GYROtoIMU = calib.q_GYROtoIMU;
    state.q_ACCtoIMU = calib.q_ACCtoIMU;
    state.base_size = id;
    // initial covariance (State.cpp:134-165)
    const int N = id;
    std::vector<double> P((size_t)N * N, 0.0);
    auto diag = [&](int off, int n, double sigma) {
      for (int k = 0; k < n; k++)
        P[(size_t)(off + k) * N + off + k] = sigma * sigma;
    };
    diag(0, N, 1e-3);
    if (opt.do_calib_imu_intrinsics) {
      diag(state.dw_id, 6, 0.005);
      diag(state.da_id, 6, 0.008);
      if (opt.do_calib_imu_g_sensitivity)
        diag(state.tg_id, 9, 0.005);
      diag(state.gyro_id, 3, 0.005);
    }
    if (opt.do_calib_camera_timeoffset)
      diag(state.dt_id, 1, 0.01);
    for (auto &c : state.cams) {
      if (opt.do_calib_camera_pose) {
        diag(c.ext_id, 3, 0.005);
        diag(c.ext_id + 3, 3, 0.015);
      }
      if (opt.do_calib_camera_intrinsics) {
        diag(c.intr_id, 4, 1.0);
        diag(c.intr_id + 4, 4, 0.005);
      }
    }
    P0_ = P;
  }

  // VioManager::initialize_with_gt (core/VioManagerHelper.cpp:40-76): imustate = [t q p v bg ba]
  void initialize_with_gt(const std::array<double, 17> &imustate) {
    state.q = state.q_fej = {imustate[1], imustate[2], imustate[3], imustate[4]};
    state.p = state.p_fej = {imustate[5], imustate[6], imustate[7]};
    state.v = state.v_fej = {imustate[8], imustate[9], imustate[10]};
    state.bg = {imustate[11], imustate[12], imustate[13]};
    state.ba = {imustate[14], imustate[15], imustate[16]};
    const int N = state.base_size;
    std::vector<double> P = P0_;
    for (int k = 0; k < 15; k++) {
      const double s = k < 3 ? 0.017 : (k < 6 ? 0.05 : (k < 9 ? 0.01 : 0.02));
      for (int j = 0; j < 15; j++)
        P[(size_t)k * N + j] = P[(size_t)j * N + k] = 0.0;
      P[(size_t)k * N + k] = s * s;
    }
    cov->set(P, N);
    state.timestamp = imustate[0];
    startup_time = imustate[0];
    is_initialized_vio = true;
    database.cleanup_measurements(state.timestamp);
  }

  void feed_measurement_imu(const ImuData &message) { // core/VioManager.cpp:166-189
    double oldest_time = state.margtimestep();
    if (oldest_time > state.timestamp)
      oldest_time = -1;
    propagator.feed_imu(message, oldest_time);
  }

  // VioManager::feed_measurement_simulation (:191-254) with TrackSIM::feed_measurement_simulation (track/TrackSIM.cpp:30-79)
  void feed_measurement_simulation(double timestamp, const std::vector<int> &camids, const std::vector<std::vector<SimFeat>> &feats) {
    const auto rT1 = clock_now();
    for (size_t i = 0; i < camids.size(); i++) {
      const int cam_id = camids[i];
      for (const auto &feat : feats[i]) {
        float xn, yn;
        state.cams[(size_t)cam_id].model.undistort_f(feat.u, feat.v, xn, yn); // camera_calib.at(cam_id)->undistort_cv
        database.update_feature(feat.id, timestamp, (size_t)cam_id, feat.u, feat.v, xn, yn);
      }
    }
    const auto rT2 = clock_now();
    if (!is_initialized_vio)
      throw Error(OVB_ERR_ARG, "[SIM]: your vio system should already be initialized before simulating features");
    do_feature_propagate_update(timestamp, camids, rT1, rT2);
  }

  // ov_eval: position ATE RMSE with alignment "none" (ResultTrajectory.cpp:82-109 after AlignTrajectory "none")
  static void calculate_ate(const std::vector<TrajSample> &est, const std::vector<TrajSample> &gt, double &rmse_ori_deg, double &rmse_pos) {
    double so = 0, sp = 0;
    const size_t n = std::min(est.size(), gt.size());
    for (size_t i = 0; i < n; i++) {
      const Mat3 e_R = transpose(quat_2_Rot(est[i].q)) * quat_2_Rot(gt[i].q);
      const double ori_err = 180.0 / M_PI * norm(log_so3(e_R));
      const double pos_err = norm(gt[i].p - est[i].p);
      so += ori_err * ori_err;
      sp += pos_err * pos_err;
    }
    rmse_ori_deg = n ? std::sqrt(so / (double)n) : 0.0;
    rmse_pos = n ? std::sqrt(sp / (double)n) : 0.0;
  }

  // timing file in the reference's format (core/VioManager.cpp:117-121 header, :631-644 rows; the SLAM columns only when
  // max_slam_features > 0)
  void write_timing_csv(const std::string &path) const {
    FILE *f = std::fopen(path.c_str(), "w");
    if (!f)
      return;
    const bool slam = state.opt.max_slam_features > 0;
    std::fprintf(f, "# timestamp (sec),tracking,propagation,msckf update,%smarginalization,total\n", slam ? "slam update,slam delayed," : "");
    for (const auto &t : timing) {
      std::fprintf(f, "%.15f,%.5f,%.5f,%.5f,", t.timestamp_inI, t.time_track, t.time_prop, t.time_msckf);
      if (slam)
        std::fprintf(f, "%.5f,%.5f,", t.time_slam_update, t.time_slam_delayed);
      std::fprintf(f, "%.5f,%.5f\n", t.time_marg, t.time_total);
    }
    std::fclose(f);
  }

private:
  std::vector<double> P0_;
  bool is_initialized_vio = false;
  double startup_time = -1;
  using clk = std::chrono::steady_clock;
  static clk::time_point clock_now() { return clk::now(); }
  static double secs(clk::time_point a, clk::time_point b) { return std::chrono::duration<double>(b - a).count(); }

  // VioManager::do_feature_propagate_update (:323-644)
  void do_feature_propagate_update(double timestamp, const std::vector<int> &sensor_ids, clk::time_point rT1, clk::time_point rT2) {
    if (state.timestamp > timestamp)
      return; // image received out of order
    if (state.timestamp != timestamp)
      propagator.propagate_and_clone(state, *cov, timestamp);
    const auto rT3 = clock_now();
    if ((int)state.clones.size() < std::min(state.opt.max_clone_size, 5))
      return;
    if (state.timestamp != timestamp)
      return;
    // ---- feature selection (:368-453, :509-524)
    std::vector<std::shared_ptr<Feature>> feats_lost, feats_marg;
    feats_lost = database.features_not_containing_newer(state.timestamp, false, true);
    if ((int)state.clones.size() > state.opt.max_clone_size || (int)state.clones.size() > 5)
      feats_marg = database.features_containing(state.margtimestep(), false, true);
    for (auto it1 = feats_lost.begin(); it1 != feats_lost.end();) { // keep features seen from a camera of this message
      bool found = false;
      for (const auto &camuvpair : (*it1)->uvs)
        if (std::find(sensor_ids.begin(), sensor_ids.end(), (int)camuvpair.first) != sensor_ids.end()) {
          found = true;
          break;
        }
      it1 = found ? it1 + 1 : feats_lost.erase(it1);
    }
    for (auto it1 = feats_lost.begin(); it1 != feats_lost.end();) // no duplicates with the marg list
      it1 = (std::find(feats_marg.begin(), feats_marg.end(), *it1) != feats_marg.end()) ? feats_lost.erase(it1) : it1 + 1;
    std::vector<std::shared_ptr<Feature>> feats_maxtracks;
    for (auto it2 = feats_marg.begin(); it2 != feats_marg.end();) {
      bool reached_max = false;
      for (const auto &cams : (*it2)->timestamps)
        if ((int)cams.second.size() > state.opt.max_clone_size) {
          reached_max = true;
          break;
        }
      if (reached_max) {
        feats_maxtracks.push_back(*it2);
        it2 = feats_marg.erase(it2);
      } else {
        ++it2;
      }
    }
    // ---- SLAM features (:455-507). The runner has no ArUco tracker, so no landmark is a tag: the reference's featid tests
    // against 4 * max_aruco_features (which count feature 0 as a tag when max_aruco_features = 0) are left out.
    SlamFrameRecord rec;
    std::vector<std::shared_ptr<Feature>> feats_slam;
    const int max_slam = state.opt.max_slam_features;
    if (max_slam > 0 && timestamp - startup_time >= state.opt.dt_slam_delay && (int)state.features_SLAM.size() < max_slam) {
      // the reference takes them from the end of feats_maxtracks
      const int valid_amount = std::min(max_slam - (int)state.features_SLAM.size(), (int)feats_maxtracks.size());
      if (valid_amount > 0) {
        feats_slam.insert(feats_slam.end(), feats_maxtracks.end() - valid_amount, feats_maxtracks.end());
        feats_maxtracks.erase(feats_maxtracks.end() - valid_amount, feats_maxtracks.end());
      }
    }
    for (const auto &f : feats_slam)
      rec.promoted.push_back(f->featid);
    for (auto &lm : state.features_SLAM) { // the landmarks' tracks of this frame; lost or twice-failed landmarks are flagged
      std::shared_ptr<Feature> feat2 = database.get_feature(lm.second.featid);
      if (feat2)
        feats_slam.push_back(feat2);
      const bool current_unique_cam = std::find(sensor_ids.begin(), sensor_ids.end(), lm.second.unique_camera_id) != sensor_ids.end();
      if (!feat2 && current_unique_cam)
        lm.second.should_marg = true;
      if (lm.second.update_fail_count > 1)
        lm.second.should_marg = true;
    }
    // StateHelper::marginalize_slam where the reference calls it (:497): a landmark dropped here whose track goes on is
    // initialised again by delayed_init below, in this frame
    marginalize_slam(rec);
    std::vector<std::shared_ptr<Feature>> feats_slam_DELAYED, feats_slam_UPDATE;
    for (const auto &f : feats_slam)
      (state.features_SLAM.count(f->featid) ? feats_slam_UPDATE : feats_slam_DELAYED).push_back(f);
    std::vector<std::shared_ptr<Feature>> featsup_MSCKF = feats_lost;
    featsup_MSCKF.insert(featsup_MSCKF.end(), feats_marg.begin(), feats_marg.end());
    featsup_MSCKF.insert(featsup_MSCKF.end(), feats_maxtracks.begin(), feats_maxtracks.end());
    // the reference sorts by track length with std::sort (unstable) on an unordered_map-ordered list: ties are
    // implementation-defined there; a stable sort keyed (length, featid) gives both backends one total order (SURVEY.md App. A.5)
    auto nmeas = [](const std::shared_ptr<Feature> &a) {
      size_t s = 0;
      for (const auto &pair : a->timestamps)
        s += pair.second.size();
      return s;
    };
    std::stable_sort(featsup_MSCKF.begin(), featsup_MSCKF.end(), [&](const std::shared_ptr<Feature> &a, const std::shared_ptr<Feature> &b) {
      const size_t na = nmeas(a), nb = nmeas(b);
      return na != nb ? na < nb : a->featid < b->featid;
    });
    if ((int)featsup_MSCKF.size() > state.opt.max_msckf_in_update)
      featsup_MSCKF.erase(featsup_MSCKF.begin(), featsup_MSCKF.end() - state.opt.max_msckf_in_update);
    FrameTiming ft;
    ft.feats_in = (int)featsup_MSCKF.size();
    if (record_slam_frames)
      for (const auto &f : featsup_MSCKF)
        rec.msckf.push_back(f->featid);
    msckf_update(featsup_MSCKF);
    ft.feats_used = last_stats.n_feats_used, ft.rows = last_stats.rows_stacked, ft.cols = last_stats.cols_stacked;
    const auto rT4 = clock_now();
    // UpdaterSLAM::update in batches of max_slam_in_update (:531-545), then delayed_init (:547)
    for (const auto &f : feats_slam_UPDATE)
      rec.slam_update.push_back(f->featid);
    for (size_t b = 0; b < feats_slam_UPDATE.size(); b += (size_t)state.opt.max_slam_in_update) {
      std::vector<std::shared_ptr<Feature>> batch(feats_slam_UPDATE.begin() + (long)b,
                                                  feats_slam_UPDATE.begin() + (long)std::min(b + (size_t)state.opt.max_slam_in_update, feats_slam_UPDATE.size()));
      slam_update(batch);
    }
    const auto rT5 = clock_now();
    for (const auto &f : feats_slam_DELAYED)
      rec.delayed.push_back(f->featid);
    delayed_init(feats_slam_DELAYED, rec);
    const auto rT6 = clock_now();
    for (auto const &feat : featsup_MSCKF)
      feat->to_delete = true;
    database.cleanup();
    if ((int)state.clones.size() > state.opt.max_clone_size)
      database.cleanup_measurements(state.margtimestep());
    change_anchors_and_marginalize_old_clone();
    const auto rT7 = clock_now();
    ft.timestamp_inI = state.timestamp + state.dt_CAMtoIMU;
    ft.time_track = secs(rT1, rT2), ft.time_prop = secs(rT2, rT3), ft.time_msckf = secs(rT3, rT4), ft.time_slam_update = secs(rT4, rT5);
    ft.time_slam_delayed = secs(rT5, rT6), ft.time_marg = secs(rT6, rT7), ft.time_total = secs(rT1, rT7);
    ft.slam_live = (int)state.features_SLAM.size();
    timing.push_back(ft);
    trajectory_est.push_back({state.timestamp, state.q, state.p});
    if (record_slam_frames) {
      rec.t = state.timestamp, rec.since_start = timestamp - startup_time, rec.N = cov->dim(), rec.n_clones = (int)state.clones.size();
      for (const auto &lm : state.features_SLAM)
        rec.landmarks.push_back({(long)lm.first, lm.second.id, lm.second.size(),
                                 SlamLandmark::anchored(lm.second.rep) ? (long)state.clones.count(lm.second.anchor_clone_timestamp) : -1L});
      slam_frames.push_back(std::move(rec));
    }
    frames_done++;
  }

  // ---- marshalling of the state and of feature tracks into the ABI's structs; every backend call of a frame goes through these
  // the window and the cameras (UpdaterMSCKF.cpp:98-115 read exactly these); the clone times give the clone indices.
  // Marshalling again into the same FrameMarshal rewrites its arrays in place, so `frame` keeps pointing at them.
  struct FrameMarshal {
    std::vector<double> clonetimes, cR, cp, cRf, cpf, kR, kp, kin, cq, kq;
    std::vector<int> coff, kmodel, kext, kintr;
    ovb_frame frame{};
    ovb_frame_quat quat{}; // the quaternions behind cR and kR
  };
  void marshal_frame(FrameMarshal &m) const {
    const int C = (int)state.clones.size(), K = (int)state.cams.size();
    m.clonetimes.resize((size_t)C), m.cR.resize((size_t)9 * C), m.cp.resize((size_t)3 * C), m.cRf.resize((size_t)9 * C), m.cpf.resize((size_t)3 * C);
    m.kR.resize((size_t)9 * K), m.kp.resize((size_t)3 * K), m.kin.resize((size_t)8 * K), m.cq.resize((size_t)4 * C), m.kq.resize((size_t)4 * K);
    m.coff.resize((size_t)C), m.kmodel.resize((size_t)K), m.kext.resize((size_t)K), m.kintr.resize((size_t)K);
    int c = 0;
    for (const auto &cl : state.clones) {
      const Mat3 R = quat_2_Rot(cl.second.q), Rf = quat_2_Rot(cl.second.q_fej);
      m.clonetimes[(size_t)c] = cl.first;
      std::copy(R.begin(), R.end(), m.cR.begin() + 9 * c);
      std::copy(Rf.begin(), Rf.end(), m.cRf.begin() + 9 * c);
      std::copy(cl.second.q.begin(), cl.second.q.end(), m.cq.begin() + 4 * c);
      std::copy(cl.second.p.begin(), cl.second.p.end(), m.cp.begin() + 3 * c);
      std::copy(cl.second.p_fej.begin(), cl.second.p_fej.end(), m.cpf.begin() + 3 * c);
      m.coff[(size_t)c] = cl.second.id;
      c++;
    }
    for (int k = 0; k < K; k++) {
      const auto &cam = state.cams[(size_t)k];
      const Mat3 R = quat_2_Rot(cam.q_ItoC);
      std::copy(R.begin(), R.end(), m.kR.begin() + 9 * k);
      std::copy(cam.q_ItoC.begin(), cam.q_ItoC.end(), m.kq.begin() + 4 * k);
      std::copy(cam.p_IinC.begin(), cam.p_IinC.end(), m.kp.begin() + 3 * k);
      std::copy(cam.intr, cam.intr + 8, m.kin.begin() + 8 * k);
      m.kmodel[(size_t)k] = cam.model.model;
      m.kext[(size_t)k] = state.opt.do_calib_camera_pose ? cam.ext_id : -1;
      m.kintr[(size_t)k] = state.opt.do_calib_camera_intrinsics ? cam.intr_id : -1;
    }
    m.frame = ovb_frame{C,       K,         m.cR.data(),  m.cp.data(),     m.cRf.data(),   m.cpf.data(), m.coff.data(),
                        m.kR.data(), m.kp.data(), m.kin.data(), m.kmodel.data(), m.kext.data(), m.kintr.data()};
    m.quat = ovb_frame_quat{m.cq.data(), m.kq.data()};
  }
  // the tracks as a structure of arrays: cameras in the visit order of the unordered_map (SURVEY.md App. A.4)
  struct FeatMarshal {
    std::vector<int32_t> meas_off{0}, keys_off{0};
    std::vector<uint8_t> cam, keys;
    std::vector<uint16_t> clone;
    std::vector<float> uv, uvn;
    ovb_feat_batch batch{};
  };
  static void marshal_feats(const std::vector<std::shared_ptr<Feature>> &feature_vec, const std::vector<double> &clonetimes, FeatMarshal &b) {
    for (const auto &feat : feature_vec) {
      for (const auto &pair : feat->timestamps) {
        b.keys.push_back((uint8_t)pair.first);
        const auto &fuv = feat->uvs.at(pair.first);
        const auto &fuvn = feat->uvs_norm.at(pair.first);
        for (size_t m = 0; m < pair.second.size(); m++) {
          const int ci = (int)(std::lower_bound(clonetimes.begin(), clonetimes.end(), pair.second[m]) - clonetimes.begin());
          b.cam.push_back((uint8_t)pair.first);
          b.clone.push_back((uint16_t)ci);
          b.uv.push_back(fuv[m][0]), b.uv.push_back(fuv[m][1]);
          b.uvn.push_back(fuvn[m][0]), b.uvn.push_back(fuvn[m][1]);
        }
      }
      b.meas_off.push_back((int32_t)b.cam.size());
      b.keys_off.push_back((int32_t)b.keys.size());
    }
    b.batch = ovb_feat_batch{(int)feature_vec.size(), (int)b.cam.size(), b.meas_off.data(), b.cam.data(),     b.clone.data(),
                             b.uv.data(),             b.uvn.data(),      b.keys_off.data(), b.keys.data()};
  }
  // FeatureInitializerOptions + the MSCKF UpdaterOptions + the StateOptions fields; `slam` puts the SLAM noise and gate in
  ovb_opts make_opts(bool slam = false) const {
    ovb_opts o;
    ovb_opts_default(&o);
    const auto &fi = state.opt.featinit_options;
    o.triangulate_1d = fi.triangulate_1d, o.refine_features = fi.refine_features, o.max_runs = fi.max_runs;
    o.init_lamda = fi.init_lamda, o.max_lamda = fi.max_lamda, o.min_dx = fi.min_dx, o.min_dcost = fi.min_dcost, o.lam_mult = fi.lam_mult;
    o.min_dist = fi.min_dist, o.max_dist = fi.max_dist, o.max_baseline = fi.max_baseline, o.max_cond_number = fi.max_cond_number;
    const UpdaterOptions &u = slam ? state.opt.slam_options : state.opt.msckf_options;
    o.sigma_pix = u.sigma_pix;
    o.chi2_multipler = u.chi2_multipler;
    o.do_fej = state.opt.do_fej;
    o.feat_rep = state.opt.feat_rep_msckf;
    o.do_calib_camera_pose = state.opt.do_calib_camera_pose;
    o.do_calib_camera_intrinsics = state.opt.do_calib_camera_intrinsics;
    o.col_order = state.opt.col_order;
    o.compress = state.opt.compress;
    return o;
  }
  // Feature::clean_old_measurements to the clone times; a track with fewer than `min_meas` measurements leaves the list and
  // is marked to_delete (UpdaterMSCKF.cpp:75-94, UpdaterSLAM.cpp:75-90)
  static void clean_to_clones(std::vector<std::shared_ptr<Feature>> &feature_vec, const std::vector<double> &clonetimes, int min_meas) {
    for (auto it = feature_vec.begin(); it != feature_vec.end();) {
      (*it)->clean_old_measurements(clonetimes);
      int ct_meas = 0;
      for (const auto &pair : (*it)->timestamps)
        ct_meas += (int)pair.second.size();
      if (ct_meas < min_meas) {
        (*it)->to_delete = true;
        it = feature_vec.erase(it);
      } else {
        ++it;
      }
    }
  }

  // UpdaterMSCKF::update (update/UpdaterMSCKF.cpp:58-295): host steps 0-1, marshalling, device pipeline, mean update
  void msckf_update(std::vector<std::shared_ptr<Feature>> &feature_vec) {
    last_stats = ovb_stats{};
    if (feature_vec.empty())
      return;
    FrameMarshal m;
    marshal_frame(m);
    clean_to_clones(feature_vec, m.clonetimes, 2);
    if (feature_vec.empty())
      return;
    const int N = cov->dim();
    FeatMarshal b;
    marshal_feats(feature_vec, m.clonetimes, b);
    const ovb_opts o = make_opts();
    if (on_update)
      on_update(m.frame, b.batch, o, frames_done);
    const int F = (int)feature_vec.size();
    std::vector<int32_t> status((size_t)F), acam((size_t)F), aclone((size_t)F);
    std::vector<double> pA((size_t)3 * F), pG((size_t)3 * F), chi2((size_t)F), dx((size_t)N, 0.0);
    ovb_feat_out out{status.data(), pA.data(), pG.data(), acam.data(), aclone.data(), chi2.data()};
    cov->msckf_update(&m.frame, &b.batch, &o, &out, dx.data(), &last_stats);
    for (int f = 0; f < F; f++) {
      Feature &feat = *feature_vec[(size_t)f];
      feat.last_status = status[(size_t)f];
      feat.last_chi2 = chi2[(size_t)f];
      feat.to_delete = true;
      status_hist[status[(size_t)f] & 15]++;
    }
    apply_dx(dx.data());
  }

  // UpdaterSLAM::update (update/UpdaterSLAM.cpp:253-479) on one batch: tracks without measurements at the clone times are
  // dropped and deleted, a single-depth landmark needs two (:278-290); a landmark that fails the gate counts the failure
  // (:409-420); every track used ends to_delete (:452-454)
  void slam_update(std::vector<std::shared_ptr<Feature>> &feature_vec) {
    FrameMarshal m;
    marshal_frame(m);
    clean_to_clones(feature_vec, m.clonetimes, 1);
    for (auto it = feature_vec.begin(); it != feature_vec.end();) {
      int ct_meas = 0;
      for (const auto &pair : (*it)->timestamps)
        ct_meas += (int)pair.second.size();
      const bool single = state.features_SLAM.at((*it)->featid).rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE;
      it = single && ct_meas < 2 ? feature_vec.erase(it) : it + 1;
    }
    if (feature_vec.empty())
      return;
    FeatMarshal b;
    marshal_feats(feature_vec, m.clonetimes, b);
    const int F = (int)feature_vec.size(), N = cov->dim();
    std::vector<int32_t> lm_off, reps, acam, aclone;
    std::vector<double> val, val_fej;
    for (const auto &feat : feature_vec) {
      const SlamLandmark &lm = state.features_SLAM.at(feat->featid);
      lm_off.push_back(lm.id);
      reps.push_back(lm.rep);
      const Vec3 v = lm.get_xyz(false), vf = lm.get_xyz(true);
      val.insert(val.end(), v.begin(), v.end());
      val_fej.insert(val_fej.end(), vf.begin(), vf.end());
      acam.push_back(lm.anchor_cam_id);
      aclone.push_back(SlamLandmark::anchored(lm.rep)
                           ? (int32_t)(std::lower_bound(m.clonetimes.begin(), m.clonetimes.end(), lm.anchor_clone_timestamp) - m.clonetimes.begin())
                           : -1);
    }
    ovb_landmarks lms{lm_off.data(), val.data(), val_fej.data(), acam.data(), aclone.data(), nullptr, nullptr};
    const ovb_opts o = make_opts(true);
    std::vector<int32_t> status((size_t)F), ocam((size_t)F), oclone((size_t)F);
    std::vector<double> pA((size_t)3 * F), pG((size_t)3 * F), chi2((size_t)F), dx((size_t)N, 0.0);
    ovb_feat_out out{status.data(), pA.data(), pG.data(), ocam.data(), oclone.data(), chi2.data()};
    ovb_stats st{};
    cov->slam_update(&m.frame, &b.batch, &lms, reps.data(), &o, &out, dx.data(), &st);
    for (int f = 0; f < F; f++) {
      Feature &feat = *feature_vec[(size_t)f];
      feat.last_status = status[(size_t)f];
      feat.last_chi2 = chi2[(size_t)f];
      feat.to_delete = true;
      slam_status_hist[status[(size_t)f] & 15]++;
      if (status[(size_t)f] == OVB_FEAT_CHI2)
        state.features_SLAM.at(feat.featid).update_fail_count++;
    }
    apply_dx(dx.data());
  }

  // UpdaterSLAM::delayed_init (update/UpdaterSLAM.cpp:61-251): tracks cleaned to the clone times (two measurements at least),
  // then one backend call triangulates them all and initialises them one after the other, moving its copy of the frame in
  // between; its records are replayed here in feature order. Every track ends to_delete, initialised or not.
  void delayed_init(std::vector<std::shared_ptr<Feature>> &feature_vec, SlamFrameRecord &rec) {
    if (feature_vec.empty())
      return;
    FrameMarshal m;
    marshal_frame(m);
    clean_to_clones(feature_vec, m.clonetimes, 2);
    if (feature_vec.empty())
      return;
    FeatMarshal b;
    marshal_feats(feature_vec, m.clonetimes, b);
    const int F = (int)feature_vec.size();
    const std::vector<int32_t> reps((size_t)F, state.opt.feat_rep_slam);
    const ovb_opts o = make_opts(true);
    std::vector<int32_t> status((size_t)F), acam((size_t)F), aclone((size_t)F), lm_off((size_t)F);
    std::vector<double> pA((size_t)3 * F), pG((size_t)3 * F), chi2((size_t)F);
    ovb_feat_out out{status.data(), pA.data(), pG.data(), acam.data(), aclone.data(), chi2.data()};
    const int ld_dx = cov->dim() + 3 * F;
    std::vector<double> dx_new((size_t)3 * F), dx((size_t)F * ld_dx);
    cov->slam_delayed_init_batch(&m.frame, &m.quat, &b.batch, &o, reps.data(), nullptr, nullptr, &out, lm_off.data(), dx_new.data(), dx.data(), ld_dx);
    for (int f = 0; f < F; f++)
      if (lm_off[(size_t)f] >= 0)
        init_landmark(feature_vec[(size_t)f]->featid, out, f, m.clonetimes, lm_off[(size_t)f], &dx_new[(size_t)3 * f], &dx[(size_t)f * ld_dx], rec);
    for (int f = 0; f < F; f++) {
      feature_vec[(size_t)f]->last_status = status[(size_t)f];
      feature_vec[(size_t)f]->to_delete = true;
      init_status_hist[status[(size_t)f] & 15]++;
    }
  }
  // what StateHelper::initialize leaves behind for an accepted feature (UpdaterSLAM.cpp:190-238, StateHelper.cpp:540-577):
  // the new landmark at its triangulated point moved by dx_new, then every variable, the landmark included, moved by dx
  void init_landmark(size_t featid, const ovb_feat_out &out, int f, const std::vector<double> &clonetimes, int lm_off, const double *dx_new,
                     const double *dx, SlamFrameRecord &rec) {
    SlamLandmark lm;
    lm.featid = featid;
    lm.rep = state.opt.feat_rep_slam;
    lm.unique_camera_id = out.anchor_cam[f];
    const double *p = out.p_FinG + 3 * f;
    if (SlamLandmark::anchored(lm.rep)) {
      lm.anchor_cam_id = out.anchor_cam[f];
      lm.anchor_clone_timestamp = clonetimes[(size_t)out.anchor_clone[f]];
      p = out.p_FinA + 3 * f;
    }
    lm.set_from_xyz({p[0], p[1], p[2]}, false);
    lm.set_from_xyz({p[0], p[1], p[2]}, true);
    lm.update(dx_new);
    lm.id = lm_off;
    state.features_SLAM[lm.featid] = lm;
    apply_dx(dx);
    slam_initialized++;
    rec.initialized.push_back(lm.featid);
  }

  // every id behind a removed block moves up by its size, once per block (StateHelper.cpp:318-326); the base state's ids lie
  // in front of every clone and landmark
  void shift_ids(const std::vector<int32_t> &off, const std::vector<int32_t> &sz) {
    auto shift = [&](int &id) {
      int d = 0;
      for (size_t i = 0; i < off.size(); i++)
        if (id > off[i])
          d += sz[i];
      id -= d;
    };
    for (auto &c : state.clones)
      shift(c.second.id);
    for (auto &lm : state.features_SLAM)
      shift(lm.second.id);
  }

  // StateHelper::marginalize_slam (state/StateHelper.cpp): the flagged landmarks leave the state in one marginalize_window
  // call without anchor changes; no call when none is flagged
  void marginalize_slam(SlamFrameRecord &rec) {
    std::vector<int32_t> off, sz;
    std::vector<size_t> lost;
    for (const auto &lm : state.features_SLAM)
      if (lm.second.should_marg) {
        off.push_back(lm.second.id);
        sz.push_back(lm.second.size());
        lost.push_back(lm.first);
        rec.marginalized.push_back(lm.first);
        rec.marg_fail_count.push_back({lm.first, lm.second.update_fail_count});
      }
    if (lost.empty())
      return;
    FrameMarshal m;
    marshal_frame(m);
    const ovb_opts o = make_opts();
    cov->marginalize_window(&m.frame, &o, off.data(), sz.data(), (int)off.size(), nullptr);
    for (size_t id : lost)
      state.features_SLAM.erase(id);
    shift_ids(off, sz);
    slam_marginalized += (long)lost.size();
  }

  // UpdaterSLAM::change_anchors (UpdaterSLAM.cpp:481-504) + StateHelper::marginalize_old_clone (StateHelper.cpp:618-629) in
  // one marginalize_window call once the window is full: every anchored landmark of the oldest clone moves to the newest
  // clone, same camera, then the oldest clone leaves the state
  void change_anchors_and_marginalize_old_clone() {
    if ((int)state.clones.size() <= state.opt.max_clone_size)
      return;
    FrameMarshal m;
    marshal_frame(m);
    const double marg_t = state.margtimestep(), new_t = state.timestamp;
    const int C = (int)state.clones.size();
    std::vector<SlamLandmark *> moved;
    std::vector<int32_t> lm_off, reps, ocam, oclone, ncam, nclone;
    std::vector<double> val, val_fej;
    for (auto &f : state.features_SLAM) {
      SlamLandmark &lm = f.second;
      if (!SlamLandmark::anchored(lm.rep) || lm.anchor_clone_timestamp != marg_t)
        continue;
      moved.push_back(&lm);
      lm_off.push_back(lm.id), reps.push_back(lm.rep);
      ocam.push_back(lm.anchor_cam_id), oclone.push_back(0), ncam.push_back(lm.anchor_cam_id), nclone.push_back(C - 1);
      const Vec3 v = lm.get_xyz(false), vf = lm.get_xyz(true);
      val.insert(val.end(), v.begin(), v.end());
      val_fej.insert(val_fej.end(), vf.begin(), vf.end());
    }
    const int n = (int)moved.size();
    std::vector<double> nv((size_t)3 * n), nvf((size_t)3 * n);
    ovb_anchor_changes an{n, lm_off.data(), reps.data(), val.data(), val_fej.data(), ocam.data(), oclone.data(), ncam.data(), nclone.data(), nv.data(), nvf.data()};
    const std::vector<int32_t> off{state.clones.at(marg_t).id}, sz{6};
    const ovb_opts o = make_opts();
    cov->marginalize_window(&m.frame, &o, off.data(), sz.data(), 1, n ? &an : nullptr);
    for (int l = 0; l < n; l++) { // perform_anchor_change's set_from_xyz in the new anchor (:636-641)
      moved[(size_t)l]->set_from_xyz({nv[(size_t)3 * l], nv[(size_t)3 * l + 1], nv[(size_t)3 * l + 2]}, false);
      moved[(size_t)l]->set_from_xyz({nvf[(size_t)3 * l], nvf[(size_t)3 * l + 1], nvf[(size_t)3 * l + 2]}, true);
      moved[(size_t)l]->anchor_clone_timestamp = new_t;
    }
    anchor_changes += n;
    state.clones.erase(marg_t);
    shift_ids(off, sz);
  }

  // the mean side of StateHelper::EKFUpdate (state/StateHelper.cpp:185-196): Type::update of every variable
  void apply_dx(const double *dx) {
    auto qupdate = jpl_update;
    const double *d = dx + state.imu_id; // IMU::update (types/IMU.h:78-96)
    qupdate(state.q, d);
    for (int k = 0; k < 3; k++) {
      state.p[(size_t)k] += d[3 + k];
      state.v[(size_t)k] += d[6 + k];
      state.bg[(size_t)k] += d[9 + k];
      state.ba[(size_t)k] += d[12 + k];
    }
    if (state.opt.do_calib_imu_intrinsics) {
      for (int k = 0; k < 6; k++) {
        state.dw[k] += dx[state.dw_id + k];
        state.da[k] += dx[state.da_id + k];
      }
      if (state.opt.do_calib_imu_g_sensitivity)
        for (int k = 0; k < 9; k++)
          state.tg[k] += dx[state.tg_id + k];
      qupdate(state.q_GYROtoIMU, dx + state.gyro_id);
    }
    if (state.opt.do_calib_camera_timeoffset)
      state.dt_CAMtoIMU += dx[state.dt_id];
    for (auto &c : state.cams) {
      if (state.opt.do_calib_camera_pose) { // PoseJPL::update (types/PoseJPL.h:74-91)
        qupdate(c.q_ItoC, dx + c.ext_id);
        for (int k = 0; k < 3; k++)
          c.p_IinC[(size_t)k] += dx[c.ext_id + 3 + k];
      }
      if (state.opt.do_calib_camera_intrinsics) {
        for (int k = 0; k < 8; k++)
          c.intr[k] += dx[c.intr_id + k];
        std::memcpy(c.model.d, c.intr, sizeof(c.intr)); // StateHelper.cpp:192-196
      }
    }
    for (auto &cl : state.clones) {
      qupdate(cl.second.q, dx + cl.second.id);
      for (int k = 0; k < 3; k++)
        cl.second.p[(size_t)k] += dx[cl.second.id + 3 + k];
    }
    for (auto &lm : state.features_SLAM) // Landmark::update
      lm.second.update(dx + lm.second.id);
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// Filter consistency (the reference's Monte-Carlo studies: sim_save_total_state_to_file, then ov_eval's NEES and ±3σ
// plots): per frame, the error of every base-state variable against the truth in the convention of P's error state, the
// base block's σ, and the NEES of the IMU orientation and position (3 DOF each). The base state is one contiguous block
// of P, ids [0, base_size): IMU 15 | dw 6 | da 6 | tg 9 | R_GYROtoIMU 3 | dt 1 | per camera: extrinsics 6, intrinsics 8.
struct ConsistencySample {
  double t = 0, nees_ori = 0, nees_pos = 0;
  double cov6[21] = {0};          // upper triangle of the 6x6 [theta, p] IMU block, row by row
  std::vector<double> err, sigma; // base_size each: truth (-) estimate, sqrt(P_ii)
};

// orientation error of a JPL quaternion in P's convention: updates are q <- dq(dtheta) ⊗ q (JPLQuat::update), so
// q_true = dq(dtheta) ⊗ q_est gives R_true = exp(-[dtheta]x) R_est and dtheta = -log(R_true R_est')
inline Vec3 ori_error(const Vec4 &q_true, const Vec4 &q_est) { return -log_so3(quat_2_Rot(q_true) * transpose(quat_2_Rot(q_est))); }

// x' A^-1 x for the symmetric 3x3 block A of a row-major matrix with leading dimension lda, through A = L L' (no inverse);
// NaN when the block is not positive definite
inline double nees3(const double *A, int lda, const Vec3 &x) {
  double L[3][3] = {{0}};
  for (int j = 0; j < 3; j++) {
    double d = A[(size_t)j * lda + j];
    for (int k = 0; k < j; k++)
      d -= L[j][k] * L[j][k];
    if (!(d > 0))
      return std::numeric_limits<double>::quiet_NaN();
    L[j][j] = std::sqrt(d);
    for (int i = j + 1; i < 3; i++) {
      double s = A[(size_t)i * lda + j];
      for (int k = 0; k < j; k++)
        s -= L[i][k] * L[j][k];
      L[i][j] = s / L[j][j];
    }
  }
  double y[3], r = 0; // L y = x, then x' A^-1 x = |y|^2
  for (int i = 0; i < 3; i++) {
    double s = x[(size_t)i];
    for (int k = 0; k < i; k++)
      s -= L[i][k] * y[k];
    y[i] = s / L[i][i];
    r += y[i] * y[i];
  }
  return r;
}

// one frame: `st` after the update and the clone marginalization, `gt` = Simulator::get_state's [t q p v bg ba] at the
// frame's IMU time, `truth` = Simulator::get_true_parameters (with sim_do_perturbation the filter starts from a perturbed
// copy), P = the base block [0, base_size)^2 of the covariance, row-major
inline ConsistencySample consistency_sample(const VioState &st, const SimParams &truth, const std::array<double, 17> &gt, const std::vector<double> &P) {
  const int n = st.base_size;
  ConsistencySample s;
  s.t = st.timestamp;
  s.err.assign((size_t)n, 0.0);
  s.sigma.assign((size_t)n, 0.0);
  auto put3 = [&](int id, const Vec3 &e) {
    for (int k = 0; k < 3; k++)
      s.err[(size_t)(id + k)] = e[(size_t)k];
  };
  auto diff = [&](int id, int m, const double *tru, const double *est) {
    for (int k = 0; k < m; k++)
      s.err[(size_t)(id + k)] = tru[k] - est[k];
  };
  const int i = st.imu_id;
  put3(i, ori_error({gt[1], gt[2], gt[3], gt[4]}, st.q));
  put3(i + 3, Vec3{gt[5], gt[6], gt[7]} - st.p);
  put3(i + 6, Vec3{gt[8], gt[9], gt[10]} - st.v);
  put3(i + 9, Vec3{gt[11], gt[12], gt[13]} - st.bg);
  put3(i + 12, Vec3{gt[14], gt[15], gt[16]} - st.ba);
  if (st.dw_id >= 0) {
    diff(st.dw_id, 6, truth.vec_dw, st.dw);
    diff(st.da_id, 6, truth.vec_da, st.da);
  }
  if (st.tg_id >= 0)
    diff(st.tg_id, 9, truth.vec_tg, st.tg);
  if (st.gyro_id >= 0)
    put3(st.gyro_id, ori_error(truth.q_GYROtoIMU, st.q_GYROtoIMU));
  if (st.dt_id >= 0)
    diff(st.dt_id, 1, &truth.calib_camimu_dt, &st.dt_CAMtoIMU);
  for (size_t c = 0; c < st.cams.size(); c++) {
    const auto &cam = st.cams[c];
    if (cam.ext_id >= 0) {
      put3(cam.ext_id, ori_error(truth.camera_extrinsics[c].first, cam.q_ItoC));
      put3(cam.ext_id + 3, truth.camera_extrinsics[c].second - cam.p_IinC);
    }
    if (cam.intr_id >= 0)
      diff(cam.intr_id, 8, truth.camera_intrinsics[c].d, cam.intr);
  }
  for (int k = 0; k < n; k++)
    s.sigma[(size_t)k] = std::sqrt(P[(size_t)k * n + k]);
  for (int a = 0, u = 0; a < 6; a++)
    for (int b = a; b < 6; b++)
      s.cov6[u++] = P[(size_t)(i + a) * n + i + b];
  s.nees_ori = nees3(P.data() + (size_t)i * n + i, n, {s.err[(size_t)i], s.err[(size_t)i + 1], s.err[(size_t)i + 2]});
  s.nees_pos = nees3(P.data() + (size_t)(i + 3) * n + i + 3, n, {s.err[(size_t)i + 3], s.err[(size_t)i + 4], s.err[(size_t)i + 5]});
  return s;
}

// the consistency file: a '#' header with the layout and the variable ids, then one row per frame:
// t nees_ori nees_pos cov6[21] err[n] sigma[n]
inline void write_consistency_file(const std::string &path, const VioState &st, const std::vector<ConsistencySample> &rows) {
  FILE *f = std::fopen(path.c_str(), "w");
  if (!f)
    return;
  std::fprintf(f, "# t nees_ori nees_pos cov6[21] err[n] sigma[n] | cov6: upper triangle of the [theta p] IMU block, row by row | err: truth - "
                  "estimate, orientations -log(R_true R_est') | ids: imu=%d",
               st.imu_id);
  if (st.dw_id >= 0)
    std::fprintf(f, " dw=%d da=%d", st.dw_id, st.da_id);
  if (st.tg_id >= 0)
    std::fprintf(f, " tg=%d", st.tg_id);
  if (st.gyro_id >= 0)
    std::fprintf(f, " gyro=%d", st.gyro_id);
  if (st.dt_id >= 0)
    std::fprintf(f, " dt=%d", st.dt_id);
  for (size_t c = 0; c < st.cams.size(); c++) {
    if (st.cams[c].ext_id >= 0)
      std::fprintf(f, " cam%zu_ext=%d", c, st.cams[c].ext_id);
    if (st.cams[c].intr_id >= 0)
      std::fprintf(f, " cam%zu_intr=%d", c, st.cams[c].intr_id);
  }
  std::fprintf(f, " n=%d\n", st.base_size);
  for (const auto &r : rows) {
    std::fprintf(f, "%.9f %.17g %.17g", r.t, r.nees_ori, r.nees_pos);
    for (double x : r.cov6)
      std::fprintf(f, " %.17g", x);
    for (double x : r.err)
      std::fprintf(f, " %.17g", x);
    for (double x : r.sigma)
      std::fprintf(f, " %.17g", x);
    std::fprintf(f, "\n");
  }
  std::fclose(f);
}

// ---------------------------------------------------------------------------------------------------------------------
// run_simulation main loop (ov_msckf/src/run_simulation.cpp:117-176): initialise from the simulator's ground truth, feed
// IMU at sim_freq_imu and camera frames with the reference's one-frame delay buffer. Stops after max_frames camera updates
// (0 = whole trajectory). Ground truth samples are taken at the estimate's timestamps (+dt) from the simulator's spline.
// record_consistency: after every frame, outside the frame's timed region, read the base block of P (one
// get_marginal) and append a ConsistencySample; off, the loop makes exactly the backend calls it makes without it.
struct SimRunResult {
  std::vector<TrajSample> est, gt;
  double ate_ori_deg = 0, ate_pos = 0;
  int frames = 0;
  std::vector<ConsistencySample> consistency;
};
inline SimRunResult run_simulation(Simulator &sim, VioManager &sys, int max_frames = 0, bool record_consistency = false) {
  const double next_imu_time = sim.current_timestamp() + 1.0 / sim.params.sim_freq_imu;
  std::array<double, 17> imustate;
  if (!sim.get_state(next_imu_time, imustate))
    throw Error(OVB_ERR_ARG, "[SIM]: could not initialize the filter to the first state");
  const SimParams &truth = sim.get_true_parameters();
  imustate[0] -= truth.calib_camimu_dt;
  sys.initialize_with_gt(imustate);
  double buffer_timecam = -1;
  std::vector<int> buffer_camids;
  std::vector<std::vector<SimFeat>> buffer_feats;
  SimRunResult res;
  while (sim.ok()) {
    ImuData message_imu;
    if (sim.get_next_imu(message_imu.timestamp, message_imu.wm, message_imu.am))
      sys.feed_measurement_imu(message_imu);
    double time_cam;
    std::vector<int> camids;
    std::vector<std::vector<SimFeat>> feats;
    if (sim.get_next_cam(time_cam, camids, feats)) {
      if (buffer_timecam != -1) {
        const size_t before = sys.trajectory_est.size();
        sys.feed_measurement_simulation(buffer_timecam, buffer_camids, buffer_feats);
        if (sys.trajectory_est.size() > before) {
          std::array<double, 17> gt;
          const TrajSample &e = sys.trajectory_est.back();
          const bool have_gt = sim.get_state(e.t + truth.calib_camimu_dt, gt);
          if (have_gt)
            res.gt.push_back({e.t, {gt[1], gt[2], gt[3], gt[4]}, {gt[5], gt[6], gt[7]}});
          else
            res.gt.push_back(e);
          if (record_consistency) {
            const VioState &st = sys.state;
            if (!have_gt) // past the trajectory's end: like the ATE, the estimate stands in for the truth
              gt = {st.timestamp, st.q[0], st.q[1], st.q[2], st.q[3], st.p[0], st.p[1], st.p[2], st.v[0], st.v[1], st.v[2],
                    st.bg[0], st.bg[1], st.bg[2], st.ba[0], st.ba[1], st.ba[2]};
            res.consistency.push_back(consistency_sample(st, truth, gt, sys.cov->get_marginal({0}, {st.base_size})));
          }
        }
        if (max_frames > 0 && sys.frames_done >= max_frames)
          break;
      }
      buffer_timecam = time_cam;
      buffer_camids = camids;
      buffer_feats = feats;
    }
  }
  res.est = sys.trajectory_est;
  res.frames = sys.frames_done;
  VioManager::calculate_ate(res.est, res.gt, res.ate_ori_deg, res.ate_pos);
  return res;
}

} // namespace ovb200
#endif
