// run_simulation.cpp — rpng_sim runner (ov_msckf/src/run_simulation.cpp) on the host layer of include/ovb200_vio.hpp.
//   ovb_run_simulation   (this file, -DOVB_SIM_ENGINE): covariance and MSCKF updates on the CUDA engine (libovb200.so)
//   tests/cpp/run_simulation_oracle (same file, -DOVB_SIM_ORACLE, test infrastructure): the CPU oracle behind the same interface
//   -DOVB_SIM_HOST_PROPAGATION (test infrastructure): the engine with the IMU covariance accumulation on the host
// Usage: <exe> --traj FILE(.txt|.bin) [--cams K] [--clones C] [--msckf M] [--pts P] [--frames F] [--calib 0|1]
//              [--est OUT.txt] [--timing [OUT.csv]] [--capture FRAME PREFIX] [--integration discrete|rk4|analytical]
//              [--seed-init S] [--seed-perturb S] [--seed-meas S] [--runs K [--jobs J] [--out-dir DIR]] [--consistency [OUT.txt]]
//              [--cam-model M[,M...]] [--slam M [--slam-in-update U] [--slam-delay S] [--feat-rep-slam NAME] [--slam-log OUT.txt]]
//              [--perturb] [--feat-rep-msckf NAME] [--use-fej 0|1] [--fi-triangulate-1d 0|1] [--fi-refine-features 0|1]
//              [--up-msckf-sigma-px X] [--up-msckf-chi2-multipler X] [--up-slam-sigma-px X] [--up-slam-chi2-multipler X]
//              [--calib-cam-extrinsics 0|1] [--calib-cam-intrinsics 0|1] [--calib-cam-timeoffset 0|1] [--calib-imu-intrinsics 0|1]
//              [--calib-imu-g-sensitivity 0|1]
// Prints one JSON line: frames, ATE (alignment none), mean per-stage host times.
// --cam-model radtan|equi: the camera model of every camera, or one per camera (a mixed rig, e.g. radtan,equi). Equidistant
// cameras take the TUM-VI cam0 intrinsics on a 512 x 512 image and the rpng_sim extrinsics of their slot (rpng_sim_cameras
// in include/ovb200_sim.hpp); the JSON line gains "cam_model", one entry per camera. Without the flag every camera is the
// rpng_sim radtan camera.
// --consistency OUT.txt: after every frame, read the base block of the covariance and write one row of errors against the
// truth, σ and the orientation / position NEES (write_consistency_file in include/ovb200_vio.hpp; INTEGRATION.md §8); the
// JSON line gains the run's mean nees_ori and nees_pos. With --runs, --consistency takes no path: DIR/consistency_<seed>.txt
// per run, nees_ori / nees_pos per run and their mean and population standard deviation over the runs.
// --runs K: a Monte-Carlo batch of K runs in this process, run r with measurement seed seed_meas + r (same map and initial
// state, different noise). J host threads (default min(K, hardware threads)) take runs from a shared counter; each run owns
// its Simulator, VioManager and backend (with the engine: its own ovb_ctx on device 0), so a run computes the same bits
// whether it runs alone or beside others. Per run, DIR/est_<seed>.txt and, with --timing, DIR/timing_<seed>.csv. The JSON
// line then lists every run and the mean / population standard deviation of both ATEs, the wall time and runs/s.
// --slam M: at most M SLAM landmarks in the state (StateOptions::max_slam_features; 0 = MSCKF only, the default), updated in
// batches of --slam-in-update U (25), promoted from --slam-delay S seconds after the start (1), every landmark in --feat-rep-slam
// NAME (GLOBAL_3D; one of the six ovb_feat_rep names). The timing CSV gains the "slam update" and "slam delayed" columns when
// M > 0; so does the JSON line (and every per_run entry), which gains the SLAM and delayed-init status histograms, the mean and
// maximum live landmarks, the landmarks initialised and marginalised, the anchor changes and the two SLAM stage times.
// --slam-log OUT.txt (single run, for tests): what every frame did with the landmarks (write_slam_log).
// --perturb (rpng_sim's sim_do_perturbation; needs all five calibration blocks on): the filter starts from a calibration the
// simulator perturbs with --seed-perturb (Simulator::perturb_parameters), while the measurements and the truth stay the true
// ones. With --runs, run r also takes perturbation seed seed_perturb + r. The JSON line (and every per_run entry) gains
// "perturb" and the RMS of err/σ per calibration block at the first and the last frame (calib_nerr_json); a batch, their
// mean and population standard deviation over the runs.
// Estimator options, named after the keys of the reference's config/rpng_sim/estimator_config.yaml (INTEGRATION.md §8):
// --feat-rep-msckf NAME (GLOBAL_3D), --use-fej (1), --fi-triangulate-1d (0), --fi-refine-features (1), --up-msckf-sigma-px,
// --up-msckf-chi2-multipler, --up-slam-sigma-px, --up-slam-chi2-multipler (1 each; the SLAM pair serves the SLAM updates and
// the delayed initialisation), and one 0|1 flag per calibration block that overrides --calib for that block. A SINGLE MSCKF
// representation runs as ANCHORED_MSCKF_INVERSE_DEPTH (UpdaterMSCKF.cpp:180-183; the engine remaps it in ovb_api.cu's
// per-call options, the oracle in msckf_update). The JSON line (and every per_run entry) gains "estimator" with the options
// that differ from their defaults (estimator_json).
#ifdef OVB_SIM_ORACLE
#include "oracle_slam_backend.hpp"
#elif defined(OVB_SIM_HOST_PROPAGATION)
#include "host_propagation_backend.hpp"
#else
#include "../include/ovb200_vio.hpp"
#endif
#include <atomic>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <filesystem>
#include <string>
#include <thread>

using namespace ovb200;

static void write_blob(FILE *f, const void *p, size_t bytes) { std::fwrite(p, 1, bytes, f); }

struct RunnerOptions {
  std::string traj, integration = "rk4", compress = "cholqr2";
  int cams = 2, clones = 11, msckf = 10, pts = 250, frames = 0, calib = 1;
  int seed_init = 0, seed_perturb = 0, seed_meas = 0;
  std::vector<int> cam_models; // per camera (--cam-model); empty = all radtan
  int slam = 0, slam_in_update = 25, feat_rep_slam = OVB_REP_GLOBAL_3D;
  double slam_delay = 1.0;
  bool perturb = false;
  // the estimator options of the flags named after the reference's YAML keys (INTEGRATION.md §8, "Estimator options"):
  // feat_rep_msckf, do_fej, featinit_options.triangulate_1d / refine_features, msckf_options, slam_options and, once main
  // has resolved calib_block against --calib, the five do_calib_* flags; every other field stays VioOptions's default
  VioOptions est;
  int calib_block[5] = {-1, -1, -1, -1, -1}; // per calib_block_keys entry: 0 / 1 as given, -1 = as --calib
};

static const char *const rep_names[] = {"GLOBAL_3D", "GLOBAL_FULL_INVERSE_DEPTH", "ANCHORED_3D", "ANCHORED_FULL_INVERSE_DEPTH",
                                        "ANCHORED_MSCKF_INVERSE_DEPTH", "ANCHORED_INVERSE_DEPTH_SINGLE"};

// the calibration blocks of the --calib-* flags (the YAML keys), in RunnerOptions::calib_block's order
static const char *const calib_block_keys[5] = {"calib_cam_extrinsics", "calib_cam_intrinsics", "calib_cam_timeoffset", "calib_imu_intrinsics",
                                                "calib_imu_g_sensitivity"};
static bool *calib_block_flag(VioOptions &v, int b) {
  bool *const f[5] = {&v.do_calib_camera_pose, &v.do_calib_camera_intrinsics, &v.do_calib_camera_timeoffset, &v.do_calib_imu_intrinsics,
                      &v.do_calib_imu_g_sensitivity};
  return f[b];
}
// the calib_block_keys index of a --calib-* flag (the key with '-' for '_'), -1 for any other argument
static int calib_block_of_flag(const std::string &a) {
  for (int b = 0; b < 5; b++) {
    std::string flag = std::string("--") + calib_block_keys[b];
    std::replace(flag.begin(), flag.end(), '_', '-');
    if (a == flag)
      return b;
  }
  return -1;
}
static bool all_calib_blocks(const RunnerOptions &o) {
  const VioOptions &v = o.est;
  return v.do_calib_camera_pose && v.do_calib_camera_intrinsics && v.do_calib_camera_timeoffset && v.do_calib_imu_intrinsics && v.do_calib_imu_g_sensitivity;
}

// a whole decimal integer / number, nothing else
static bool parse_int(const std::string &a, int &v) {
  char *e = nullptr;
  const long x = std::strtol(a.c_str(), &e, 10);
  if (a.empty() || *e || x < INT32_MIN || x > INT32_MAX)
    return false;
  v = (int)x;
  return true;
}
static bool parse_double(const std::string &a, double &v) {
  char *e = nullptr;
  v = std::strtod(a.c_str(), &e);
  return !a.empty() && !*e && std::isfinite(v);
}
static bool parse_01(const std::string &a, int &v) { return parse_int(a, v) && (v == 0 || v == 1); }
static bool parse_rep(const std::string &a, int &v) {
  const auto it = std::find(std::begin(rep_names), std::end(rep_names), a);
  v = (int)(it - std::begin(rep_names));
  return it != std::end(rep_names);
}

#ifndef OVB_SIM_ORACLE
// the covariance the engine context must hold: the base state (State.cpp:28-131 with the calibration blocks in it), max_clones
// + 1 clone poses during the update, max_slam landmarks three wide (one for ANCHORED_INVERSE_DEPTH_SINGLE)
static int state_size_bound(const RunnerOptions &o) {
  const VioOptions &v = o.est;
  const int base = 15 + (v.do_calib_imu_intrinsics ? 15 + (v.do_calib_imu_g_sensitivity ? 9 : 0) : 0) + (v.do_calib_camera_timeoffset ? 1 : 0) +
                   o.cams * ((v.do_calib_camera_pose ? 6 : 0) + (v.do_calib_camera_intrinsics ? 8 : 0));
  return base + 6 * (o.clones + 1) + o.slam * (o.feat_rep_slam == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3);
}
static const int engine_max_state = 640; // ovb_config::max_state of the runner's engine context
#endif

// the SLAM part of a run's JSON (empty without --slam M, M > 0: such a run prints what a run without the flag prints)
static std::string slam_json(const RunnerOptions &o, const struct RunSummary &s);

// the JSON field of --cam-model (empty without the flag): , "cam_model": ["radtan", "equi", ...]
static std::string cam_model_json(const RunnerOptions &o) {
  if (o.cam_models.empty())
    return "";
  std::string s = ", \"cam_model\": [";
  for (size_t k = 0; k < o.cam_models.size(); k++)
    s += std::string(k ? ", " : "") + (o.cam_models[k] == OVB_CAM_EQUI ? "\"equi\"" : "\"radtan\"");
  return s + "]";
}

// --cam-model M[,M...] for `cams` cameras: false on an unknown model or a count other than 1 or cams
static bool parse_cam_models(const std::string &arg, int cams, std::vector<int> &out) {
  out.clear();
  size_t a = 0;
  while (true) {
    const size_t b = arg.find(',', a);
    const std::string m = arg.substr(a, b == std::string::npos ? std::string::npos : b - a);
    if (m == "radtan")
      out.push_back(OVB_CAM_RADTAN);
    else if (m == "equi")
      out.push_back(OVB_CAM_EQUI);
    else
      return false;
    if (b == std::string::npos)
      break;
    a = b + 1;
  }
  if (out.size() == 1)
    out.assign((size_t)std::max(cams, 1), out[0]);
  return (int)out.size() == cams;
}

// what one run reports (the single-run JSON line, and one entry of a --runs batch)
struct RunSummary {
  int frames = 0, state_dim = 0;
  double ate_pos = 0, ate_ori_deg = 0, feats_in = 0, feats_used = 0, rows = 0, ms_prop = 0, ms_msckf = 0, ms_total = 0;
  double nees_ori = 0, nees_pos = 0; // means over the run's frames (with --consistency)
  size_t map_points = 0;
  long status_hist[9] = {0};
  long slam_hist[9] = {0}, init_hist[9] = {0}, slam_initialized = 0, slam_marginalized = 0, anchor_changes = 0;
  double slam_live_mean = 0, ms_slam_update = 0, ms_slam_delayed = 0;
  int slam_live_max = 0;
  double nerr_first[9] = {0}, nerr_last[9] = {0}; // with --perturb: calib_nerr of the first and the last frame
};

// the calibration blocks of --perturb's report, in calib_nerr's order
static const char *const calib_blocks[9] = {"dt", "ext_ori", "ext_pos", "intr_fc", "intr_dist", "dw", "da", "tg", "gyro"};

// RMS of err/σ over the coordinates of each calibration block of one consistency sample, pooled over the cameras for the
// per-camera blocks (every block is in the state: --perturb needs --calib 1)
static void calib_nerr(const VioState &st, const ConsistencySample &c, double out[9]) {
  double ss[9] = {0};
  int n[9] = {0};
  auto add = [&](int b, int id, int m) {
    for (int k = id; k < id + m; k++) {
      const double z = c.err[(size_t)k] / c.sigma[(size_t)k];
      ss[b] += z * z, n[b]++;
    }
  };
  add(0, st.dt_id, 1);
  for (const auto &cam : st.cams) {
    add(1, cam.ext_id, 3), add(2, cam.ext_id + 3, 3);
    add(3, cam.intr_id, 4), add(4, cam.intr_id + 4, 4);
  }
  add(5, st.dw_id, 6), add(6, st.da_id, 6), add(7, st.tg_id, 9), add(8, st.gyro_id, 3);
  for (int b = 0; b < 9; b++)
    out[b] = std::sqrt(ss[b] / n[b]);
}

// {"dt": x, "ext_ori": x, ...} with printf format `fmt` per number
static std::string blocks_json(const double v[9], const char *fmt) {
  std::string r = "{";
  for (int b = 0; b < 9; b++) {
    char buf[64];
    std::snprintf(buf, sizeof(buf), fmt, v[b]);
    r += std::string(b ? ", \"" : "\"") + calib_blocks[b] + "\": " + buf;
  }
  return r + "}";
}

// the --perturb part of a run's JSON (empty without the flag)
static std::string calib_nerr_json(const RunnerOptions &o, const RunSummary &s, const char *fmt) {
  if (!o.perturb)
    return "";
  return ", \"perturb\": true, \"calib_nerr_first\": " + blocks_json(s.nerr_first, fmt) + ", \"calib_nerr_last\": " + blocks_json(s.nerr_last, fmt);
}

// the estimator options that differ from their defaults (VioOptions's; a calibration block's is --calib's value), as
// , "estimator": {"use_fej": 0, ...}; empty when none does, so that such a run prints what a run without the flags prints
static std::string estimator_json(const RunnerOptions &o) {
  const VioOptions d;
  VioOptions e = o.est;
  std::string r;
  auto add = [&](const char *key, const std::string &v) { r += std::string(r.empty() ? "" : ", ") + "\"" + key + "\": " + v; };
  auto num = [](double x) {
    char buf[64];
    std::snprintf(buf, sizeof(buf), "%.17g", x);
    return std::string(buf);
  };
  if (e.feat_rep_msckf != d.feat_rep_msckf)
    add("feat_rep_msckf", std::string("\"") + rep_names[e.feat_rep_msckf] + "\"");
  if (e.do_fej != d.do_fej)
    add("use_fej", std::to_string((int)e.do_fej));
  if (e.featinit_options.triangulate_1d != d.featinit_options.triangulate_1d)
    add("fi_triangulate_1d", std::to_string((int)e.featinit_options.triangulate_1d));
  if (e.featinit_options.refine_features != d.featinit_options.refine_features)
    add("fi_refine_features", std::to_string((int)e.featinit_options.refine_features));
  if (e.msckf_options.sigma_pix != d.msckf_options.sigma_pix)
    add("up_msckf_sigma_px", num(e.msckf_options.sigma_pix));
  if (e.msckf_options.chi2_multipler != d.msckf_options.chi2_multipler)
    add("up_msckf_chi2_multipler", num(e.msckf_options.chi2_multipler));
  if (e.slam_options.sigma_pix != d.slam_options.sigma_pix)
    add("up_slam_sigma_px", num(e.slam_options.sigma_pix));
  if (e.slam_options.chi2_multipler != d.slam_options.chi2_multipler)
    add("up_slam_chi2_multipler", num(e.slam_options.chi2_multipler));
  for (int b = 0; b < 5; b++)
    if (*calib_block_flag(e, b) != (o.calib != 0))
      add(calib_block_keys[b], std::to_string((int)*calib_block_flag(e, b)));
  return r.empty() ? "" : ", \"estimator\": {" + r + "}";
}

static std::string slam_json(const RunnerOptions &o, const RunSummary &s) {
  if (o.slam <= 0)
    return "";
  auto hist = [](const long *h) {
    std::string r = "[";
    for (int k = 0; k < 9; k++)
      r += (k ? ", " : "") + std::to_string(h[k]);
    return r + "]";
  };
  char buf[512];
  std::snprintf(buf, sizeof(buf), ", \"max_slam\": %d, \"max_slam_in_update\": %d, \"dt_slam_delay\": %.17g, \"feat_rep_slam\": \"%s\", \"mean_slam_live\": %.4f, "
                "\"max_slam_live\": %d, \"slam_initialized\": %ld, \"slam_marginalized\": %ld, \"anchor_changes\": %ld, \"mean_ms_slam_update\": %.4f, "
                "\"mean_ms_slam_delayed\": %.4f",
                o.slam, o.slam_in_update, o.slam_delay, rep_names[o.feat_rep_slam], s.slam_live_mean, s.slam_live_max, s.slam_initialized, s.slam_marginalized,
                s.anchor_changes, s.ms_slam_update, s.ms_slam_delayed);
  return std::string(buf) + ", \"slam_status_hist\": " + hist(s.slam_hist) + ", \"init_status_hist\": " + hist(s.init_hist);
}

// --slam-log: per frame a line "F t since_start N n_clones n_landmarks", then one line per list, each "<tag> featid...": P promoted,
// M the MSCKF batch, U the SLAM updates, D the delayed initialisations, X the landmarks marginalize_slam removed (as
// featid:update_fail_count), I the landmarks initialised; then "L featid id size anchor_in_window" per landmark at the frame's
// end (anchor_in_window -1 for the global representations)
static void write_slam_log(const std::string &path, const std::vector<SlamFrameRecord> &frames) {
  FILE *f = std::fopen(path.c_str(), "w");
  if (!f)
    return;
  auto ids = [&](const char *tag, const std::vector<size_t> &v) {
    std::fprintf(f, "%s", tag);
    for (size_t id : v)
      std::fprintf(f, " %zu", id);
    std::fprintf(f, "\n");
  };
  for (const auto &r : frames) {
    std::fprintf(f, "F %.9f %.9f %d %d %zu\n", r.t, r.since_start, r.N, r.n_clones, r.landmarks.size());
    ids("P", r.promoted), ids("M", r.msckf), ids("U", r.slam_update), ids("D", r.delayed);
    std::fprintf(f, "X");
    for (const auto &x : r.marg_fail_count)
      std::fprintf(f, " %zu:%d", x.first, x.second);
    std::fprintf(f, "\n");
    ids("I", r.initialized);
    for (const auto &l : r.landmarks)
      std::fprintf(f, "L %ld %ld %ld %ld\n", l[0], l[1], l[2], l[3]);
  }
  std::fclose(f);
}

#ifdef OVB_SIM_ORACLE
static const char *const backend_name = "oracle";
#else
static const char *const backend_name = "engine";
#endif

// one closed-loop run with measurement seed `seed_meas` and perturbation seed `seed_perturb`; empty paths write nothing,
// capture_frame < 0 captures nothing, consistency = record the consistency samples (written to consistency_path unless it
// is empty)
static RunSummary run_one(const RunnerOptions &o, const std::vector<std::array<double, 8>> &traj_data, int seed_meas, int seed_perturb, const std::string &est_path,
                          const std::string &timing_path, bool consistency, const std::string &consistency_path, int capture_frame,
                          const std::string &capture_prefix, const std::string &slam_log_path = "") {
  SimParams sp;
  rpng_sim_cameras(o.cams, sp, o.cam_models);
  sp.use_stereo = o.cams > 1;
  sp.num_pts = o.pts;
  sp.seed_state_init = o.seed_init;
  sp.seed_preturb = seed_perturb;
  sp.seed_measurements = seed_meas;
  sp.sim_do_perturbation = o.perturb;
  VioOptions vo = o.est;
  vo.num_cameras = o.cams;
  vo.max_clone_size = o.clones;
  vo.max_msckf_in_update = o.msckf;
  vo.compress = o.compress == "tsqr" ? OVB_COMPRESS_HOUSEHOLDER_TSQR : (o.compress == "gram" ? OVB_COMPRESS_NORMAL_EQUATIONS : OVB_COMPRESS_CHOLQR2);
  vo.integration_method = o.integration == "discrete" ? INTEGRATION_DISCRETE : (o.integration == "analytical" ? INTEGRATION_ANALYTICAL : INTEGRATION_RK4);
  vo.max_slam_features = o.slam;
  vo.max_slam_in_update = o.slam_in_update;
  vo.dt_slam_delay = o.slam_delay;
  vo.feat_rep_slam = o.feat_rep_slam;
  Simulator sim(sp, traj_data);
#ifdef OVB_SIM_ORACLE
  auto backend = std::make_shared<OracleSlamCov>();
#else
  ovb_config cfg{0, engine_max_state, std::max(1024, o.msckf), std::max(1024, o.msckf) * 2 * (o.clones + 1) * o.cams / 2 + 1024, 0};
#ifdef OVB_SIM_HOST_PROPAGATION
  auto backend = std::make_shared<HostPropagationEngineCov>(cfg);
#else
  auto backend = std::make_shared<EngineCov>(cfg);
#endif
#endif
  VioManager sys(vo, sim.get_estimator_parameters(), backend);
  sys.record_slam_frames = !slam_log_path.empty();
  if (capture_frame >= 0) {
    // dump the marshalled inputs of ONE update (the golden "update case" wire format of tests/golden_io.py:
    // little-endian, a text header line with the array shapes followed by the raw arrays) and the prior covariance
    sys.on_update = [&](const ovb_frame &fr, const ovb_feat_batch &fb, const ovb_opts &op, int frame_index) {
      if (frame_index != capture_frame)
        return;
      FILE *f = std::fopen((capture_prefix + ".case").c_str(), "wb");
      if (!f)
        return;
      const int N = backend->dim();
      const std::vector<double> P = backend->get();
      int nkeys = fb.cam_keys_off ? fb.cam_keys_off[fb.n_feats] : 0;
      std::fprintf(f, "OVBCASE1 n_clones=%d n_cams=%d n_feats=%d n_meas=%d n_keys=%d N=%d opts=%zu\n", fr.n_clones, fr.n_cams, fb.n_feats, fb.n_meas, nkeys, N,
                   sizeof(ovb_opts));
      write_blob(f, fr.clone_R, sizeof(double) * 9 * fr.n_clones);
      write_blob(f, fr.clone_p, sizeof(double) * 3 * fr.n_clones);
      write_blob(f, fr.clone_R_fej, sizeof(double) * 9 * fr.n_clones);
      write_blob(f, fr.clone_p_fej, sizeof(double) * 3 * fr.n_clones);
      write_blob(f, fr.clone_off, sizeof(int) * fr.n_clones);
      write_blob(f, fr.cam_R, sizeof(double) * 9 * fr.n_cams);
      write_blob(f, fr.cam_p, sizeof(double) * 3 * fr.n_cams);
      write_blob(f, fr.cam_intr, sizeof(double) * 8 * fr.n_cams);
      write_blob(f, fr.cam_model, sizeof(int) * fr.n_cams);
      write_blob(f, fr.cam_ext_off, sizeof(int) * fr.n_cams);
      write_blob(f, fr.cam_intr_off, sizeof(int) * fr.n_cams);
      write_blob(f, fb.meas_off, sizeof(int32_t) * (fb.n_feats + 1));
      write_blob(f, fb.cam, fb.n_meas);
      write_blob(f, fb.clone, sizeof(uint16_t) * fb.n_meas);
      write_blob(f, fb.uv, sizeof(float) * 2 * fb.n_meas);
      write_blob(f, fb.uvn, sizeof(float) * 2 * fb.n_meas);
      write_blob(f, fb.cam_keys_off, sizeof(int32_t) * (fb.n_feats + 1));
      write_blob(f, fb.cam_keys, (size_t)nkeys);
      write_blob(f, &op, sizeof(ovb_opts));
      write_blob(f, P.data(), sizeof(double) * P.size());
      std::fclose(f);
    };
  }
  SimRunResult res = run_simulation(sim, sys, o.frames, consistency || o.perturb);
  if (!est_path.empty()) {
    FILE *f = std::fopen(est_path.c_str(), "w");
    if (f) {
      std::fprintf(f, "# timestamp(s) tx ty tz qx qy qz qw | gt: tx ty tz qx qy qz qw\n");
      for (size_t i = 0; i < res.est.size(); i++) {
        const auto &e = res.est[i];
        const auto &g = res.gt[i];
        std::fprintf(f, "%.9f %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", e.t, e.p[0], e.p[1], e.p[2], e.q[0],
                     e.q[1], e.q[2], e.q[3], g.p[0], g.p[1], g.p[2], g.q[0], g.q[1], g.q[2], g.q[3]);
      }
      std::fclose(f);
    }
  }
  if (!timing_path.empty())
    sys.write_timing_csv(timing_path);
  if (!consistency_path.empty())
    write_consistency_file(consistency_path, sys.state, res.consistency);
  if (!slam_log_path.empty())
    write_slam_log(slam_log_path, sys.slam_frames);
  double t_prop = 0, t_msckf = 0, t_total = 0, feats = 0, used = 0, rows = 0, t_su = 0, t_sd = 0, live = 0;
  RunSummary s;
  for (const auto &t : sys.timing) {
    t_prop += t.time_prop, t_msckf += t.time_msckf, t_total += t.time_total;
    feats += t.feats_in, used += t.feats_used, rows += t.rows;
    t_su += t.time_slam_update, t_sd += t.time_slam_delayed, live += t.slam_live;
    s.slam_live_max = std::max(s.slam_live_max, t.slam_live);
  }
  const double n = sys.timing.empty() ? 1.0 : (double)sys.timing.size();
  s.slam_live_mean = live / n, s.ms_slam_update = 1e3 * t_su / n, s.ms_slam_delayed = 1e3 * t_sd / n;
  for (int k = 0; k < 9; k++)
    s.slam_hist[k] = sys.slam_status_hist[k], s.init_hist[k] = sys.init_status_hist[k];
  s.slam_initialized = sys.slam_initialized, s.slam_marginalized = sys.slam_marginalized, s.anchor_changes = sys.anchor_changes;
  s.feats_in = feats / n, s.feats_used = used / n, s.rows = rows / n;
  s.ms_prop = 1e3 * t_prop / n, s.ms_msckf = 1e3 * t_msckf / n, s.ms_total = 1e3 * t_total / n;
  s.frames = res.frames;
  s.state_dim = backend->dim();
  s.ate_pos = res.ate_pos, s.ate_ori_deg = res.ate_ori_deg;
  s.map_points = sim.featmap.size();
  for (int k = 0; k < 9; k++)
    s.status_hist[k] = sys.status_hist[k];
  for (const auto &c : res.consistency)
    s.nees_ori += c.nees_ori, s.nees_pos += c.nees_pos;
  if (!res.consistency.empty())
    s.nees_ori /= (double)res.consistency.size(), s.nees_pos /= (double)res.consistency.size();
  if (o.perturb && !res.consistency.empty()) {
    calib_nerr(sys.state, res.consistency.front(), s.nerr_first);
    calib_nerr(sys.state, res.consistency.back(), s.nerr_last);
  }
  return s;
}

// the --runs batch: returns the process exit code
static int run_batch(const RunnerOptions &o, const std::vector<std::array<double, 8>> &traj_data, int runs, int jobs, const std::string &out_dir, bool timing,
                     bool consistency) {
  std::vector<RunSummary> out((size_t)runs);
  std::vector<std::string> err((size_t)runs);
  std::atomic<int> next{0};
  std::atomic<bool> failed{false};
  auto worker = [&]() {
    for (int r; !failed.load() && (r = next.fetch_add(1)) < runs;) {
      const int seed = o.seed_meas + r;
      const std::string stem = out_dir.empty() ? std::string() : out_dir + "/";
      try {
        out[(size_t)r] = run_one(o, traj_data, seed, o.seed_perturb + r, stem.empty() ? "" : stem + "est_" + std::to_string(seed) + ".txt",
                                 stem.empty() || !timing ? "" : stem + "timing_" + std::to_string(seed) + ".csv", consistency,
                                 stem.empty() || !consistency ? "" : stem + "consistency_" + std::to_string(seed) + ".txt", -1, "");
      } catch (const std::exception &e) {
        err[(size_t)r] = e.what();
        failed = true; // the runs already started finish; no new one starts
      } catch (...) {
        err[(size_t)r] = "unknown exception";
        failed = true;
      }
    }
  };
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> pool;
  for (int j = 0; j < jobs; j++)
    pool.emplace_back(worker);
  for (auto &t : pool)
    t.join();
  const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (failed) {
    for (int r = 0; r < runs; r++)
      if (!err[(size_t)r].empty())
        std::fprintf(stderr, "run_simulation failed: run %d (seed_meas %d): %s\n", r, o.seed_meas + r, err[(size_t)r].c_str());
    return 1;
  }
  // mean and population standard deviation (numpy's default ddof = 0) of both ATEs
  double mp = 0, mo = 0, vp = 0, vo = 0;
  long frames = 0;
  for (const auto &s : out)
    mp += s.ate_pos, mo += s.ate_ori_deg, frames += s.frames;
  mp /= runs, mo /= runs;
  for (const auto &s : out)
    vp += (s.ate_pos - mp) * (s.ate_pos - mp), vo += (s.ate_ori_deg - mo) * (s.ate_ori_deg - mo);
  std::string per_run;
  for (int r = 0; r < runs; r++) {
    const RunSummary &s = out[(size_t)r];
    char buf[512];
    std::snprintf(buf, sizeof(buf), "%s{\"seed\": %d, \"frames\": %d, \"ate_pos_m\": %.17g, \"ate_ori_deg\": %.17g, \"status_hist\": [%ld, %ld, %ld, %ld, %ld, %ld, %ld, %ld, %ld]",
                  r ? ", " : "", o.seed_meas + r, s.frames, s.ate_pos, s.ate_ori_deg, s.status_hist[0], s.status_hist[1], s.status_hist[2], s.status_hist[3],
                  s.status_hist[4], s.status_hist[5], s.status_hist[6], s.status_hist[7], s.status_hist[8]);
    per_run += buf;
    if (consistency) {
      std::snprintf(buf, sizeof(buf), ", \"nees_ori\": %.17g, \"nees_pos\": %.17g", s.nees_ori, s.nees_pos);
      per_run += buf;
    }
    if (o.perturb) {
      std::snprintf(buf, sizeof(buf), ", \"seed_perturb\": %d", o.seed_perturb + r);
      per_run += buf;
    }
    per_run += slam_json(o, s) + calib_nerr_json(o, s, "%.17g") + estimator_json(o) + "}";
  }
  // the same statistics of the per-run mean NEES
  std::string stats;
  if (consistency) {
    double no = 0, np = 0, vno = 0, vnp = 0;
    for (const auto &s : out)
      no += s.nees_ori, np += s.nees_pos;
    no /= runs, np /= runs;
    for (const auto &s : out)
      vno += (s.nees_ori - no) * (s.nees_ori - no), vnp += (s.nees_pos - np) * (s.nees_pos - np);
    char buf[256];
    std::snprintf(buf, sizeof(buf), ", \"nees_ori_mean\": %.17g, \"nees_ori_std\": %.17g, \"nees_pos_mean\": %.17g, \"nees_pos_std\": %.17g", no,
                  std::sqrt(vno / runs), np, std::sqrt(vnp / runs));
    stats = buf;
  }
  // and of the per-block calibration errors
  if (o.perturb) {
    stats += ", \"perturb\": true";
    for (int last = 0; last < 2; last++) {
      double m[9] = {0}, sd[9] = {0};
      for (const auto &s : out)
        for (int b = 0; b < 9; b++)
          m[b] += (last ? s.nerr_last : s.nerr_first)[b] / runs;
      for (const auto &s : out)
        for (int b = 0; b < 9; b++) {
          const double d = (last ? s.nerr_last : s.nerr_first)[b] - m[b];
          sd[b] += d * d / runs;
        }
      for (int b = 0; b < 9; b++)
        sd[b] = std::sqrt(sd[b]);
      const std::string key = last ? "calib_nerr_last" : "calib_nerr_first";
      stats += ", \"" + key + "_mean\": " + blocks_json(m, "%.17g") + ", \"" + key + "_std\": " + blocks_json(sd, "%.17g");
    }
  }
  stats += estimator_json(o);
  std::printf("{\"backend\": \"%s\", \"runs\": %d, \"jobs\": %d, \"cams\": %d%s, \"max_clones\": %d, \"max_msckf_in_update\": %d, \"num_pts\": %d, \"calib\": %d, "
              "\"seed_init\": %d, \"seed_perturb\": %d, \"seed_meas\": %d, \"state_dim\": %d, \"map_points\": %zu, \"per_run\": [%s], "
              "\"ate_pos_m_mean\": %.17g, \"ate_pos_m_std\": %.17g, \"ate_ori_deg_mean\": %.17g, \"ate_ori_deg_std\": %.17g, \"frames_total\": %ld, "
              "\"wall_s\": %.6f, \"runs_per_s\": %.6f, \"frames_per_s\": %.3f%s}\n",
              backend_name, runs, jobs, o.cams, cam_model_json(o).c_str(), o.clones, o.msckf, o.pts, o.calib, o.seed_init, o.seed_perturb, o.seed_meas, out[0].state_dim, out[0].map_points,
              per_run.c_str(), mp, std::sqrt(vp / runs), mo, std::sqrt(vo / runs), frames, wall, runs / wall, frames / wall, stats.c_str());
  return 0;
}

int main(int argc, char **argv) {
  RunnerOptions o;
  std::string est_path, timing_path, consistency_path, capture_prefix, out_dir, cam_model_arg, slam_log_path;
  std::string bad_slam, bad_est; // the first malformed SLAM / estimator option
  int capture_frame = -1, runs = 0, jobs = 0;
  bool timing = false, consistency = false, cam_model = false;
  for (int i = 1; i < argc; i++) {
    auto next = [&]() { return std::string(i + 1 < argc ? argv[++i] : ""); };
    const std::string a = argv[i];
    if (a == "--traj") o.traj = next();
    else if (a == "--cams") o.cams = std::stoi(next());
    else if (a == "--clones") o.clones = std::stoi(next());
    else if (a == "--msckf") o.msckf = std::stoi(next());
    else if (a == "--pts") o.pts = std::stoi(next());
    else if (a == "--frames") o.frames = std::stoi(next());
    else if (a == "--calib") o.calib = std::stoi(next());
    else if (a == "--est") est_path = next();
    else if (a == "--timing") { // the path is optional: a --runs batch names its files itself
      timing = true;
      if (i + 1 < argc && std::strncmp(argv[i + 1], "--", 2) != 0)
        timing_path = next();
    }
    else if (a == "--consistency") { // like --timing: a --runs batch names its files itself
      consistency = true;
      if (i + 1 < argc && std::strncmp(argv[i + 1], "--", 2) != 0)
        consistency_path = next();
    }
    else if (a == "--integration") o.integration = next();
    else if (a == "--compress") o.compress = next();
    else if (a == "--capture") { capture_frame = std::stoi(next()); capture_prefix = next(); }
    else if (a == "--seed-init") o.seed_init = std::stoi(next());
    else if (a == "--seed-perturb") o.seed_perturb = std::stoi(next());
    else if (a == "--seed-meas") o.seed_meas = std::stoi(next());
    else if (a == "--runs") runs = std::stoi(next());
    else if (a == "--jobs") jobs = std::stoi(next());
    else if (a == "--out-dir") out_dir = next();
    else if (a == "--cam-model") { cam_model = true; cam_model_arg = next(); }
    else if (a == "--slam") { const std::string v = next(); if (!parse_int(v, o.slam) || o.slam < 0) bad_slam = a + " " + v; }
    else if (a == "--slam-in-update") { const std::string v = next(); if (!parse_int(v, o.slam_in_update) || o.slam_in_update < 1) bad_slam = a + " " + v; }
    else if (a == "--slam-delay") { const std::string v = next(); if (!parse_double(v, o.slam_delay) || o.slam_delay < 0) bad_slam = a + " " + v; }
    else if (a == "--feat-rep-slam") {
      const std::string v = next();
      int rep;
      if (!parse_rep(v, rep))
        bad_slam = a + " " + v;
      else
        o.feat_rep_slam = rep;
    }
    else if (a == "--slam-log") slam_log_path = next();
    else if (a == "--perturb") o.perturb = true;
    else if (a == "--feat-rep-msckf") { const std::string v = next(); if (!parse_rep(v, o.est.feat_rep_msckf)) bad_est = a + " " + v; }
    else if (a == "--use-fej" || a == "--fi-triangulate-1d" || a == "--fi-refine-features") {
      const std::string v = next();
      int x;
      if (!parse_01(v, x))
        bad_est = a + " " + v;
      else
        (a == "--use-fej" ? o.est.do_fej : a == "--fi-triangulate-1d" ? o.est.featinit_options.triangulate_1d : o.est.featinit_options.refine_features) = x;
    }
    else if (a == "--up-msckf-sigma-px" || a == "--up-msckf-chi2-multipler" || a == "--up-slam-sigma-px" || a == "--up-slam-chi2-multipler") {
      const std::string v = next();
      UpdaterOptions &u = a.compare(0, 10, "--up-msckf") == 0 ? o.est.msckf_options : o.est.slam_options;
      double &x = a.find("sigma") != std::string::npos ? u.sigma_pix : u.chi2_multipler;
      if (!parse_double(v, x) || x <= 0)
        bad_est = a + " " + v;
    }
    else if (const int b = calib_block_of_flag(a); b >= 0) {
      const std::string v = next();
      if (!parse_01(v, o.calib_block[b]))
        bad_est = a + " " + v;
    }
  }
  if (!bad_slam.empty()) {
    std::fprintf(stderr, "malformed '%s': --slam takes an integer >= 0, --slam-in-update an integer >= 1, --slam-delay seconds >= 0, --feat-rep-slam one of "
                 "GLOBAL_3D GLOBAL_FULL_INVERSE_DEPTH ANCHORED_3D ANCHORED_FULL_INVERSE_DEPTH ANCHORED_MSCKF_INVERSE_DEPTH ANCHORED_INVERSE_DEPTH_SINGLE\n",
                 bad_slam.c_str());
    return 2;
  }
  if (!bad_est.empty()) {
    std::fprintf(stderr, "malformed '%s': --feat-rep-msckf takes one of GLOBAL_3D GLOBAL_FULL_INVERSE_DEPTH ANCHORED_3D ANCHORED_FULL_INVERSE_DEPTH "
                 "ANCHORED_MSCKF_INVERSE_DEPTH ANCHORED_INVERSE_DEPTH_SINGLE, --use-fej, --fi-* and --calib-* 0 or 1, --up-* a number > 0\n",
                 bad_est.c_str());
    return 2;
  }
  for (int b = 0; b < 5; b++) // a --calib-* flag overrides --calib for its block, wherever either stands
    *calib_block_flag(o.est, b) = o.calib_block[b] >= 0 ? o.calib_block[b] != 0 : o.calib != 0;
  if (!o.est.do_calib_imu_intrinsics) { // the state holds Tg only inside the IMU intrinsics (State.h:126-135)
    if (o.calib_block[4] == 1) {
      std::fprintf(stderr, "--calib-imu-g-sensitivity 1 needs the IMU intrinsics in the state: Tg is part of them (State.h:126-135)\n");
      return 2;
    }
    o.est.do_calib_imu_g_sensitivity = false;
  }
  if (o.perturb && !all_calib_blocks(o)) {
    std::fprintf(stderr, "--perturb needs all five calibration blocks on (--calib 1 and no --calib-* 0): without online calibration of a block "
                 "the filter could not estimate the error it starts with\n");
    return 2;
  }
  if (runs > 0 && !slam_log_path.empty()) {
    std::fprintf(stderr, "--slam-log is a single-run option\n");
    return 2;
  }
#ifndef OVB_SIM_ORACLE
  if (state_size_bound(o) > engine_max_state) {
    std::fprintf(stderr, "a state of up to %d variables (--cams %d --clones %d --calib %d --slam %d) does not fit the engine context's %d\n", state_size_bound(o),
                 o.cams, o.clones, o.calib, o.slam, engine_max_state);
    return 2;
  }
#endif
  if (runs < 0 || jobs < 0 || (runs == 0 && (jobs > 0 || !out_dir.empty())) || (runs > 0 && (!est_path.empty() || capture_frame >= 0))) {
    std::fprintf(stderr, "--runs K takes --jobs J >= 1 and --out-dir DIR; --jobs and --out-dir need --runs; --est and --capture are single-run options\n");
    return 2;
  }
  if (cam_model && !parse_cam_models(cam_model_arg, o.cams, o.cam_models)) {
    std::fprintf(stderr, "--cam-model takes radtan or equi, once for every camera or once per camera (--cams %d), not '%s'\n", o.cams,
                 cam_model_arg.c_str());
    return 2;
  }
  if (consistency && runs == 0 && consistency_path.empty()) {
    std::fprintf(stderr, "--consistency takes the output file's path on a single run (a --runs batch writes DIR/consistency_<seed>.txt)\n");
    return 2;
  }
  std::vector<std::array<double, 8>> traj_data =
      o.traj.size() > 4 && o.traj.substr(o.traj.size() - 4) == ".bin" ? load_trajectory_bin(o.traj) : load_simulated_trajectory(o.traj);
  if (traj_data.size() < 4) {
    std::fprintf(stderr, "could not load the trajectory '%s'\n", o.traj.c_str());
    return 2;
  }
  if (runs > 0) {
    if (jobs == 0)
      jobs = (int)std::max(1u, std::min((unsigned)runs, std::thread::hardware_concurrency()));
    jobs = std::min(jobs, runs);
    if (!out_dir.empty()) {
      std::error_code ec;
      std::filesystem::create_directories(out_dir, ec);
      if (!std::filesystem::is_directory(out_dir)) {
        std::fprintf(stderr, "could not create the output directory '%s'\n", out_dir.c_str());
        return 2;
      }
    }
    return run_batch(o, traj_data, runs, jobs, out_dir, timing, consistency);
  }
  try {
    const RunSummary s = run_one(o, traj_data, o.seed_meas, o.seed_perturb, est_path, timing_path, consistency, consistency_path, capture_frame, capture_prefix, slam_log_path);
    char nees[128] = "";
    if (consistency)
      std::snprintf(nees, sizeof(nees), ", \"nees_ori\": %.12g, \"nees_pos\": %.12g", s.nees_ori, s.nees_pos);
    std::printf("{\"backend\": \"%s\", \"frames\": %d, \"cams\": %d%s, \"max_clones\": %d, \"max_msckf_in_update\": %d, \"num_pts\": %d, \"calib\": %d, "
                "\"state_dim\": %d, \"ate_pos_m\": %.12g, \"ate_ori_deg\": %.12g, \"mean_feats_in\": %.2f, \"mean_feats_used\": %.2f, \"mean_rows\": %.1f, "
                "\"mean_ms_propagation\": %.4f, \"mean_ms_msckf_update\": %.4f, \"mean_ms_total\": %.4f, \"map_points\": %zu, \"status_hist\": [%ld, %ld, %ld, %ld, %ld, %ld, %ld, %ld, %ld]%s}\n",
                backend_name, s.frames, o.cams, cam_model_json(o).c_str(), o.clones, o.msckf, o.pts, o.calib, s.state_dim, s.ate_pos, s.ate_ori_deg, s.feats_in, s.feats_used, s.rows,
                s.ms_prop, s.ms_msckf, s.ms_total, s.map_points, s.status_hist[0], s.status_hist[1], s.status_hist[2], s.status_hist[3], s.status_hist[4],
                s.status_hist[5], s.status_hist[6], s.status_hist[7], s.status_hist[8], (nees + slam_json(o, s) + calib_nerr_json(o, s, "%.12g") + estimator_json(o)).c_str());
  } catch (const std::exception &e) {
    std::fprintf(stderr, "run_simulation failed: %s\n", e.what());
    return 1;
  }
  return 0;
}
