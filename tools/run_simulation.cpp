// run_simulation.cpp — rpng_sim runner (ov_msckf/src/run_simulation.cpp) on the host layer of include/ovb200_vio.hpp.
//   ovb_run_simulation   (this file, -DOVB_SIM_ENGINE): covariance and MSCKF updates on the CUDA engine (libovb200.so)
//   tests/cpp/run_simulation_oracle (same file, -DOVB_SIM_ORACLE, test infrastructure): the CPU oracle behind the same interface
//   -DOVB_SIM_HOST_PROPAGATION (test infrastructure): the engine with the IMU covariance accumulation on the host
// Usage: <exe> --traj FILE(.txt|.bin) [--cams K] [--clones C] [--msckf M] [--pts P] [--frames F] [--calib 0|1]
//              [--est OUT.txt] [--timing [OUT.csv]] [--capture FRAME PREFIX] [--integration discrete|rk4|analytical]
//              [--seed-init S] [--seed-perturb S] [--seed-meas S] [--runs K [--jobs J] [--out-dir DIR]] [--consistency [OUT.txt]]
//              [--cam-model M[,M...]]
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
#ifdef OVB_SIM_ORACLE
#include "oracle_backend.hpp"
#elif defined(OVB_SIM_HOST_PROPAGATION)
#include "host_propagation_backend.hpp"
#else
#include "../include/ovb200_vio.hpp"
#endif
#include <atomic>
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
};

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
};

#ifdef OVB_SIM_ORACLE
static const char *const backend_name = "oracle";
#else
static const char *const backend_name = "engine";
#endif

// one closed-loop run with measurement seed `seed_meas`; empty paths write nothing, capture_frame < 0 captures nothing,
// consistency = record the consistency samples (written to consistency_path unless it is empty)
static RunSummary run_one(const RunnerOptions &o, const std::vector<std::array<double, 8>> &traj_data, int seed_meas, const std::string &est_path,
                          const std::string &timing_path, bool consistency, const std::string &consistency_path, int capture_frame,
                          const std::string &capture_prefix) {
  SimParams sp;
  rpng_sim_cameras(o.cams, sp, o.cam_models);
  sp.use_stereo = o.cams > 1;
  sp.num_pts = o.pts;
  sp.seed_state_init = o.seed_init;
  sp.seed_preturb = o.seed_perturb;
  sp.seed_measurements = seed_meas;
  VioOptions vo;
  vo.num_cameras = o.cams;
  vo.max_clone_size = o.clones;
  vo.max_msckf_in_update = o.msckf;
  vo.do_calib_camera_pose = vo.do_calib_camera_intrinsics = vo.do_calib_camera_timeoffset = vo.do_calib_imu_intrinsics = vo.do_calib_imu_g_sensitivity =
      o.calib != 0;
  vo.compress = o.compress == "tsqr" ? OVB_COMPRESS_HOUSEHOLDER_TSQR : (o.compress == "gram" ? OVB_COMPRESS_NORMAL_EQUATIONS : OVB_COMPRESS_CHOLQR2);
  vo.integration_method = o.integration == "discrete" ? INTEGRATION_DISCRETE : (o.integration == "analytical" ? INTEGRATION_ANALYTICAL : INTEGRATION_RK4);
  Simulator sim(sp, traj_data);
#ifdef OVB_SIM_ORACLE
  auto backend = std::make_shared<OracleCov>();
#else
  ovb_config cfg{0, 640, std::max(1024, o.msckf), std::max(1024, o.msckf) * 2 * (o.clones + 1) * o.cams / 2 + 1024, 0};
#ifdef OVB_SIM_HOST_PROPAGATION
  auto backend = std::make_shared<HostPropagationEngineCov>(cfg);
#else
  auto backend = std::make_shared<EngineCov>(cfg);
#endif
#endif
  VioManager sys(vo, sp, backend);
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
  SimRunResult res = run_simulation(sim, sys, o.frames, consistency);
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
  double t_prop = 0, t_msckf = 0, t_total = 0, feats = 0, used = 0, rows = 0;
  for (const auto &t : sys.timing) {
    t_prop += t.time_prop, t_msckf += t.time_msckf, t_total += t.time_total;
    feats += t.feats_in, used += t.feats_used, rows += t.rows;
  }
  const double n = sys.timing.empty() ? 1.0 : (double)sys.timing.size();
  RunSummary s;
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
        out[(size_t)r] = run_one(o, traj_data, seed, stem.empty() ? "" : stem + "est_" + std::to_string(seed) + ".txt",
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
    per_run += "}";
  }
  // the same statistics of the per-run mean NEES
  std::string nees;
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
    nees = buf;
  }
  std::printf("{\"backend\": \"%s\", \"runs\": %d, \"jobs\": %d, \"cams\": %d%s, \"max_clones\": %d, \"max_msckf_in_update\": %d, \"num_pts\": %d, \"calib\": %d, "
              "\"seed_init\": %d, \"seed_perturb\": %d, \"seed_meas\": %d, \"state_dim\": %d, \"map_points\": %zu, \"per_run\": [%s], "
              "\"ate_pos_m_mean\": %.17g, \"ate_pos_m_std\": %.17g, \"ate_ori_deg_mean\": %.17g, \"ate_ori_deg_std\": %.17g, \"frames_total\": %ld, "
              "\"wall_s\": %.6f, \"runs_per_s\": %.6f, \"frames_per_s\": %.3f%s}\n",
              backend_name, runs, jobs, o.cams, cam_model_json(o).c_str(), o.clones, o.msckf, o.pts, o.calib, o.seed_init, o.seed_perturb, o.seed_meas, out[0].state_dim, out[0].map_points,
              per_run.c_str(), mp, std::sqrt(vp / runs), mo, std::sqrt(vo / runs), frames, wall, runs / wall, frames / wall, nees.c_str());
  return 0;
}

int main(int argc, char **argv) {
  RunnerOptions o;
  std::string est_path, timing_path, consistency_path, capture_prefix, out_dir, cam_model_arg;
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
  }
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
    const RunSummary s = run_one(o, traj_data, o.seed_meas, est_path, timing_path, consistency, consistency_path, capture_frame, capture_prefix);
    char nees[128] = "";
    if (consistency)
      std::snprintf(nees, sizeof(nees), ", \"nees_ori\": %.12g, \"nees_pos\": %.12g", s.nees_ori, s.nees_pos);
    std::printf("{\"backend\": \"%s\", \"frames\": %d, \"cams\": %d%s, \"max_clones\": %d, \"max_msckf_in_update\": %d, \"num_pts\": %d, \"calib\": %d, "
                "\"state_dim\": %d, \"ate_pos_m\": %.12g, \"ate_ori_deg\": %.12g, \"mean_feats_in\": %.2f, \"mean_feats_used\": %.2f, \"mean_rows\": %.1f, "
                "\"mean_ms_propagation\": %.4f, \"mean_ms_msckf_update\": %.4f, \"mean_ms_total\": %.4f, \"map_points\": %zu, \"status_hist\": [%ld, %ld, %ld, %ld, %ld, %ld, %ld, %ld, %ld]%s}\n",
                backend_name, s.frames, o.cams, cam_model_json(o).c_str(), o.clones, o.msckf, o.pts, o.calib, s.state_dim, s.ate_pos, s.ate_ori_deg, s.feats_in, s.feats_used, s.rows,
                s.ms_prop, s.ms_msckf, s.ms_total, s.map_points, s.status_hist[0], s.status_hist[1], s.status_hist[2], s.status_hist[3], s.status_hist[4],
                s.status_hist[5], s.status_hist[6], s.status_hist[7], s.status_hist[8], nees);
  } catch (const std::exception &e) {
    std::fprintf(stderr, "run_simulation failed: %s\n", e.what());
    return 1;
  }
  return 0;
}
