// equi_probe.cpp — test helper: the equidistant camera of the host pipeline (SimCamera in include/ovb200_sim.hpp) for
// tests/test_sim_equi_cpu.py. The camera is the fisheye camera of rpng_sim_cameras (TUM-VI cam0 intrinsics, 512 x 512).
//   equi_probe undistort [k1..k4]   stdin: lines "u v" (float pixels)  -> xn yn per line (undistort_f), optionally with
//                                      other distortion coefficients
//   equi_probe oracle               -> points compared, points whose distort_f differs from the oracle's distort_d in any bit
//   equi_probe simproj TRAJ M[,M]   -> noise-free simulator frames of a rig with these models (radtan / equi): state,
//                                      calibration, map points and their pixels
#include "../../include/ovb200_vio.hpp"
#include "../../oracle/ovo_core.hpp"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
using namespace ovb200;

static std::vector<int> parse_models(const std::string &arg) {
  std::vector<int> m;
  size_t a = 0;
  while (true) {
    const size_t b = arg.find(',', a);
    m.push_back(arg.substr(a, b == std::string::npos ? std::string::npos : b - a) == "equi" ? OVB_CAM_EQUI : OVB_CAM_RADTAN);
    if (b == std::string::npos)
      return m;
    a = b + 1;
  }
}

int main(int argc, char **argv) {
  if (argc < 2)
    return 2;
  const std::string cmd = argv[1];
  SimParams sp;
  rpng_sim_cameras(1, sp, {OVB_CAM_EQUI});
  SimCamera cam = sp.camera_intrinsics[0];
  if (cmd == "undistort") {
    for (int k = 0; k < 4 && argc >= 6; k++)
      cam.d[4 + k] = std::atof(argv[2 + k]);
    float u, v;
    while (std::scanf("%f %f", &u, &v) == 2) {
      float x, y;
      cam.undistort_f(u, v, x, y);
      std::printf("%.9g %.9g\n", x, y);
    }
    return 0;
  }
  if (cmd == "oracle") {
    // float normalized coordinates over |x|, |y| <= 3 (theta up to 1.34 rad, past the 512 x 512 image's corners), and
    // around the r = 1e-8 switch of the small-radius branch
    long n = 0, diff = 0;
    auto check = [&](float x, float y) {
      float u, v;
      cam.distort_f(x, y, u, v);
      double uo, vo;
      ovo::distort_d(OVB_CAM_EQUI, cam.d, (double)x, (double)y, uo, vo);
      n++;
      if ((double)u != uo || (double)v != vo || std::signbit(u) != std::signbit(uo) || std::signbit(v) != std::signbit(vo))
        diff++;
    };
    for (int i = -600; i <= 600; i++)
      for (int j = -600; j <= 600; j++)
        check((float)(i * 0.005), (float)(j * 0.005));
    for (int k = -40; k <= 40; k++)
      for (int s = 0; s < 4; s++) {
        const float t = (float)(1e-8 * std::pow(10.0, k / 20.0));
        check(s & 1 ? -t : t, s & 2 ? t : 0.0f);
      }
    std::printf("%ld %ld\n", n, diff);
    return 0;
  }
  if (cmd == "simproj" && argc >= 4) {
    // first camera frames of a noise-free simulator: ground-truth IMU state, extrinsics, model, intrinsics and, per camera,
    // the map points with their simulated pixels — for a projection with OpenCV on the Python side
    const std::string traj = argv[2];
    auto data = traj.substr(traj.size() - 4) == ".bin" ? load_trajectory_bin(traj) : load_simulated_trajectory(traj);
    const std::vector<int> models = parse_models(argv[3]);
    rpng_sim_cameras((int)models.size(), sp, models);
    sp.use_stereo = models.size() > 1;
    sp.sigma_pix = 0.0;
    sp.num_pts = 60;
    Simulator sim(sp, data);
    int frames = 0;
    bool pending = false;
    double tc_pending = 0;
    std::vector<int> camids_p;
    std::vector<std::vector<SimFeat>> feats_p;
    while (sim.ok() && frames < 3) {
      double t;
      Vec3 wm, am;
      sim.get_next_imu(t, wm, am);
      std::array<double, 17> st;
      // the true-bias history (which get_state interpolates) trails the camera time by an IMU sample: ask again after the next one
      if (pending && sim.get_state(tc_pending + sp.calib_camimu_dt, st)) {
        pending = false;
        frames++;
        for (size_t c = 0; c < camids_p.size(); c++) {
          const int ci = camids_p[c];
          const SimCamera &k = sp.camera_intrinsics[(size_t)ci];
          std::printf("FRAME %d %zu", ci, feats_p[c].size());
          for (int i = 1; i < 8; i++) std::printf(" %.17g", st[(size_t)i]); // q_GtoI (JPL xyzw), p_IinG
          const Vec4 &qe = sp.camera_extrinsics[(size_t)ci].first;
          const Vec3 &pe = sp.camera_extrinsics[(size_t)ci].second;
          std::printf(" %.17g %.17g %.17g %.17g %.17g %.17g %.17g", qe[0], qe[1], qe[2], qe[3], pe[0], pe[1], pe[2]);
          std::printf(" %d %d %d", k.model, k.w, k.h);
          for (int i = 0; i < 8; i++) std::printf(" %.17g", k.d[i]);
          std::printf("\n");
          for (const SimFeat &f : feats_p[c]) {
            const size_t id = sp.use_stereo ? f.id : f.id - (size_t)ci * sim.featmap.size();
            const Vec3 &P = sim.featmap.at(id);
            std::printf("%.17g %.17g %.17g %.9g %.9g\n", P[0], P[1], P[2], (double)f.u, (double)f.v);
          }
        }
      }
      double tc;
      std::vector<int> camids;
      std::vector<std::vector<SimFeat>> feats;
      if (!pending && sim.get_next_cam(tc, camids, feats)) {
        pending = true;
        tc_pending = tc;
        camids_p = camids;
        feats_p = feats;
      }
    }
    return 0;
  }
  return 2;
}
