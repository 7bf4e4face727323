// Drives the end-of-frame window shift through the C++ host mirror (include/ovb200_host.hpp) twice on the same synthetic
// state: the reference's three steps (StateHelper::marginalize_slam, UpdaterSLAM::change_anchors,
// StateHelper::marginalize_old_clone) on one State, ovb200::marginalize_window on the other. The covariance must agree bit
// for bit, and so must every id, landmark value and anchor. Prints "window_shim_test: ok" on success.
// build: g++ -std=c++17 -O2 -I include tests/cpp/window_shim_test.cpp -L open_vins_b200 -lovb200 -Wl,-rpath,... -o window_shim_test
#include "ovb200_host.hpp"

#include <cmath>
#include <cstdio>
#include <cstring>

using namespace ovb200;

static void rot(double ax, double ay, double az, double R[9]) { // Rodrigues
  const double th = std::sqrt(ax * ax + ay * ay + az * az), k[3] = {ax / th, ay / th, az / th};
  const double c = std::cos(th), s = std::sin(th), K[9] = {0, -k[2], k[1], k[2], 0, -k[0], -k[1], k[0], 0};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      double k2 = 0;
      for (int m = 0; m < 3; m++)
        k2 += K[3 * i + m] * K[3 * m + j];
      R[3 * i + j] = (i == j ? 1.0 : 0.0) + s * K[3 * i + j] + (1 - c) * k2;
    }
}

static const int C = 8, NCAM = 2, NLM = 14;

// IMU (15), extrinsics of both cameras, the clone window, then the landmarks; a symmetric positive definite P
static void fill(State &st, UpdaterSLAM &) {
  int id = 15;
  for (int k = 0; k < NCAM; k++) {
    Camera &cam = st._cameras[(size_t)k];
    cam.calib_id = id;
    id += 6;
    rot(0.1 + 0.2 * k, -0.3, 1.2 + 0.1 * k, cam.R_ItoC);
    cam.p_IinC[0] = 0.05 * (k + 1), cam.p_IinC[1] = -0.02, cam.p_IinC[2] = 0.01 * k;
  }
  for (int c = 0; c < C; c++) {
    auto pose = std::make_shared<PoseJPL>();
    pose->id = id;
    id += 6;
    rot(0.05 * c + 0.1, 0.02 * c - 0.2, 0.3, pose->Rot);
    rot(0.05 * c + 0.1001, 0.02 * c - 0.2, 0.3002, pose->Rot_fej);
    pose->pos[0] = 0.4 * c, pose->pos[1] = 0.1 * std::sin(c), pose->pos[2] = 0.05 * c;
    for (int i = 0; i < 3; i++)
      pose->pos_fej[i] = pose->pos[i] + 1e-3 * (i + 1);
    st._clones_IMU[10.0 + 0.1 * c] = pose;
  }
  const int reps[3] = {OVB_REP_ANCHORED_3D, OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH, OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE};
  for (int l = 0; l < NLM; l++) {
    auto lm = std::make_shared<Landmark>();
    lm->_featid = (size_t)(100 + l);
    lm->_feat_representation = reps[l % 3];
    lm->id = id;
    id += lm->size();
    lm->_anchor_cam_id = l % NCAM;
    lm->_anchor_clone_timestamp = (l % 4 == 3) ? 10.2 : 10.0; // most of them in the oldest clone
    lm->xyz[0] = 0.3 * std::sin(l), lm->xyz[1] = 0.2 * std::cos(l), lm->xyz[2] = 3.0 + 0.1 * l;
    for (int i = 0; i < 3; i++)
      lm->xyz_fej[i] = lm->xyz[i] + 2e-3 * (i - 1);
    lm->should_marg = (l % 5 == 4);
    st._features_SLAM[lm->_featid] = lm;
  }
  const int N = id;
  std::vector<double> P((size_t)N * N);
  for (int i = 0; i < N; i++)
    for (int j = 0; j < N; j++) {
      const int d = i > j ? i - j : j - i;
      P[(size_t)i * N + j] = 0.01 * std::exp(-0.3 * d) * (1.0 + 0.1 * std::cos(0.7 * (i + j))) + (i == j ? 0.02 : 0.0);
    }
  StateHelper::set_initial_covariance(st, P, N);
}

int main() {
  try {
    StateOptions so;
    so.do_fej = true;
    so.do_calib_camera_pose = true;
    so.num_cameras = NCAM;
    so.max_clone_size = C - 1;
    ovb_config cfg{0, 256, 16, 256, 0};
    UpdaterOptions uo;
    FeatureInitializerOptions fo;
    State a(so, cfg), b(so, cfg);
    UpdaterSLAM ua(uo, uo, fo), ub(uo, uo, fo);
    fill(a, ua);
    fill(b, ub);
    // ---- the reference's three steps on a
    for (auto it = a._features_SLAM.begin(); it != a._features_SLAM.end();) { // StateHelper::marginalize_slam
      if (it->second->should_marg && (int)it->first > 4 * a._options.max_aruco_features) {
        const Var v(it->second->id, it->second->size());
        StateHelper::marginalize(a, v);
        for (auto &c : a._clones_IMU)
          if (c.second->id > v.first)
            c.second->id -= v.second;
        for (auto &cam : a._cameras)
          if (cam.calib_id > v.first)
            cam.calib_id -= v.second;
        for (auto &f : a._features_SLAM)
          if (f.second->id > v.first)
            f.second->id -= v.second;
        it = a._features_SLAM.erase(it);
      } else {
        ++it;
      }
    }
    ua.change_anchors(a);
    StateHelper::marginalize_old_clone(a);
    // ---- one call on b
    marginalize_window(b, ub);
    const std::vector<double> Pa = StateHelper::get_full_covariance(a), Pb = StateHelper::get_full_covariance(b);
    if (Pa.size() != Pb.size() || std::memcmp(Pa.data(), Pb.data(), sizeof(double) * Pa.size()) != 0)
      throw std::runtime_error("covariances differ");
    if (a._clones_IMU.size() != b._clones_IMU.size() || a._features_SLAM.size() != b._features_SLAM.size())
      throw std::runtime_error("different variables left");
    for (auto ia = a._clones_IMU.begin(), ib = b._clones_IMU.begin(); ia != a._clones_IMU.end(); ++ia, ++ib)
      if (ia->first != ib->first || ia->second->id != ib->second->id)
        throw std::runtime_error("clone ids differ");
    for (int k = 0; k < NCAM; k++)
      if (a._cameras[(size_t)k].calib_id != b._cameras[(size_t)k].calib_id)
        throw std::runtime_error("camera ids differ");
    int moved = 0;
    for (auto &f : a._features_SLAM) {
      const Landmark &la = *f.second, &lb = *b._features_SLAM.at(f.first);
      if (la.id != lb.id || la._anchor_cam_id != lb._anchor_cam_id || la._anchor_clone_timestamp != lb._anchor_clone_timestamp ||
          std::memcmp(la.xyz, lb.xyz, sizeof(la.xyz)) != 0 || std::memcmp(la.xyz_fej, lb.xyz_fej, sizeof(la.xyz_fej)) != 0)
        throw std::runtime_error("landmark " + std::to_string(f.first) + " differs");
      moved += la._anchor_clone_timestamp == a._clones_IMU.rbegin()->first;
    }
    if (moved < 5 || (int)a._features_SLAM.size() >= NLM)
      throw std::runtime_error("the case re-anchored or lost too few landmarks");
    std::printf("window_shim_test: ok (N %d, %d landmarks re-anchored, %d lost)\n", a.max_covariance_size(), moved, NLM - (int)a._features_SLAM.size());
    return 0;
  } catch (const std::exception &e) {
    std::fprintf(stderr, "window_shim_test: %s\n", e.what());
    return 1;
  }
}
