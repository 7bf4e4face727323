// Drives one UpdaterSLAM::update through the C++ host mirror (include/ovb200_host.hpp) with landmarks of two classes in
// their own representations (Landmark::_feat_representation): reads a flat little-endian case file written by
// tests/test_gpu_slam_reps.py, rebuilds State / Feature / Landmark objects, runs the update and writes dx, P and the
// per-feature status back.
#include "ovb200_host.hpp"

#include <cstdio>
#include <fstream>

using namespace ovb200;

template <class T> static std::vector<T> rd(std::ifstream &f, size_t n) {
  std::vector<T> v(n);
  f.read(reinterpret_cast<char *>(v.data()), (std::streamsize)(n * sizeof(T)));
  if (!f)
    throw std::runtime_error("short read");
  return v;
}
template <class T> static void wr(std::ofstream &f, const std::vector<T> &v) { f.write(reinterpret_cast<const char *>(v.data()), (std::streamsize)(v.size() * sizeof(T))); }

int main(int argc, char **argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: %s case.bin out.bin\n", argv[0]);
    return 2;
  }
  try {
    std::ifstream in(argv[1], std::ios::binary);
    auto hdr = rd<int32_t>(in, 8);
    const int C = hdr[0], K = hdr[1], N = hdr[2], F = hdr[3], M = hdr[4];
    auto dpar = rd<double>(in, 4); // sigma_pix / chi2_multipler of the SLAM class, then of the ArUco class
    auto clone_times = rd<double>(in, C);
    auto clone_R = rd<double>(in, 9 * C), clone_p = rd<double>(in, 3 * C), clone_Rf = rd<double>(in, 9 * C), clone_pf = rd<double>(in, 3 * C);
    auto clone_off = rd<int32_t>(in, C);
    auto cam_R = rd<double>(in, 9 * K), cam_p = rd<double>(in, 3 * K), cam_intr = rd<double>(in, 8 * K);
    auto cam_model = rd<int32_t>(in, K), cam_ext = rd<int32_t>(in, K), cam_in = rd<int32_t>(in, K);
    auto P = rd<double>(in, (size_t)N * N);
    auto meas_off = rd<int32_t>(in, F + 1);
    auto mcam = rd<uint8_t>(in, M);
    auto mclone = rd<uint16_t>(in, M);
    auto uv = rd<float>(in, 2 * (size_t)M), uvn = rd<float>(in, 2 * (size_t)M);
    auto lm_off = rd<int32_t>(in, F), rep = rd<int32_t>(in, F), acam = rd<int32_t>(in, F), aclone = rd<int32_t>(in, F);
    auto value = rd<double>(in, 3 * (size_t)F), value_fej = rd<double>(in, 3 * (size_t)F);

    StateOptions so;
    so.do_fej = hdr[5];
    so.do_calib_camera_pose = hdr[6];
    so.do_calib_camera_intrinsics = hdr[6];
    so.num_cameras = K;
    so.max_clone_size = C;
    so.max_aruco_features = hdr[7];
    ovb_config cfg{0, 512, 256, 8192, 0};
    State state(so, cfg);
    for (int c = 0; c < C; c++) {
      auto pose = std::make_shared<PoseJPL>();
      pose->id = clone_off[c];
      std::copy(clone_R.begin() + 9 * c, clone_R.begin() + 9 * c + 9, pose->Rot);
      std::copy(clone_p.begin() + 3 * c, clone_p.begin() + 3 * c + 3, pose->pos);
      std::copy(clone_Rf.begin() + 9 * c, clone_Rf.begin() + 9 * c + 9, pose->Rot_fej);
      std::copy(clone_pf.begin() + 3 * c, clone_pf.begin() + 3 * c + 3, pose->pos_fej);
      state._clones_IMU[clone_times[c]] = pose;
    }
    for (int k = 0; k < K; k++) {
      Camera &cam = state._cameras[k];
      cam.calib_id = cam_ext[k];
      cam.intrinsics_id = cam_in[k];
      std::copy(cam_R.begin() + 9 * k, cam_R.begin() + 9 * k + 9, cam.R_ItoC);
      std::copy(cam_p.begin() + 3 * k, cam_p.begin() + 3 * k + 3, cam.p_IinC);
      std::copy(cam_intr.begin() + 8 * k, cam_intr.begin() + 8 * k + 8, cam.intrinsics);
      cam.model = cam_model[k];
    }
    StateHelper::set_initial_covariance(state, P, N);

    std::vector<std::shared_ptr<Feature>> all, feature_vec;
    for (int f = 0; f < F; f++) {
      auto feat = std::make_shared<Feature>();
      feat->featid = (size_t)f;
      for (int i = meas_off[f]; i < meas_off[f + 1]; i++) {
        const size_t cam = mcam[i];
        feat->uvs[cam].push_back({uv[2 * i], uv[2 * i + 1]});
        feat->uvs_norm[cam].push_back({uvn[2 * i], uvn[2 * i + 1]});
        feat->timestamps[cam].push_back(clone_times[mclone[i]]);
      }
      auto lm = std::make_shared<Landmark>();
      lm->id = lm_off[f];
      lm->_featid = (size_t)f;
      lm->_feat_representation = rep[f];
      lm->_anchor_cam_id = acam[f];
      lm->_anchor_clone_timestamp = aclone[f] >= 0 ? clone_times[aclone[f]] : -1.0;
      std::copy(value.begin() + 3 * f, value.begin() + 3 * f + 3, lm->xyz);
      std::copy(value_fej.begin() + 3 * f, value_fej.begin() + 3 * f + 3, lm->xyz_fej);
      state._features_SLAM[(size_t)f] = lm;
      all.push_back(feat);
      feature_vec.push_back(feat);
    }
    UpdaterOptions o_slam, o_aruco;
    o_slam.sigma_pix = dpar[0];
    o_slam.chi2_multipler = dpar[1];
    o_aruco.sigma_pix = dpar[2];
    o_aruco.chi2_multipler = dpar[3];
    FeatureInitializerOptions fo;
    UpdaterSLAM updater(o_slam, o_aruco, fo);
    updater.col_order = OVB_COLS_CANONICAL;
    std::vector<double> dx = updater.update(state, feature_vec);
    std::vector<double> Ppost = StateHelper::get_full_covariance(state);
    std::vector<int32_t> st(F);
    for (int f = 0; f < F; f++)
      st[f] = all[f]->last_status;
    std::ofstream out(argv[2], std::ios::binary);
    wr(out, dx);
    wr(out, Ppost);
    wr(out, st);
    return 0;
  } catch (const std::exception &e) {
    std::fprintf(stderr, "slam_reps_host_test: %s\n", e.what());
    return 1;
  }
}
