// ovb200_host.hpp — header-only C++17 host side above the C ABI of ovb200.h.
//
// Mirrors the slice of the reference's C++ class surface that sits on the MSCKF-update path, with the same names,
// argument meaning and call order, so that code written against the reference reads the same here:
//   ov_core::Feature                      ov_core/src/feat/Feature.h:39-83, Feature.cpp:26-110
//   ov_type::PoseJPL (clone poses)        ov_core/src/types/PoseJPL.h
//   ov_msckf::State                       ov_msckf/src/state/State.h:49-193
//   ov_msckf::StateHelper                 ov_msckf/src/state/StateHelper.h (EKFPropagation, EKFUpdate, clone, marginalize, ...)
//   ov_msckf::UpdaterMSCKF::update        ov_msckf/src/update/UpdaterMSCKF.cpp:58-295
//   ov_type::Landmark, UpdaterSLAM::update ov_core/src/types/Landmark.h, ov_msckf/src/update/UpdaterSLAM.cpp:253-479
// What differs, on purpose:
//   * no Eigen: matrices are row-major std::vector<double>; rotations are 3x3 row-major R_GtoI / R_ItoC (JPL convention);
//   * the covariance lives on the GPU inside the engine context (State owns an ovb_ctx instead of an Eigen _Cov);
//   * errors: where the reference calls std::exit(EXIT_FAILURE) (StateHelper.cpp:131-145, :192-195) this layer throws
//     ovb200::Error carrying the ovb_status and ovb_last_error() text;
//   * EKFUpdate / UpdaterMSCKF::update RETURN the correction dx = K*res instead of applying it: the mean of the state
//     (quaternions, FEJ bookkeeping: Type::update, StateHelper.cpp:185-188) stays with the caller's State types.
// Link with -lovb200 (open_vins_b200/libovb200.so).
#ifndef OVB200_HOST_HPP
#define OVB200_HOST_HPP

#include "ovb200.h"

#include <algorithm>
#include <array>
#include <cstdint>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace ovb200 {

struct Error : std::runtime_error {
  ovb_status status;
  Error(ovb_status s, const std::string &what) : std::runtime_error(what), status(s) {}
};

// ---------------------------------------------------------------------------------------------------------------------
// ov_core::Feature (feat/Feature.h:39-83). uvs / uvs_norm are float32 pairs as in the reference (Eigen::VectorXf).
struct Feature {
  size_t featid = 0;
  bool to_delete = false;
  std::unordered_map<size_t, std::vector<std::array<float, 2>>> uvs;
  std::unordered_map<size_t, std::vector<std::array<float, 2>>> uvs_norm;
  std::unordered_map<size_t, std::vector<double>> timestamps;
  int anchor_cam_id = -1;
  double anchor_clone_timestamp = -1;
  double p_FinA[3] = {0, 0, 0};
  double p_FinG[3] = {0, 0, 0};
  // diagnostics of the last update this feature entered (not in the reference): ovb_feat_status and chi²
  int last_status = OVB_FEAT_OK;
  double last_chi2 = 0;

  // Feature::clean_old_measurements(const std::vector<double>&) — keep only measurements at the given times
  // (feat/Feature.cpp:26-53)
  void clean_old_measurements(const std::vector<double> &valid_times) {
    for (auto &pair : timestamps) {
      auto &ts = pair.second;
      auto &uv = uvs[pair.first];
      auto &uvn = uvs_norm[pair.first];
      size_t w = 0;
      for (size_t i = 0; i < ts.size(); i++) {
        if (std::find(valid_times.begin(), valid_times.end(), ts[i]) != valid_times.end()) {
          ts[w] = ts[i];
          uv[w] = uv[i];
          uvn[w] = uvn[i];
          w++;
        }
      }
      ts.resize(w);
      uv.resize(w);
      uvn.resize(w);
    }
  }
};

// ov_type::PoseJPL reduced to what the path reads: Rot(), pos(), Rot_fej(), pos_fej(), id() (types/PoseJPL.h, Type.h:57)
struct PoseJPL {
  int id = -1; // first row/column of the 6-wide (theta, p) block in the covariance
  double Rot[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  double pos[3] = {0, 0, 0};
  double Rot_fej[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  double pos_fej[3] = {0, 0, 0};
  int size() const { return 6; }
};

// one camera of State::_calib_IMUtoCAM / _cam_intrinsics / _cam_intrinsics_cameras (state/State.h:157-166)
struct Camera {
  int calib_id = -1;      // covariance id of the 6-wide extrinsics (or -1 when not estimated)
  int intrinsics_id = -1; // covariance id of the 8-wide intrinsics (or -1)
  double R_ItoC[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  double p_IinC[3] = {0, 0, 0};
  double intrinsics[8] = {0, 0, 0, 0, 0, 0, 0, 0}; // fx fy cx cy d0 d1 d2 d3
  int model = OVB_CAM_RADTAN;                      // cam/CamRadtan.h or cam/CamEqui.h
};

// ov_type::Landmark (types/Landmark.h:35-97) reduced to what UpdaterSLAM::update reads. xyz / xyz_fej are what
// Landmark::get_xyz(false) / get_xyz(true) return (p_FinG for the global representations, p_FinA for the anchored ones);
// the caller's Landmark keeps the representation's own parameters and applies dx to them.
struct Landmark {
  int id = -1; // first row/column of the 3-wide block in the covariance
  size_t _featid = 0;
  int _feat_representation = OVB_REP_GLOBAL_3D;
  int _anchor_cam_id = -1;
  double _anchor_clone_timestamp = -1;
  double xyz[3] = {0, 0, 0};
  double xyz_fej[3] = {0, 0, 0};
  int update_fail_count = 0;
  bool should_marg = false;
  int size() const { return _feat_representation == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3; }
};

// the StateOptions fields the path reads (state/StateOptions.h:35-176)
struct StateOptions {
  bool do_fej = true;
  bool do_calib_camera_pose = false;
  bool do_calib_camera_intrinsics = false;
  int feat_rep_msckf = OVB_REP_GLOBAL_3D;
  int num_cameras = 1;
  int max_clone_size = 11;
  int feat_rep_slam = OVB_REP_GLOBAL_3D;
  int feat_rep_aruco = OVB_REP_GLOBAL_3D; // representation of new ArUco landmarks (delayed_init picks it by featid)
  int max_aruco_features = 0; // feature ids below this are ArUco tags with their own noise / gate (UpdaterSLAM.cpp:391-393)
};

// ov_msckf::State (state/State.h:49-193): the sliding window and calibration; the covariance is device-resident.
class State {
public:
  StateOptions _options;
  std::map<double, std::shared_ptr<PoseJPL>> _clones_IMU; // State.h:130
  std::vector<Camera> _cameras;                           // index = camera id
  std::unordered_map<size_t, std::shared_ptr<Landmark>> _features_SLAM; // State.h:172

  State(const StateOptions &options, const ovb_config &cfg) : _options(options) {
    ovb_status st = ovb_create(&cfg, &_ctx);
    if (st != OVB_OK)
      throw Error(st, std::string("ovb_create: ") + (_ctx ? ovb_last_error(_ctx) : "no context (is a CUDA GPU visible?)"));
    _cameras.resize((size_t)options.num_cameras);
  }
  ~State() {
    if (_ctx)
      ovb_destroy(_ctx);
  }
  State(const State &) = delete;
  State &operator=(const State &) = delete;

  int max_covariance_size() const { return ovb_cov_dim(_ctx); } // State.h:96
  ovb_ctx *ctx() const { return _ctx; }
  void check(ovb_status st, const char *where) const {
    if (st != OVB_OK)
      throw Error(st, std::string(where) + ": " + ovb_last_error(_ctx));
  }

private:
  ovb_ctx *_ctx = nullptr;
};

// (id, size) of a state variable, the role std::shared_ptr<ov_type::Type> plays in the reference's argument lists
using Var = std::pair<int, int>;

// ov_msckf::StateHelper (state/StateHelper.h) on the device-resident covariance
struct StateHelper {
  // StateHelper::set_initial_covariance / a full re-sync (StateHelper.cpp:199-224)
  static void set_initial_covariance(State &state, const std::vector<double> &P, int N) { state.check(ovb_cov_set(state.ctx(), P.data(), N), "set_initial_covariance"); }
  // StateHelper::get_full_covariance (StateHelper.cpp:256-269)
  static std::vector<double> get_full_covariance(State &state) {
    const int N = state.max_covariance_size();
    std::vector<double> P((size_t)N * N);
    state.check(ovb_cov_get(state.ctx(), P.data(), N), "get_full_covariance");
    return P;
  }
  // StateHelper::get_marginal_covariance (StateHelper.cpp:226-254)
  static std::vector<double> get_marginal_covariance(State &state, const std::vector<Var> &small_variables) {
    std::vector<int> off, sz;
    int n = 0;
    for (auto &v : small_variables) {
      off.push_back(v.first);
      sz.push_back(v.second);
      n += v.second;
    }
    std::vector<double> out((size_t)n * n);
    state.check(ovb_cov_get_marginal(state.ctx(), off.data(), sz.data(), (int)off.size(), out.data()), "get_marginal_covariance");
    return out;
  }
  // StateHelper::EKFPropagation (StateHelper.cpp:36-114). order_NEW must be contiguous in the covariance (the reference
  // asserts the same, :58-66). Phi is (sum new sizes) x (sum old sizes), Q square, both row-major.
  static void EKFPropagation(State &state, const std::vector<Var> &order_NEW, const std::vector<Var> &order_OLD, const std::vector<double> &Phi,
                             const std::vector<double> &Q) {
    if (order_NEW.empty() || order_OLD.empty())
      throw Error(OVB_ERR_ARG, "EKFPropagation: called with empty variable arrays"); // StateHelper.cpp:42-46
    int p = 0;
    for (size_t i = 0; i < order_NEW.size(); i++) {
      if (i > 0 && order_NEW[i].first != order_NEW[i - 1].first + order_NEW[i - 1].second)
        throw Error(OVB_ERR_ARG, "EKFPropagation: non-contiguous state elements"); // StateHelper.cpp:58-66
      p += order_NEW[i].second;
    }
    std::vector<int> off, sz;
    for (auto &v : order_OLD) {
      off.push_back(v.first);
      sz.push_back(v.second);
    }
    state.check(ovb_cov_propagate(state.ctx(), order_NEW[0].first, p, off.data(), sz.data(), (int)off.size(), Phi.data(), Q.data()), "EKFPropagation");
  }
  // StateHelper::EKFUpdate (StateHelper.cpp:116-197) with R = sigma2 * I (Rdiag empty) or R = diag(Rdiag).
  // H is res.size() x (sum of H_order sizes), row-major. Returns dx (length max_covariance_size()).
  static std::vector<double> EKFUpdate(State &state, const std::vector<Var> &H_order, const std::vector<double> &H, const std::vector<double> &res,
                                       double sigma2, const std::vector<double> &Rdiag = {}) {
    std::vector<int> off, sz;
    for (auto &v : H_order) {
      off.push_back(v.first);
      sz.push_back(v.second);
    }
    std::vector<double> dx((size_t)state.max_covariance_size());
    state.check(ovb_ekf_update(state.ctx(), off.data(), sz.data(), (int)off.size(), H.data(), (int)res.size(), res.data(), sigma2,
                               Rdiag.empty() ? nullptr : Rdiag.data(), dx.data()),
                "EKFUpdate");
    return dx;
  }
  // StateHelper::clone (StateHelper.cpp:341-391): appends a copy of the variable to the end of the covariance and
  // returns the id of the new block. dnc_dt (6 values) + dt_id add augment_clone's time-offset term (:604-615).
  static int clone(State &state, const Var &variable_to_clone, const double *dnc_dt = nullptr, int dt_id = -1) {
    const int new_id = state.max_covariance_size();
    state.check(ovb_cov_clone(state.ctx(), variable_to_clone.first, variable_to_clone.second, dnc_dt, dt_id), "clone");
    return new_id;
  }
  // StateHelper::initialize (StateHelper.cpp:393-482): add `new_variable` (id assigned here = old covariance size) from
  // res = H_R dx(H_order) + H_L dx(new) + n, n ~ N(0, sigma2 I). Returns false when the Mahalanobis gate rejects (state
  // untouched). dx_new = the new variable's own correction, dx = EKF correction of the projected part (length = new size).
  static bool initialize(State &state, Var &new_variable, const std::vector<Var> &H_order, const std::vector<double> &H_R,
                         const std::vector<double> &H_L, const std::vector<double> &res, double sigma2, double chi_2_mult,
                         std::vector<double> &dx_new, std::vector<double> &dx) {
    std::vector<int> off, sz;
    for (auto &v : H_order) {
      off.push_back(v.first);
      sz.push_back(v.second);
    }
    const int k = new_variable.second, old_size = state.max_covariance_size();
    int accepted = 0;
    dx_new.assign((size_t)k, 0.0);
    dx.assign((size_t)(old_size + k), 0.0);
    state.check(ovb_cov_initialize(state.ctx(), off.data(), sz.data(), (int)off.size(), H_R.data(), H_L.data(), res.data(), (int)res.size(), k,
                                   sigma2, chi_2_mult, &accepted, dx_new.data(), dx.data()),
                "initialize");
    if (!accepted)
      return false;
    new_variable.first = old_size; // new_variable->set_local_id(oldSize) (StateHelper.cpp:571)
    return true;
  }
  // StateHelper::marginalize (StateHelper.cpp:271-339). The caller shifts the ids of the variables behind the removed one
  // exactly as the reference does (:318-326); marginalize_old_clone below does it for the clone window.
  static void marginalize(State &state, const Var &marg) { state.check(ovb_cov_marginalize(state.ctx(), marg.first, marg.second), "marginalize"); }
  // StateHelper::marginalize_old_clone (StateHelper.cpp:618-629)
  static void marginalize_old_clone(State &state) {
    if ((int)state._clones_IMU.size() <= state._options.max_clone_size)
      return;
    auto it = state._clones_IMU.begin();
    const Var marg(it->second->id, it->second->size());
    marginalize(state, marg);
    state._clones_IMU.erase(it);
    for (auto &c : state._clones_IMU)
      if (c.second->id > marg.first)
        c.second->id -= marg.second;
    for (auto &cam : state._cameras) {
      if (cam.calib_id > marg.first)
        cam.calib_id -= marg.second;
      if (cam.intrinsics_id > marg.first)
        cam.intrinsics_id -= marg.second;
    }
    // every variable behind the removed block moves up (StateHelper.cpp:318-326): SLAM landmarks are appended at the end of
    // the covariance by initialize(), i.e. always behind the oldest clone
    for (auto &lm : state._features_SLAM)
      if (lm.second->id > marg.first)
        lm.second->id -= marg.second;
  }
};

// ov_msckf::UpdaterOptions (update/UpdaterOptions.h:32-48) and ov_core::FeatureInitializerOptions
// (feat/FeatureInitializerOptions.h:33-69), same field names and defaults
struct UpdaterOptions {
  double chi2_multipler = 5;
  double sigma_pix = 1;
};
struct FeatureInitializerOptions {
  bool triangulate_1d = false;
  bool refine_features = true;
  int max_runs = 5;
  double init_lamda = 1e-3;
  double max_lamda = 1e10;
  double min_dx = 1e-6;
  double min_dcost = 1e-6;
  double lam_mult = 10;
  double min_dist = 0.10;
  double max_dist = 60;
  double max_baseline = 40;
  double max_cond_number = 10000;
};

// ov_msckf::UpdaterMSCKF (update/UpdaterMSCKF.h, UpdaterMSCKF.cpp:58-295)
class UpdaterMSCKF {
public:
  UpdaterMSCKF(const UpdaterOptions &options, const FeatureInitializerOptions &feat_init_options) : _options(options), _init(feat_init_options) {}

  // Engine-specific knobs (no counterpart in the reference): column order of the stacked system, compression mode
  int col_order = OVB_COLS_REFERENCE_FIRST_SEEN;
  int compress = OVB_COMPRESS_HOUSEHOLDER_TSQR;
  ovb_stats last_stats{};

  // update(state, feature_vec): cleans the features' measurements to the clone times, drops features with < 2
  // measurements, triangulates, builds/gates/stacks/compresses and updates the covariance on the GPU. As in the
  // reference, feature_vec shrinks to the features that were used (all marked to_delete, UpdaterMSCKF.cpp:276-279);
  // rejected features are marked to_delete and erased (:139-149, :226-231). Returns dx.
  std::vector<double> update(State &state, std::vector<std::shared_ptr<Feature>> &feature_vec) {
    std::vector<double> dx((size_t)state.max_covariance_size(), 0.0);
    if (feature_vec.empty())
      return dx; // UpdaterMSCKF.cpp:61-62
    // 0. clone times (UpdaterMSCKF.cpp:70-74); std::map iterates oldest -> newest: that is the engine's clone index
    std::vector<double> clonetimes;
    for (const auto &c : state._clones_IMU)
      clonetimes.push_back(c.first);
    // 1. clean measurements, drop features with fewer than two (UpdaterMSCKF.cpp:77-96)
    for (auto it = feature_vec.begin(); it != feature_vec.end();) {
      (*it)->clean_old_measurements(clonetimes);
      int ct_meas = 0;
      for (const auto &pair : (*it)->timestamps)
        ct_meas += (int)pair.second.size();
      if (ct_meas < 2) {
        (*it)->to_delete = true;
        it = feature_vec.erase(it);
      } else
        ++it;
    }
    if (feature_vec.empty())
      return dx;
    // 2. marshal the window (UpdaterMSCKF.cpp:98-115 reads exactly these) and the features (structure-of-arrays;
    //    cameras in the visit order of `for (auto const &pair : feat->timestamps)`, SURVEY.md App. A.4)
    const int C = (int)state._clones_IMU.size(), K = (int)state._cameras.size();
    std::vector<double> cR((size_t)9 * C), cp((size_t)3 * C), cRf((size_t)9 * C), cpf((size_t)3 * C), kR((size_t)9 * K), kp((size_t)3 * K), kin((size_t)8 * K);
    std::vector<int> coff((size_t)C), kmodel((size_t)K), kext((size_t)K), kintr((size_t)K);
    {
      int c = 0;
      for (const auto &cl : state._clones_IMU) {
        std::copy(cl.second->Rot, cl.second->Rot + 9, cR.begin() + 9 * c);
        std::copy(cl.second->pos, cl.second->pos + 3, cp.begin() + 3 * c);
        std::copy(cl.second->Rot_fej, cl.second->Rot_fej + 9, cRf.begin() + 9 * c);
        std::copy(cl.second->pos_fej, cl.second->pos_fej + 3, cpf.begin() + 3 * c);
        coff[c] = cl.second->id;
        c++;
      }
      for (int k = 0; k < K; k++) {
        const Camera &cam = state._cameras[k];
        std::copy(cam.R_ItoC, cam.R_ItoC + 9, kR.begin() + 9 * k);
        std::copy(cam.p_IinC, cam.p_IinC + 3, kp.begin() + 3 * k);
        std::copy(cam.intrinsics, cam.intrinsics + 8, kin.begin() + 8 * k);
        kmodel[k] = cam.model;
        kext[k] = state._options.do_calib_camera_pose ? cam.calib_id : -1;
        kintr[k] = state._options.do_calib_camera_intrinsics ? cam.intrinsics_id : -1;
      }
    }
    ovb_frame frame{C, K, cR.data(), cp.data(), cRf.data(), cpf.data(), coff.data(), kR.data(), kp.data(), kin.data(), kmodel.data(), kext.data(), kintr.data()};
    const int F = (int)feature_vec.size();
    meas_off.assign(1, 0);
    keys_off.assign(1, 0);
    cam.clear();
    clone.clear();
    uv.clear();
    uvn.clear();
    keys.clear();
    for (const auto &feat : feature_vec) {
      for (const auto &pair : feat->timestamps) {
        keys.push_back((uint8_t)pair.first);
        const auto &fuv = feat->uvs.at(pair.first);
        const auto &fuvn = feat->uvs_norm.at(pair.first);
        for (size_t m = 0; m < pair.second.size(); m++) {
          const int ci = (int)(std::lower_bound(clonetimes.begin(), clonetimes.end(), pair.second[m]) - clonetimes.begin());
          cam.push_back((uint8_t)pair.first);
          clone.push_back((uint16_t)ci);
          uv.push_back(fuv[m][0]);
          uv.push_back(fuv[m][1]);
          uvn.push_back(fuvn[m][0]);
          uvn.push_back(fuvn[m][1]);
        }
      }
      meas_off.push_back((int32_t)cam.size());
      keys_off.push_back((int32_t)keys.size());
    }
    ovb_feat_batch batch{F, (int)cam.size(), meas_off.data(), cam.data(), clone.data(), uv.data(), uvn.data(), keys_off.data(), keys.data()};
    // 3. options: UpdaterOptions + FeatureInitializerOptions + the StateOptions fields
    ovb_opts o;
    ovb_opts_default(&o);
    o.triangulate_1d = _init.triangulate_1d;
    o.refine_features = _init.refine_features;
    o.max_runs = _init.max_runs;
    o.init_lamda = _init.init_lamda;
    o.max_lamda = _init.max_lamda;
    o.min_dx = _init.min_dx;
    o.min_dcost = _init.min_dcost;
    o.lam_mult = _init.lam_mult;
    o.min_dist = _init.min_dist;
    o.max_dist = _init.max_dist;
    o.max_baseline = _init.max_baseline;
    o.max_cond_number = _init.max_cond_number;
    o.sigma_pix = _options.sigma_pix;
    o.chi2_multipler = _options.chi2_multipler;
    o.do_fej = state._options.do_fej;
    o.feat_rep = state._options.feat_rep_msckf;
    o.do_calib_camera_pose = state._options.do_calib_camera_pose;
    o.do_calib_camera_intrinsics = state._options.do_calib_camera_intrinsics;
    o.col_order = col_order;
    o.compress = compress;
    // 4. the device pipeline (UpdaterMSCKF.cpp:117-285)
    std::vector<int32_t> status((size_t)F), acam((size_t)F), aclone((size_t)F);
    std::vector<double> pA((size_t)3 * F), pG((size_t)3 * F), chi2((size_t)F);
    ovb_feat_out out{status.data(), pA.data(), pG.data(), acam.data(), aclone.data(), chi2.data()};
    state.check(ovb_msckf_update(state.ctx(), &frame, &batch, &o, &out, dx.data(), &last_stats), "UpdaterMSCKF::update");
    // 5. write back and shrink feature_vec to the used features
    std::vector<std::shared_ptr<Feature>> used;
    for (int f = 0; f < F; f++) {
      Feature &feat = *feature_vec[(size_t)f];
      feat.last_status = status[(size_t)f];
      feat.last_chi2 = chi2[(size_t)f];
      if (acam[(size_t)f] >= 0) { // triangulated: FeatureInitializer writes these (feat/FeatureInitializer.cpp:45-46, :129-130)
        feat.anchor_cam_id = acam[(size_t)f];
        feat.anchor_clone_timestamp = clonetimes[(size_t)aclone[(size_t)f]];
        std::copy(pA.begin() + 3 * f, pA.begin() + 3 * f + 3, feat.p_FinA);
        std::copy(pG.begin() + 3 * f, pG.begin() + 3 * f + 3, feat.p_FinG);
      }
      feat.to_delete = true;
      if (status[(size_t)f] == OVB_FEAT_OK)
        used.push_back(feature_vec[(size_t)f]);
    }
    feature_vec.swap(used);
    return dx;
  }

  // the structure-of-arrays batch of the last update() (kept for inspection/tests)
  std::vector<int32_t> meas_off, keys_off;
  std::vector<uint8_t> cam, keys;
  std::vector<uint16_t> clone;
  std::vector<float> uv, uvn;

private:
  UpdaterOptions _options;
  FeatureInitializerOptions _init;
};

// ov_msckf::UpdaterSLAM::update (update/UpdaterSLAM.cpp:253-479): update of the landmarks that already live in the state.
// delayed_init composes from ovb_triangulate + ovb_feature_jacobians + StateHelper::initialize (INTEGRATION.md §3b).
class UpdaterSLAM {
public:
  UpdaterSLAM(const UpdaterOptions &options_slam, const UpdaterOptions &options_aruco, const FeatureInitializerOptions &feat_init_options)
      : _options_slam(options_slam), _options_aruco(options_aruco), _init(feat_init_options) {}

  int col_order = OVB_COLS_REFERENCE_FIRST_SEEN;
  ovb_stats last_stats{};

  // Same contract as the reference: measurements are cleaned to the clone times; features without measurements are
  // marked to_delete and dropped (:283-285); a chi² rejection bumps Landmark::update_fail_count (non-ArUco), marks the
  // feature to_delete and erases it (:409-420); what remains in feature_vec was used (all to_delete, :452-454). Returns dx.
  std::vector<double> update(State &state, std::vector<std::shared_ptr<Feature>> &feature_vec) {
    std::vector<double> dx((size_t)state.max_covariance_size(), 0.0);
    if (feature_vec.empty())
      return dx;
    std::vector<double> clonetimes;
    for (const auto &c : state._clones_IMU)
      clonetimes.push_back(c.first);
    for (auto it = feature_vec.begin(); it != feature_vec.end();) {
      (*it)->clean_old_measurements(clonetimes);
      int ct_meas = 0;
      for (const auto &pair : (*it)->timestamps)
        ct_meas += (int)pair.second.size();
      // a landmark in the single-depth representation projects the bearing out and needs two measurements (UpdaterSLAM.cpp:278-290)
      const int rep = state._features_SLAM.at((*it)->featid)->_feat_representation;
      const int required_meas = (rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE) ? 2 : 1;
      if (ct_meas < 1) {
        (*it)->to_delete = true;
        it = feature_vec.erase(it);
      } else if (ct_meas < required_meas) {
        it = feature_vec.erase(it);
      } else
        ++it;
    }
    if (feature_vec.empty())
      return dx;
    // window + cameras (same marshalling as UpdaterMSCKF::update)
    const int C = (int)state._clones_IMU.size(), K = (int)state._cameras.size();
    std::vector<double> cR((size_t)9 * C), cp((size_t)3 * C), cRf((size_t)9 * C), cpf((size_t)3 * C), kR((size_t)9 * K), kp((size_t)3 * K), kin((size_t)8 * K);
    std::vector<int> coff((size_t)C), kmodel((size_t)K), kext((size_t)K), kintr((size_t)K);
    int ci = 0;
    for (const auto &cl : state._clones_IMU) {
      std::copy(cl.second->Rot, cl.second->Rot + 9, cR.begin() + 9 * ci);
      std::copy(cl.second->pos, cl.second->pos + 3, cp.begin() + 3 * ci);
      std::copy(cl.second->Rot_fej, cl.second->Rot_fej + 9, cRf.begin() + 9 * ci);
      std::copy(cl.second->pos_fej, cl.second->pos_fej + 3, cpf.begin() + 3 * ci);
      coff[(size_t)ci++] = cl.second->id;
    }
    for (int k = 0; k < K; k++) {
      const Camera &cam = state._cameras[(size_t)k];
      std::copy(cam.R_ItoC, cam.R_ItoC + 9, kR.begin() + 9 * k);
      std::copy(cam.p_IinC, cam.p_IinC + 3, kp.begin() + 3 * k);
      std::copy(cam.intrinsics, cam.intrinsics + 8, kin.begin() + 8 * k);
      kmodel[(size_t)k] = cam.model;
      kext[(size_t)k] = state._options.do_calib_camera_pose ? cam.calib_id : -1;
      kintr[(size_t)k] = state._options.do_calib_camera_intrinsics ? cam.intrinsics_id : -1;
    }
    ovb_frame frame{C, K, cR.data(), cp.data(), cRf.data(), cpf.data(), coff.data(), kR.data(), kp.data(), kin.data(), kmodel.data(), kext.data(), kintr.data()};
    // features + their landmarks
    const int F = (int)feature_vec.size();
    std::vector<int32_t> meas_off(1, 0), keys_off(1, 0), lm_off, acam, aclone, reps;
    std::vector<uint8_t> cam, keys;
    std::vector<uint16_t> clone;
    std::vector<float> uv, uvn;
    std::vector<double> val, val_fej, sig, mult;
    for (const auto &feat : feature_vec) {
      const std::shared_ptr<Landmark> &lm = state._features_SLAM.at(feat->featid); // UpdaterSLAM.cpp:316
      for (const auto &pair : feat->timestamps) {
        keys.push_back((uint8_t)pair.first);
        const auto &fuv = feat->uvs.at(pair.first);
        const auto &fuvn = feat->uvs_norm.at(pair.first);
        for (size_t m = 0; m < pair.second.size(); m++) {
          cam.push_back((uint8_t)pair.first);
          clone.push_back((uint16_t)(std::lower_bound(clonetimes.begin(), clonetimes.end(), pair.second[m]) - clonetimes.begin()));
          uv.push_back(fuv[m][0]);
          uv.push_back(fuv[m][1]);
          uvn.push_back(fuvn[m][0]);
          uvn.push_back(fuvn[m][1]);
        }
      }
      meas_off.push_back((int32_t)cam.size());
      keys_off.push_back((int32_t)keys.size());
      lm_off.push_back(lm->id);
      reps.push_back(lm->_feat_representation);
      for (int k = 0; k < 3; k++) {
        val.push_back(lm->xyz[k]);
        val_fej.push_back(lm->xyz_fej[k]);
      }
      acam.push_back(lm->_anchor_cam_id);
      aclone.push_back(lm->_anchor_cam_id >= 0
                           ? (int32_t)(std::lower_bound(clonetimes.begin(), clonetimes.end(), lm->_anchor_clone_timestamp) - clonetimes.begin())
                           : -1);
      const bool aruco = (int)feat->featid < state._options.max_aruco_features;
      sig.push_back(aruco ? _options_aruco.sigma_pix : _options_slam.sigma_pix);
      mult.push_back(aruco ? _options_aruco.chi2_multipler : _options_slam.chi2_multipler);
    }
    ovb_feat_batch batch{F, (int)cam.size(), meas_off.data(), cam.data(), clone.data(), uv.data(), uvn.data(), keys_off.data(), keys.data()};
    ovb_landmarks lms{lm_off.data(), val.data(), val_fej.data(), acam.data(), aclone.data(), sig.data(), mult.data()};
    ovb_opts o;
    ovb_opts_default(&o);
    o.sigma_pix = _options_slam.sigma_pix;
    o.chi2_multipler = _options_slam.chi2_multipler;
    o.do_fej = state._options.do_fej;
    o.do_calib_camera_pose = state._options.do_calib_camera_pose;
    o.do_calib_camera_intrinsics = state._options.do_calib_camera_intrinsics;
    o.col_order = col_order;
    std::vector<int32_t> status((size_t)F);
    std::vector<double> chi2((size_t)F);
    ovb_feat_out out{status.data(), nullptr, nullptr, nullptr, nullptr, chi2.data()};
    // every landmark in its own representation (landmark->_feat_representation, UpdaterSLAM.cpp:327-329)
    state.check(ovb_slam_update_reps(state.ctx(), &frame, &batch, &lms, reps.data(), &o, &out, dx.data(), &last_stats), "UpdaterSLAM::update");
    std::vector<std::shared_ptr<Feature>> used;
    for (int f = 0; f < F; f++) {
      Feature &feat = *feature_vec[(size_t)f];
      feat.last_status = status[(size_t)f];
      feat.last_chi2 = chi2[(size_t)f];
      feat.to_delete = true;
      if (status[(size_t)f] == OVB_FEAT_OK)
        used.push_back(feature_vec[(size_t)f]);
      else if ((int)feat.featid >= state._options.max_aruco_features)
        state._features_SLAM.at(feat.featid)->update_fail_count++; // UpdaterSLAM.cpp:414
    }
    feature_vec.swap(used);
    return dx;
  }

  // UpdaterSLAM::change_anchors (update/UpdaterSLAM.cpp:481-504): before the oldest clone is marginalised, every landmark
  // anchored in it moves to the newest clone (same camera). The host math is ovb_slam_anchor_change, the covariance step
  // StateHelper::EKFPropagation with the 3-wide (1-wide) landmark block and Q = 0.
  void change_anchors(State &state) {
    if ((int)state._clones_IMU.size() <= state._options.max_clone_size)
      return;
    const double marg_timestep = state._clones_IMU.begin()->first; // State::margtimestep(): the oldest clone
    const double new_timestep = state._clones_IMU.rbegin()->first; // state->_timestamp: the newest clone
    std::vector<double> clonetimes;
    for (const auto &c : state._clones_IMU)
      clonetimes.push_back(c.first);
    auto clone_index = [&](double t) { return (int)(std::lower_bound(clonetimes.begin(), clonetimes.end(), t) - clonetimes.begin()); };
    for (auto &f : state._features_SLAM) {
      Landmark &lm = *f.second;
      if (lm._feat_representation == OVB_REP_GLOBAL_3D || lm._feat_representation == OVB_REP_GLOBAL_FULL_INVERSE_DEPTH)
        continue;
      if (lm._anchor_clone_timestamp != marg_timestep)
        continue;
      perform_anchor_change(state, lm, clone_index(marg_timestep), clone_index(new_timestep), new_timestep, lm._anchor_cam_id);
    }
  }

  // UpdaterSLAM::perform_anchor_change (update/UpdaterSLAM.cpp:506-647)
  void perform_anchor_change(State &state, Landmark &lm, int old_clone, int new_clone, double new_anchor_timestamp, int new_cam_id) {
    const int C = (int)state._clones_IMU.size(), K = (int)state._cameras.size();
    std::vector<double> cR((size_t)9 * C), cp((size_t)3 * C), cRf((size_t)9 * C), cpf((size_t)3 * C), kR((size_t)9 * K), kp((size_t)3 * K), kin((size_t)8 * K);
    std::vector<int> coff((size_t)C), kmodel((size_t)K), kext((size_t)K), kintr((size_t)K, -1);
    int ci = 0;
    for (const auto &cl : state._clones_IMU) {
      std::copy(cl.second->Rot, cl.second->Rot + 9, cR.begin() + 9 * ci);
      std::copy(cl.second->pos, cl.second->pos + 3, cp.begin() + 3 * ci);
      std::copy(cl.second->Rot_fej, cl.second->Rot_fej + 9, cRf.begin() + 9 * ci);
      std::copy(cl.second->pos_fej, cl.second->pos_fej + 3, cpf.begin() + 3 * ci);
      coff[(size_t)ci++] = cl.second->id;
    }
    for (int k = 0; k < K; k++) {
      const Camera &cam = state._cameras[(size_t)k];
      std::copy(cam.R_ItoC, cam.R_ItoC + 9, kR.begin() + 9 * k);
      std::copy(cam.p_IinC, cam.p_IinC + 3, kp.begin() + 3 * k);
      std::copy(cam.intrinsics, cam.intrinsics + 8, kin.begin() + 8 * k);
      kmodel[(size_t)k] = cam.model;
      kext[(size_t)k] = state._options.do_calib_camera_pose ? cam.calib_id : -1;
    }
    ovb_frame frame{C, K, cR.data(), cp.data(), cRf.data(), cpf.data(), coff.data(), kR.data(), kp.data(), kin.data(), kmodel.data(), kext.data(), kintr.data()};
    ovb_opts o;
    ovb_opts_default(&o);
    o.do_fej = state._options.do_fej;
    o.feat_rep = lm._feat_representation;
    o.do_calib_camera_pose = state._options.do_calib_camera_pose;
    double nv[3], nvf[3], Phi[3 * 27];
    int32_t off[8], sz[8], n_order = 0, n_cols = 0;
    ovb_status st = ovb_slam_anchor_change(&frame, &o, lm.id, lm.xyz, lm.xyz_fej, lm._anchor_cam_id, old_clone, new_cam_id, new_clone, nv, nvf, Phi,
                                           off, sz, &n_order, &n_cols);
    if (st != OVB_OK)
      throw Error(st, "perform_anchor_change: invalid anchor");
    const int phisize = sz[n_order - 1];
    std::vector<double> Q((size_t)phisize * phisize, 0.0);
    state.check(ovb_cov_propagate(state.ctx(), lm.id, phisize, off, sz, n_order, Phi, Q.data()), "perform_anchor_change");
    std::copy(nv, nv + 3, lm.xyz);
    std::copy(nvf, nvf + 3, lm.xyz_fej);
    lm._anchor_cam_id = new_cam_id;
    lm._anchor_clone_timestamp = new_anchor_timestamp;
  }

private:
  UpdaterOptions _options_slam, _options_aruco;
  FeatureInitializerOptions _init;
};

// The end of VioManager::do_feature_propagate_update as one ovb_marginalize_window: StateHelper::marginalize_slam (the
// landmarks with should_marg and a featid above 4 * max_aruco_features), then, when the window is full,
// UpdaterSLAM::change_anchors (every anchored landmark of the oldest clone moves to the newest clone, same camera) and
// StateHelper::marginalize_old_clone. The landmarks' values and anchors and every id afterwards are those of the three steps
// called one after the other; the covariance is bit-identical to theirs when it is symmetric, as the filter keeps it (the
// lost landmarks are then removed with the oldest clone, after the anchor changes: include/ovb200.h says why that order
// changes no bit). `updater` is the UpdaterSLAM whose change_anchors
// this replaces (it holds no state the step reads).
inline void marginalize_window(State &state, UpdaterSLAM &updater) {
  (void)updater;
  std::vector<Var> marg;
  std::vector<size_t> lost;
  for (auto &f : state._features_SLAM)
    if (f.second->should_marg && (int)f.first > 4 * state._options.max_aruco_features) {
      marg.push_back(Var(f.second->id, f.second->size()));
      lost.push_back(f.first);
    }
  const bool full = (int)state._clones_IMU.size() > state._options.max_clone_size;
  const int C = (int)state._clones_IMU.size(), K = (int)state._cameras.size();
  std::vector<double> cR((size_t)9 * C), cp((size_t)3 * C), cRf((size_t)9 * C), cpf((size_t)3 * C), kR((size_t)9 * K), kp((size_t)3 * K), kin((size_t)8 * K);
  std::vector<int> coff((size_t)C), kmodel((size_t)K), kext((size_t)K), kintr((size_t)K, -1);
  int ci = 0;
  for (const auto &cl : state._clones_IMU) {
    std::copy(cl.second->Rot, cl.second->Rot + 9, cR.begin() + 9 * ci);
    std::copy(cl.second->pos, cl.second->pos + 3, cp.begin() + 3 * ci);
    std::copy(cl.second->Rot_fej, cl.second->Rot_fej + 9, cRf.begin() + 9 * ci);
    std::copy(cl.second->pos_fej, cl.second->pos_fej + 3, cpf.begin() + 3 * ci);
    coff[(size_t)ci++] = cl.second->id;
  }
  for (int k = 0; k < K; k++) {
    const Camera &cam = state._cameras[(size_t)k];
    std::copy(cam.R_ItoC, cam.R_ItoC + 9, kR.begin() + 9 * k);
    std::copy(cam.p_IinC, cam.p_IinC + 3, kp.begin() + 3 * k);
    std::copy(cam.intrinsics, cam.intrinsics + 8, kin.begin() + 8 * k);
    kmodel[(size_t)k] = cam.model;
    kext[(size_t)k] = state._options.do_calib_camera_pose ? cam.calib_id : -1;
  }
  ovb_frame frame{C, K, cR.data(), cp.data(), cRf.data(), cpf.data(), coff.data(), kR.data(), kp.data(), kin.data(), kmodel.data(), kext.data(), kintr.data()};
  // the landmarks change_anchors would move, in its visiting order; a lost landmark is gone before it runs
  std::vector<Landmark *> moved;
  std::vector<int32_t> lm_off, reps, ocam, oclone, ncam, nclone;
  std::vector<double> val, val_fej;
  if (full) {
    const double marg_timestep = state._clones_IMU.begin()->first;
    for (auto &f : state._features_SLAM) {
      Landmark &lm = *f.second;
      if (lm._feat_representation == OVB_REP_GLOBAL_3D || lm._feat_representation == OVB_REP_GLOBAL_FULL_INVERSE_DEPTH ||
          lm._anchor_clone_timestamp != marg_timestep || std::find(lost.begin(), lost.end(), f.first) != lost.end())
        continue;
      moved.push_back(&lm);
      lm_off.push_back(lm.id);
      reps.push_back(lm._feat_representation);
      ocam.push_back(lm._anchor_cam_id);
      oclone.push_back(0);
      ncam.push_back(lm._anchor_cam_id);
      nclone.push_back(C - 1);
      val.insert(val.end(), lm.xyz, lm.xyz + 3);
      val_fej.insert(val_fej.end(), lm.xyz_fej, lm.xyz_fej + 3);
    }
    marg.push_back(Var(state._clones_IMU.begin()->second->id, state._clones_IMU.begin()->second->size()));
  }
  const int n = (int)moved.size();
  std::vector<double> nv((size_t)3 * n), nvf((size_t)3 * n);
  ovb_anchor_changes an{n, lm_off.data(), reps.data(), val.data(), val_fej.data(), ocam.data(), oclone.data(), ncam.data(), nclone.data(), nv.data(), nvf.data()};
  ovb_opts o;
  ovb_opts_default(&o);
  o.do_fej = state._options.do_fej;
  o.do_calib_camera_pose = state._options.do_calib_camera_pose;
  std::vector<int32_t> moff, msz;
  for (const Var &v : marg) {
    moff.push_back(v.first);
    msz.push_back(v.second);
  }
  if (marg.empty())
    return;
  state.check(ovb_marginalize_window(state.ctx(), &frame, &o, moff.data(), msz.data(), (int)marg.size(), n ? &an : nullptr), "marginalize_window");
  const double new_timestep = state._clones_IMU.rbegin()->first;
  for (int l = 0; l < n; l++) {
    std::copy(nv.begin() + 3 * l, nv.begin() + 3 * l + 3, moved[(size_t)l]->xyz);
    std::copy(nvf.begin() + 3 * l, nvf.begin() + 3 * l + 3, moved[(size_t)l]->xyz_fej);
    moved[(size_t)l]->_anchor_clone_timestamp = new_timestep;
  }
  for (size_t id : lost)
    state._features_SLAM.erase(id);
  if (full)
    state._clones_IMU.erase(state._clones_IMU.begin());
  // every variable moves up by the sizes of the removed blocks in front of it (StateHelper.cpp:318-326, once per block)
  auto shift = [&](int &id) {
    int d = 0;
    for (const Var &v : marg)
      if (id > v.first)
        d += v.second;
    id -= d;
  };
  for (auto &c : state._clones_IMU)
    shift(c.second->id);
  for (auto &cam : state._cameras) {
    shift(cam.calib_id);
    shift(cam.intrinsics_id);
  }
  for (auto &lm : state._features_SLAM)
    shift(lm.second->id);
}

} // namespace ovb200
#endif // OVB200_HOST_HPP
