// ovb200_sim.hpp — host-side rpng_sim input pipeline (SURVEY.md §8f row 2): the visual-inertial simulator that produces
// the IMU and camera measurements the estimator consumes. Header-only C++17, no Eigen/OpenCV. Restates
//   ov_core::BsplineSE3                ov_core/src/sim/BsplineSE3.cpp:26-358
//   ov_msckf::Simulator                ov_msckf/src/sim/Simulator.cpp:35-207, :267-547
//   ov_core::CamRadtan::distort_f      ov_core/src/cam/CamRadtan.h:127-146 (float/double mix kept, see SURVEY.md App. A.2)
//   cv::undistortPoints (pinhole + radtan, 5 fixed-point iterations, the default TermCriteria(COUNT, 5, 0.01)) as used by
//   CamRadtan::undistort_f (cam/CamRadtan.h:95-114). OpenCV is an unvendored, unpinned dependency of the reference; the
//   restatement is checked against cv2.undistortPoints of this image (tests/test_sim_cpu.py).
//   ov_core::CamEqui::distort_f        ov_core/src/cam/CamEqui.h:136-158 (float r and sqrt, double atan and std::pow, float
//   pixel); pinned bit for bit to the oracle's equidistant distort_d (oracle/ovo_core.hpp) over the fisheye image
//   cv::fisheye::undistortPoints (Newton on theta, the default TermCriteria(COUNT + EPS, 10, 1e-8)) as used by
//   CamEqui::undistort_f (cam/CamEqui.h:104-124); checked bit for bit against cv2.fisheye.undistortPoints (OpenCV 4.13)
//   over the whole 512 x 512 image and past the pi/2 clamp, and the simulated fisheye pixels against
//   cv2.fisheye.projectPoints (tests/test_sim_equi_cpu.py).
// Random streams: std::mt19937 + std::normal_distribution / std::uniform_real_distribution of libstdc++, seeded and
// drawn in the reference's order (Simulator.cpp:129-140, :361-385, :438-442, :518-531), and the feature map is a
// std::unordered_map<size_t, ...> iterated like the reference iterates it (Simulator.cpp:468), so a GCC build of the
// reference and this code walk the same sequences.
#ifndef OVB200_SIM_HPP
#define OVB200_SIM_HPP

#include "ovb200.h"
#include "ovb200_math.hpp"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <map>
#include <random>
#include <sstream>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace ovb200 {

// ---------------------------------------------------------------------------------------------------------------------
// one camera of the rig (cam/CamBase.h:65-82): the model (OVB_CAM_RADTAN or OVB_CAM_EQUI), value = [fx fy cx cy d0 d1 d2 d3]
// (radtan: k1 k2 p1 p2; equidistant: k1 k2 k3 k4) and the image size
struct SimCamera {
  int model = OVB_CAM_RADTAN;
  int w = 752, h = 480;
  double d[8] = {0, 0, 0, 0, 0, 0, 0, 0};

  void distort_f(float xn, float yn, float &u, float &v) const {
    if (model == OVB_CAM_EQUI)
      equi_distort_f(xn, yn, u, v);
    else
      radtan_distort_f(xn, yn, u, v);
  }
  void undistort_f(float u, float v, float &xn, float &yn) const {
    if (model == OVB_CAM_EQUI)
      equi_undistort_f(u, v, xn, yn);
    else
      radtan_undistort_f(u, v, xn, yn);
  }

  // CamRadtan::distort_f (cam/CamRadtan.h:127-146): Vector2f in, double arithmetic from those floats, float pixel out.
  // r comes from a FLOAT sum of float products and std::sqrt(float); 2*x*x is a float product.
  void radtan_distort_f(float xn, float yn, float &u, float &v) const {
    const double x = (double)xn, y = (double)yn;
    const float r2f = xn * xn + yn * yn;
    const double r = (double)std::sqrt(r2f);
    const double r_2 = r * r, r_4 = r_2 * r_2;
    const float two_xx = (2 * xn) * xn, two_yy = (2 * yn) * yn;
    const double x1 = x * (1 + d[4] * r_2 + d[5] * r_4) + 2 * d[6] * x * y + d[7] * (r_2 + (double)two_xx);
    const double y1 = y * (1 + d[4] * r_2 + d[5] * r_4) + d[6] * (r_2 + (double)two_yy) + 2 * d[7] * x * y;
    u = (float)(d[0] * x1 + d[2]);
    v = (float)(d[1] * y1 + d[3]);
  }

  // CamRadtan::undistort_f (cam/CamRadtan.h:95-114) = cv::undistortPoints(src, dst, K, D) with no R/P: float pixel in,
  // double fixed-point iteration, float normalized coordinates out. OpenCV (imgproc undistortPoints, pinhole model with
  // k = [k1 k2 p1 p2 0 ...]): x0 = (u-cx)/fx, y0 = (v-cy)/fy; 5 iterations of
  //   icdist = 1 / (1 + (k2 r2 + k1) r2),  dx = 2 p1 x y + p2 (r2 + 2 x^2),  dy = p1 (r2 + 2 y^2) + 2 p2 x y,
  //   x = (x0 - dx) icdist,  y = (y0 - dy) icdist           (icdist < 0 is replaced by 1).
  void radtan_undistort_f(float u, float v, float &xn, float &yn) const {
    const double ifx = 1. / d[0], ify = 1. / d[1];
    double x = ((double)u - d[2]) * ifx, y = ((double)v - d[3]) * ify;
    const double x0 = x, y0 = y;
    for (int j = 0; j < 5; j++) {
      const double r2 = x * x + y * y;
      double icdist = 1. / (1 + ((0.0 * r2 + d[5]) * r2 + d[4]) * r2);
      if (icdist < 0)
        icdist = 1;
      const double deltaX = 2 * d[6] * x * y + d[7] * (r2 + 2 * x * x);
      const double deltaY = d[6] * (r2 + 2 * y * y) + 2 * d[7] * x * y;
      x = (x0 - deltaX) * icdist;
      y = (y0 - deltaY) * icdist;
    }
    xn = (float)x;
    yn = (float)y;
  }

  // CamEqui::distort_f (cam/CamEqui.h:136-158): r from a FLOAT sum of float products and std::sqrt(float), then
  // theta = atan(r) and the odd polynomial in double (std::pow, as written there), float pixel out
  void equi_distort_f(float xn, float yn, float &u, float &v) const {
    const double r = (double)std::sqrt(xn * xn + yn * yn);
    const double theta = std::atan(r);
    const double theta_d = theta + d[4] * std::pow(theta, 3) + d[5] * std::pow(theta, 5) + d[6] * std::pow(theta, 7) + d[7] * std::pow(theta, 9);
    const double inv_r = (r > 1e-8) ? 1.0 / r : 1.0;
    const double cdist = (r > 1e-8) ? theta_d * inv_r : 1.0;
    const double x1 = (double)xn * cdist, y1 = (double)yn * cdist;
    u = (float)(d[0] * x1 + d[2]);
    v = (float)(d[1] * y1 + d[3]);
  }

  // CamEqui::undistort_f (cam/CamEqui.h:104-124) = cv::fisheye::undistortPoints(src, dst, K, D) with no R/P and the
  // default TermCriteria(COUNT + EPS, 10, 1e-8): float pixel in, double Newton iteration on theta, float out. OpenCV
  // (calib3d fisheye.cpp): pw = (uv - c) / f, theta_d = |pw| clamped to [-pi/2, pi/2]; unless theta_d <= eps (then
  // scale = 0), at most 10 steps theta -= (theta (1 + k1 t2 + k2 t4 + k3 t6 + k4 t8) - theta_d) / (1 + 3 k1 t2 + 5 k2 t4 +
  // 7 k3 t6 + 9 k4 t8), stopping after the first step below eps, and scale = tan(theta) / theta_d. A point that does not
  // converge or whose theta changes sign comes out as (-1e6, -1e6); the others as R pu / (R pu)_z with R = I.
  void equi_undistort_f(float u, float v, float &xn, float &yn) const {
    const double eps = 1e-8;
    const double pw0 = ((double)u - d[2]) / d[0], pw1 = ((double)v - d[3]) / d[1];
    double theta_d = std::sqrt(pw0 * pw0 + pw1 * pw1);
    theta_d = std::min(std::max(-M_PI / 2., theta_d), M_PI / 2.);
    bool converged = false;
    double theta = theta_d, scale = 0.0;
    if (std::fabs(theta_d) > eps) {
      for (int j = 0; j < 10; j++) {
        const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2, theta8 = theta6 * theta2;
        const double k0_theta2 = d[4] * theta2, k1_theta4 = d[5] * theta4, k2_theta6 = d[6] * theta6, k3_theta8 = d[7] * theta8;
        const double theta_fix = (theta * (1 + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d) /
                                 (1 + 3 * k0_theta2 + 5 * k1_theta4 + 7 * k2_theta6 + 9 * k3_theta8);
        theta = theta - theta_fix;
        if (std::fabs(theta_fix) < eps) {
          converged = true;
          break;
        }
      }
      scale = std::tan(theta) / theta_d;
    } else {
      converged = true;
    }
    const bool theta_flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
    if (converged && !theta_flipped) {
      const double pu[3] = {pw0 * scale, pw1 * scale, 1.0};
      double pr[3]; // Matx33d::eye() * Vec3d: every row summed from 0 in column order
      for (int i = 0; i < 3; i++) {
        double s = 0;
        for (int k = 0; k < 3; k++)
          s += (i == k ? 1.0 : 0.0) * pu[k];
        pr[i] = s;
      }
      xn = (float)(pr[0] / pr[2]);
      yn = (float)(pr[1] / pr[2]);
    } else {
      xn = yn = (float)-1000000.0;
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// ov_core::BsplineSE3 (sim/BsplineSE3.cpp). Poses are T_IinG (R_ItoG, p_IinG) 4x4.
class BsplineSE3 {
public:
  // traj_points: rows [t x y z qx qy qz qw] (JPL quaternion q_GtoI like the reference's text files)
  void feed_trajectory(const std::vector<std::array<double, 8>> &traj_points) { // BsplineSE3.cpp:26-89
    double sumdt = 0;
    for (size_t i = 0; i + 1 < traj_points.size(); i++)
      sumdt += traj_points[i + 1][0] - traj_points[i][0];
    dt = sumdt / (double)(traj_points.size() - 1);
    dt = (dt < 0.05) ? 0.05 : dt;
    std::map<double, Mat4> trajectory_points;
    for (size_t i = 0; i + 1 < traj_points.size(); i++) {
      const auto &p = traj_points[i];
      const Mat3 R_ItoG = transpose(quat_2_Rot({p[4], p[5], p[6], p[7]}));
      trajectory_points.insert({p[0], make_T(R_ItoG, {p[1], p[2], p[3]})});
    }
    double timestamp_min = INFINITY, timestamp_max = -INFINITY;
    for (const auto &pose : trajectory_points) {
      if (pose.first <= timestamp_min)
        timestamp_min = pose.first;
      if (pose.first >= timestamp_max)
        timestamp_max = pose.first;
    }
    double timestamp_curr = timestamp_min;
    while (true) {
      double t0, t1;
      Mat4 pose0, pose1;
      if (!find_bounding_poses(timestamp_curr, trajectory_points, t0, pose0, t1, pose1))
        break;
      const double lambda = (timestamp_curr - t0) / (t1 - t0);
      const Mat4 pose_interp = exp_se3(lambda * log_se3(pose1 * Inv_se3(pose0))) * pose0;
      control_points.insert({timestamp_curr, pose_interp});
      timestamp_curr += dt;
    }
    timestamp_start = timestamp_min + 2 * dt;
  }

  bool get_pose(double timestamp, Mat3 &R_GtoI, Vec3 &p_IinG) const { // :91-120
    double t0, t1, t2, t3;
    Mat4 pose0, pose1, pose2, pose3;
    if (!find_bounding_control_points(timestamp, t0, pose0, t1, pose1, t2, pose2, t3, pose3)) {
      R_GtoI = eye3();
      p_IinG = {0, 0, 0};
      return false;
    }
    const double DT = (t2 - t1), u = (timestamp - t1) / DT;
    const double b0 = 1.0 / 6.0 * (5 + 3 * u - 3 * u * u + u * u * u);
    const double b1 = 1.0 / 6.0 * (1 + 3 * u + 3 * u * u - 2 * u * u * u);
    const double b2 = 1.0 / 6.0 * (u * u * u);
    const Mat4 A0 = exp_se3(b0 * log_se3(Inv_se3(pose0) * pose1));
    const Mat4 A1 = exp_se3(b1 * log_se3(Inv_se3(pose1) * pose2));
    const Mat4 A2 = exp_se3(b2 * log_se3(Inv_se3(pose2) * pose3));
    const Mat4 pose_interp = pose0 * A0 * A1 * A2;
    R_GtoI = transpose(rot_of(pose_interp));
    p_IinG = pos_of(pose_interp);
    return true;
  }

  bool get_velocity(double timestamp, Mat3 &R_GtoI, Vec3 &p_IinG, Vec3 &w_IinI, Vec3 &v_IinG) const { // :122-167
    Vec3 alpha, a;
    return derivatives(timestamp, 1, R_GtoI, p_IinG, w_IinI, v_IinG, alpha, a);
  }
  bool get_acceleration(double timestamp, Mat3 &R_GtoI, Vec3 &p_IinG, Vec3 &w_IinI, Vec3 &v_IinG, Vec3 &alpha_IinI, Vec3 &a_IinG) const { // :169-233
    return derivatives(timestamp, 2, R_GtoI, p_IinG, w_IinI, v_IinG, alpha_IinI, a_IinG);
  }
  double get_start_time() const { return timestamp_start; }

private:
  double dt = 0.05;
  double timestamp_start = 0;
  std::map<double, Mat4> control_points;

  bool derivatives(double timestamp, int order, Mat3 &R_GtoI, Vec3 &p_IinG, Vec3 &w_IinI, Vec3 &v_IinG, Vec3 &alpha_IinI, Vec3 &a_IinG) const {
    double t0, t1, t2, t3;
    Mat4 pose0, pose1, pose2, pose3;
    w_IinI = v_IinG = alpha_IinI = a_IinG = {0, 0, 0};
    if (!find_bounding_control_points(timestamp, t0, pose0, t1, pose1, t2, pose2, t3, pose3))
      return false;
    const double DT = (t2 - t1), u = (timestamp - t1) / DT;
    const double b0 = 1.0 / 6.0 * (5 + 3 * u - 3 * u * u + u * u * u);
    const double b1 = 1.0 / 6.0 * (1 + 3 * u + 3 * u * u - 2 * u * u * u);
    const double b2 = 1.0 / 6.0 * (u * u * u);
    const double b0dot = 1.0 / (6.0 * DT) * (3 - 6 * u + 3 * u * u);
    const double b1dot = 1.0 / (6.0 * DT) * (3 + 6 * u - 6 * u * u);
    const double b2dot = 1.0 / (6.0 * DT) * (3 * u * u);
    const double b0dotdot = 1.0 / (6.0 * DT * DT) * (-6 + 6 * u);
    const double b1dotdot = 1.0 / (6.0 * DT * DT) * (6 - 12 * u);
    const double b2dotdot = 1.0 / (6.0 * DT * DT) * (6 * u);
    const Vec6 omega_10 = log_se3(Inv_se3(pose0) * pose1), omega_21 = log_se3(Inv_se3(pose1) * pose2), omega_32 = log_se3(Inv_se3(pose2) * pose3);
    const Mat4 h10 = hat_se3(omega_10), h21 = hat_se3(omega_21), h32 = hat_se3(omega_32);
    const Mat4 A0 = exp_se3(b0 * omega_10), A1 = exp_se3(b1 * omega_21), A2 = exp_se3(b2 * omega_32);
    const Mat4 A0dot = b0dot * (h10 * A0), A1dot = b1dot * (h21 * A1), A2dot = b2dot * (h32 * A2);
    const Mat4 pose_interp = pose0 * A0 * A1 * A2;
    R_GtoI = transpose(rot_of(pose_interp));
    p_IinG = pos_of(pose_interp);
    const Mat4 vel_interp = pose0 * (A0dot * A1 * A2 + A0 * A1dot * A2 + A0 * A1 * A2dot);
    w_IinI = vee(transpose(rot_of(pose_interp)) * rot_of(vel_interp));
    v_IinG = pos_of(vel_interp);
    if (order < 2)
      return true;
    const Mat4 A0dotdot = b0dot * (h10 * A0dot) + b0dotdot * (h10 * A0);
    const Mat4 A1dotdot = b1dot * (h21 * A1dot) + b1dotdot * (h21 * A1);
    const Mat4 A2dotdot = b2dot * (h32 * A2dot) + b2dotdot * (h32 * A2);
    const Mat4 acc_interp = pose0 * (A0dotdot * A1 * A2 + A0 * A1dotdot * A2 + A0 * A1 * A2dotdot + 2.0 * (A0dot * A1dot * A2) +
                                     2.0 * (A0 * A1dot * A2dot) + 2.0 * (A0dot * A1 * A2dot));
    const Mat3 omegaskew = transpose(rot_of(pose_interp)) * rot_of(vel_interp);
    alpha_IinI = vee(transpose(rot_of(pose_interp)) * (rot_of(acc_interp) - rot_of(vel_interp) * omegaskew));
    a_IinG = pos_of(acc_interp);
    return true;
  }

  static bool find_bounding_poses(double timestamp, const std::map<double, Mat4> &poses, double &t0, Mat4 &pose0, double &t1, Mat4 &pose1) { // :235-281
    t0 = t1 = -1;
    pose0 = pose1 = eye4();
    bool found_older = false, found_newer = false;
    auto lower_bound = poses.lower_bound(timestamp);
    auto upper_bound = poses.upper_bound(timestamp);
    if (lower_bound != poses.end()) {
      if (lower_bound->first == timestamp) {
        found_older = true;
      } else if (lower_bound != poses.begin()) {
        --lower_bound;
        found_older = true;
      }
    }
    if (upper_bound != poses.end())
      found_newer = true;
    if (found_older) {
      t0 = lower_bound->first;
      pose0 = lower_bound->second;
    }
    if (found_newer) {
      t1 = upper_bound->first;
      pose1 = upper_bound->second;
    }
    return found_older && found_newer;
  }
  bool find_bounding_control_points(double timestamp, double &t0, Mat4 &pose0, double &t1, Mat4 &pose1, double &t2, Mat4 &pose2, double &t3,
                                    Mat4 &pose3) const { // :283-330
    t0 = t1 = t2 = t3 = -1;
    pose0 = pose1 = pose2 = pose3 = eye4();
    if (!find_bounding_poses(timestamp, control_points, t1, pose1, t2, pose2))
      return false;
    auto iter_t1 = control_points.find(t1);
    auto iter_t2 = control_points.find(t2);
    if (iter_t1 == control_points.begin())
      return false;
    auto iter_t0 = --iter_t1;
    auto iter_t3 = ++iter_t2;
    if (iter_t3 == control_points.end())
      return false;
    t0 = iter_t0->first;
    pose0 = iter_t0->second;
    t3 = iter_t3->first;
    pose3 = iter_t3->second;
    return true;
  }
};

// ---------------------------------------------------------------------------------------------------------------------
// the slice of VioManagerOptions the simulator reads (core/VioManagerOptions.h) with the rpng_sim YAML defaults
// (config/rpng_sim/estimator_config.yaml, kalibr_imucam_chain.yaml, kalibr_imu_chain.yaml)
struct SimParams {
  int num_cameras = 2;
  bool use_stereo = true;
  int num_pts = 250;
  double gravity_mag = 9.81;
  double calib_camimu_dt = 0.0;
  // IMU noise densities (kalibr_imu_chain.yaml:9-12)
  double sigma_w = 1.6968e-04, sigma_wb = 1.9393e-05, sigma_a = 2.0000e-3, sigma_ab = 3.0000e-3;
  double sigma_pix = 1.0; // up_msckf_sigma_px
  // IMU intrinsics (identity / zero in rpng_sim): Dw, Da packed like State::Dm (KALIBR), Tg column-wise
  double vec_dw[6] = {1, 0, 0, 1, 0, 1}, vec_da[6] = {1, 0, 0, 1, 0, 1}, vec_tg[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  Vec4 q_GYROtoIMU{0, 0, 0, 1}, q_ACCtoIMU{0, 0, 0, 1};
  int seed_state_init = 0, seed_preturb = 0, seed_measurements = 0;
  bool sim_do_perturbation = false; // hand the estimator a perturbed copy of the calibration (Simulator::perturb_parameters)
  double sim_distance_threshold = 1.1, sim_freq_cam = 10, sim_freq_imu = 400;
  double sim_min_feature_gen_distance = 5.0, sim_max_feature_gen_distance = 7.0;
  std::vector<SimCamera> camera_intrinsics;                 // per camera
  std::vector<std::pair<Vec4, Vec3>> camera_extrinsics;     // per camera: q_ItoC, p_IinC
};

// kalibr_imucam_chain.yaml of rpng_sim: T_imu_cam (= T_CtoI), intrinsics, distortion of cam0..cam3. `models` (empty = all
// radtan) gives each camera's model; an equidistant camera takes the TUM-VI cam0 intrinsics on a 512 x 512 image (the
// fisheye rig of open_vins_b200/sim.py, _INTR_EQUI) and keeps the rpng_sim extrinsics of its slot.
inline void rpng_sim_cameras(int num_cameras, SimParams &p, const std::vector<int> &models = {}) {
  static const double K_EQUI[8] = {190.978, 190.973, 254.93, 256.897, 0.0034, 0.0007, -0.0020, 0.0002};
  static const double T[4][12] = {
      {0.0148655429818, -0.999880929698, 0.00414029679422, -0.0216401454975, 0.999557249008, 0.0149672133247, 0.025715529948, -0.064676986768,
       -0.0257744366974, 0.00375618835797, 0.999660727178, 0.00981073058949},
      {0.0125552670891, -0.999755099723, 0.0182237714554, -0.0198435579556, 0.999598781151, 0.0130119051815, 0.0251588363115, 0.0453689425024,
       -0.0253898008918, 0.0179005838253, 0.999517347078, 0.00786212447038},
      {0.0148655429818, -0.999880929698, 0.00414029679422, -0.0216401454975, 0.999557249008, 0.0149672133247, 0.025715529948, 0.124676986768,
       -0.0257744366974, 0.00375618835797, 0.999660727178, 0.00981073058949},
      {0.0125552670891, -0.999755099723, 0.0182237714554, -0.0198435579556, 0.999598781151, 0.0130119051815, 0.0251588363115, 0.2253689425024,
       -0.0253898008918, 0.0179005838253, 0.999517347078, 0.00786212447038}};
  static const double K[4][8] = {{458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, 0.00019359, 1.76187114e-05},
                                 {457.587, 456.134, 379.999, 255.238, -0.28368365, 0.07451284, -0.00010473, -3.55590700e-05},
                                 {458.654, 457.296, 367.215, 248.375, -0.28340811, 0.07395907, 0.00019359, 1.76187114e-05},
                                 {457.587, 456.134, 379.999, 255.238, -0.28368365, 0.07451284, -0.00010473, -3.55590700e-05}};
  p.num_cameras = num_cameras;
  p.camera_intrinsics.clear();
  p.camera_extrinsics.clear();
  for (int i = 0; i < num_cameras; i++) {
    SimCamera c;
    if (!models.empty() && models[(size_t)i] == OVB_CAM_EQUI) {
      c.model = OVB_CAM_EQUI;
      c.w = c.h = 512;
      for (int k = 0; k < 8; k++)
        c.d[k] = K_EQUI[k];
    } else {
      for (int k = 0; k < 8; k++)
        c.d[k] = K[i][k];
    }
    p.camera_intrinsics.push_back(c);
    // VioManagerOptions.h:263-269: q_ItoC = rot_2_quat(R_CtoI'), p_IinC = -R_CtoI' p_CinI
    const Mat3 R_CtoI{T[i][0], T[i][1], T[i][2], T[i][4], T[i][5], T[i][6], T[i][8], T[i][9], T[i][10]};
    const Vec3 p_CinI{T[i][3], T[i][7], T[i][11]};
    p.camera_extrinsics.push_back({rot_2_quat(transpose(R_CtoI)), -(transpose(R_CtoI) * p_CinI)});
  }
}

// DatasetReader::load_simulated_trajectory (utils/dataset_reader.h): text rows "t x y z qx qy qz qw", '#' comments
inline std::vector<std::array<double, 8>> load_simulated_trajectory(const std::string &path) {
  std::vector<std::array<double, 8>> out;
  std::ifstream f(path);
  if (!f.is_open())
    return out;
  std::string line;
  while (std::getline(f, line)) {
    if (line.empty() || line[0] == '#')
      continue;
    for (auto &c : line)
      if (c == ',')
        c = ' ';
    std::istringstream ss(line);
    std::array<double, 8> r;
    int k = 0;
    while (k < 8 && (ss >> r[(size_t)k]))
      k++;
    if (k == 8)
      out.push_back(r);
  }
  return out;
}
// the same rows as raw little-endian doubles (tests/golden/traj_*.bin, written by tools/make_traj_fixture.py)
inline std::vector<std::array<double, 8>> load_trajectory_bin(const std::string &path) {
  std::vector<std::array<double, 8>> out;
  FILE *f = std::fopen(path.c_str(), "rb");
  if (!f)
    return out;
  std::array<double, 8> r;
  while (std::fread(r.data(), sizeof(double), 8, f) == 8)
    out.push_back(r);
  std::fclose(f);
  return out;
}

struct SimFeat {
  size_t id;
  float u, v;
};

// ov_msckf::Simulator (sim/Simulator.cpp)
class Simulator {
public:
  SimParams params; // the true parameters: every measurement is generated from them
  std::unordered_map<size_t, Vec3> featmap;
  // with sim_do_perturbation, the draws of perturb_parameters in draw order (what was added to the true value, or the
  // rotation vector w of R <- exp_so3(w) R); empty without
  std::vector<double> perturbation;

  Simulator(const SimParams &params_, const std::vector<std::array<double, 8>> &traj_data) : params(params_), estimator_params(params_) { // Simulator.cpp:35-207
    spline.feed_trajectory(traj_data);
    timestamp = timestamp_last_imu = timestamp_last_cam = spline.get_start_time();
    Mat3 R_GtoI_init;
    Vec3 p_IinG_init;
    // the reference exits the process here; throwing lets a runner that holds several simulations report the failing one
    if (!spline.get_pose(timestamp, R_GtoI_init, p_IinG_init))
      throw std::runtime_error("[SIM]: unable to find the first pose in the spline");
    // find the timestamp at which we have moved enough (:76-109)
    double distance = 0.0;
    while (true) {
      Mat3 R_GtoI;
      Vec3 p_IinG;
      if (!spline.get_pose(timestamp, R_GtoI, p_IinG))
        throw std::runtime_error("[SIM]: unable to find jolt in the groundtruth data to initialize at");
      distance += norm(p_IinG - p_IinG_init);
      p_IinG_init = p_IinG;
      if (distance > params.sim_distance_threshold)
        break;
      timestamp += 1.0 / params.sim_freq_cam;
      timestamp_last_imu += 1.0 / params.sim_freq_cam;
      timestamp_last_cam += 1.0 / params.sim_freq_cam;
    }
    // bias history (:113-121)
    hist_true_bias_time = {timestamp_last_imu - 1.0 / params.sim_freq_imu, timestamp_last_imu, timestamp_last_imu + 1.0 / params.sim_freq_imu};
    hist_true_bias_accel = {true_bias_accel, true_bias_accel, true_bias_accel};
    hist_true_bias_gyro = {true_bias_gyro, true_bias_gyro, true_bias_gyro};
    is_running = true;
    // generators (:129-140)
    gen_state_init = std::mt19937((unsigned)params.seed_state_init);
    gen_state_init.seed((unsigned)params.seed_state_init);
    gen_state_perturb = std::mt19937((unsigned)params.seed_preturb);
    gen_state_perturb.seed((unsigned)params.seed_preturb);
    gen_meas_imu = std::mt19937((unsigned)params.seed_measurements);
    gen_meas_imu.seed((unsigned)params.seed_measurements);
    for (int i = 0; i < params.num_cameras; i++) {
      gen_meas_cams.push_back(std::mt19937((unsigned)params.seed_measurements));
      gen_meas_cams[(size_t)i].seed((unsigned)params.seed_measurements);
    }
    if (params.sim_do_perturbation) // (:142-160)
      perturb_parameters(estimator_params);
    // feature map: walk the whole trajectory, top up to num_pts visible points per camera (:164-201)
    const double dt = 0.25;
    for (int i = 0; i < params.num_cameras; i++) {
      double time_synth = spline.get_start_time();
      while (true) {
        Mat3 R_GtoI;
        Vec3 p_IinG;
        if (!spline.get_pose(time_synth, R_GtoI, p_IinG))
          break;
        std::vector<SimFeat> uvs = project_pointcloud(R_GtoI, p_IinG, i);
        if ((int)uvs.size() < params.num_pts)
          generate_points(R_GtoI, p_IinG, i, params.num_pts - (int)uvs.size());
        time_synth += dt;
      }
    }
  }

  bool ok() const { return is_running; }
  double current_timestamp() const { return timestamp; }
  // Simulator::get_true_parameters: what the measurements are generated from
  const SimParams &get_true_parameters() const { return params; }
  // what the estimator is built from: the true parameters, or their perturbed copy with sim_do_perturbation
  const SimParams &get_estimator_parameters() const { return estimator_params; }

  // Simulator::get_state (:267-309): [t q_GtoI(4) p(3) v(3) bg(3) ba(3)]
  bool get_state(double desired_time, std::array<double, 17> &imustate) const {
    imustate.fill(0.0);
    imustate[4] = 1;
    Mat3 R_GtoI;
    Vec3 p_IinG, w_IinI, v_IinG;
    const bool success_vel = spline.get_velocity(desired_time, R_GtoI, p_IinG, w_IinI, v_IinG);
    bool success_bias = false;
    size_t id_loc = 0;
    for (size_t i = 0; i + 1 < hist_true_bias_time.size(); i++) {
      if (hist_true_bias_time[i] < desired_time && hist_true_bias_time[i + 1] >= desired_time) {
        id_loc = i;
        success_bias = true;
        break;
      }
    }
    if (!success_vel || !success_bias)
      return false;
    const double lambda = (desired_time - hist_true_bias_time[id_loc]) / (hist_true_bias_time[id_loc + 1] - hist_true_bias_time[id_loc]);
    const Vec3 bg = (1 - lambda) * hist_true_bias_gyro[id_loc] + lambda * hist_true_bias_gyro[id_loc + 1];
    const Vec3 ba = (1 - lambda) * hist_true_bias_accel[id_loc] + lambda * hist_true_bias_accel[id_loc + 1];
    imustate[0] = desired_time;
    const Vec4 q = rot_2_quat(R_GtoI);
    for (int k = 0; k < 4; k++)
      imustate[(size_t)(1 + k)] = q[(size_t)k];
    for (int k = 0; k < 3; k++) {
      imustate[(size_t)(5 + k)] = p_IinG[(size_t)k];
      imustate[(size_t)(8 + k)] = v_IinG[(size_t)k];
      imustate[(size_t)(11 + k)] = bg[(size_t)k];
      imustate[(size_t)(14 + k)] = ba[(size_t)k];
    }
    return true;
  }

  // Simulator::get_next_imu (:311-389)
  bool get_next_imu(double &time_imu, Vec3 &wm, Vec3 &am) {
    if (timestamp_last_cam + 1.0 / params.sim_freq_cam < timestamp_last_imu + 1.0 / params.sim_freq_imu)
      return false;
    timestamp_last_imu += 1.0 / params.sim_freq_imu;
    timestamp = timestamp_last_imu;
    time_imu = timestamp_last_imu;
    Mat3 R_GtoI;
    Vec3 p_IinG, w_IinI, v_IinG, alpha_IinI, a_IinG;
    if (!spline.get_acceleration(timestamp, R_GtoI, p_IinG, w_IinI, v_IinG, alpha_IinI, a_IinG)) {
      is_running = false;
      return false;
    }
    const Vec3 gravity{0.0, 0.0, params.gravity_mag};
    const Vec3 accel_inI = R_GtoI * (a_IinG + gravity);
    const Vec3 omega_inI = w_IinI;
    // IMU intrinsics (:336-347). Dw = Da = I and Tg = 0 in rpng_sim; the general model needs the 3x3 inverses of
    // Dw/Da (colPivHouseholderQr().solve(I) in the reference) — computed by adjugate here.
    const Mat3 Tw = inv3(Dm(params.vec_dw)), Ta = inv3(Dm(params.vec_da)), Tg = Tgm(params.vec_tg);
    const Vec3 omega_inGYRO = Tw * (transpose(quat_2_Rot(params.q_GYROtoIMU)) * omega_inI) + Tg * accel_inI;
    const Vec3 accel_inACC = Ta * (transpose(quat_2_Rot(params.q_ACCtoIMU)) * accel_inI);
    const double dt = 1.0 / params.sim_freq_imu;
    std::normal_distribution<double> w(0, 1);
    if (has_skipped_first_bias) {
      true_bias_gyro[0] += params.sigma_wb * std::sqrt(dt) * w(gen_meas_imu);
      true_bias_gyro[1] += params.sigma_wb * std::sqrt(dt) * w(gen_meas_imu);
      true_bias_gyro[2] += params.sigma_wb * std::sqrt(dt) * w(gen_meas_imu);
      true_bias_accel[0] += params.sigma_ab * std::sqrt(dt) * w(gen_meas_imu);
      true_bias_accel[1] += params.sigma_ab * std::sqrt(dt) * w(gen_meas_imu);
      true_bias_accel[2] += params.sigma_ab * std::sqrt(dt) * w(gen_meas_imu);
      hist_true_bias_time.push_back(timestamp_last_imu);
      hist_true_bias_gyro.push_back(true_bias_gyro);
      hist_true_bias_accel.push_back(true_bias_accel);
    }
    has_skipped_first_bias = true;
    wm[0] = omega_inGYRO[0] + true_bias_gyro[0] + params.sigma_w / std::sqrt(dt) * w(gen_meas_imu);
    wm[1] = omega_inGYRO[1] + true_bias_gyro[1] + params.sigma_w / std::sqrt(dt) * w(gen_meas_imu);
    wm[2] = omega_inGYRO[2] + true_bias_gyro[2] + params.sigma_w / std::sqrt(dt) * w(gen_meas_imu);
    am[0] = accel_inACC[0] + true_bias_accel[0] + params.sigma_a / std::sqrt(dt) * w(gen_meas_imu);
    am[1] = accel_inACC[1] + true_bias_accel[1] + params.sigma_a / std::sqrt(dt) * w(gen_meas_imu);
    am[2] = accel_inACC[2] + true_bias_accel[2] + params.sigma_a / std::sqrt(dt) * w(gen_meas_imu);
    return true;
  }

  // Simulator::get_next_cam (:391-451)
  bool get_next_cam(double &time_cam, std::vector<int> &camids, std::vector<std::vector<SimFeat>> &feats) {
    if (timestamp_last_imu + 1.0 / params.sim_freq_imu < timestamp_last_cam + 1.0 / params.sim_freq_cam)
      return false;
    timestamp_last_cam += 1.0 / params.sim_freq_cam;
    timestamp = timestamp_last_cam;
    time_cam = timestamp_last_cam - params.calib_camimu_dt;
    Mat3 R_GtoI;
    Vec3 p_IinG;
    if (!spline.get_pose(timestamp, R_GtoI, p_IinG)) {
      is_running = false;
      return false;
    }
    for (int i = 0; i < params.num_cameras; i++) {
      std::vector<SimFeat> uvs = project_pointcloud(R_GtoI, p_IinG, i);
      if ((int)uvs.size() > params.num_pts)
        uvs.erase(uvs.begin() + params.num_pts, uvs.end());
      for (size_t f = 0; f < uvs.size() && !params.use_stereo; f++)
        uvs[f].id += (size_t)i * featmap.size();
      std::normal_distribution<double> w(0, 1);
      for (size_t j = 0; j < uvs.size(); j++) {
        // VectorXf(0) += double: the sum is formed in double, then stored as float
        uvs[j].u = (float)((double)uvs[j].u + params.sigma_pix * w(gen_meas_cams[(size_t)i]));
        uvs[j].v = (float)((double)uvs[j].v + params.sigma_pix * w(gen_meas_cams[(size_t)i]));
      }
      feats.push_back(uvs);
      camids.push_back(i);
    }
    return true;
  }

  static Mat3 Dm(const double *v) { return {v[0], 0, 0, v[1], v[3], 0, v[2], v[4], v[5]}; } // State::Dm, KALIBR (state/State.h:91-101)
  static Mat3 Tgm(const double *v) { return {v[0], v[3], v[6], v[1], v[4], v[7], v[2], v[5], v[8]}; } // State::Tg (:110-116)
  static Mat3 inv3(const Mat3 &A) {
    const double det = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
    const double id = 1.0 / det;
    return {(A[4] * A[8] - A[5] * A[7]) * id, (A[2] * A[7] - A[1] * A[8]) * id, (A[1] * A[5] - A[2] * A[4]) * id,
            (A[5] * A[6] - A[3] * A[8]) * id, (A[0] * A[8] - A[2] * A[6]) * id, (A[2] * A[3] - A[0] * A[5]) * id,
            (A[3] * A[7] - A[4] * A[6]) * id, (A[1] * A[6] - A[0] * A[7]) * id, (A[0] * A[4] - A[1] * A[3]) * id};
  }

private:
  SimParams estimator_params;
  BsplineSE3 spline;
  size_t id_map = 0;

  // Simulator::perturb_parameters (:209-265), drawing only from gen_state_perturb so the map and the measurement streams
  // do not depend on it. Each coordinate gets N(0, σ) with σ the prior σ VioManager gives its block in P0 (so the initial
  // error matches P0), in the reference's order: time offset; per camera fx fy cx cy (1 px), the four distortion terms
  // (0.005), the extrinsic rotation (0.005 rad, q_ItoC <- exp_so3(w) R_ItoC), the extrinsic position (0.015 m); then
  // dw[j], da[j] interleaved (0.005, 0.008); then R_GYROtoIMU (0.005 rad, the same way); then tg (0.005).
  void perturb_parameters(SimParams &p) {
    std::normal_distribution<double> w(0, 1);
    auto draw = [&](double sigma) {
      perturbation.push_back(sigma * w(gen_state_perturb));
      return perturbation.back();
    };
    auto rotate = [&](Vec4 &q, double sigma) {
      Vec3 wv;
      for (auto &x : wv)
        x = draw(sigma);
      q = rot_2_quat(exp_so3(wv) * quat_2_Rot(q));
    };
    p.calib_camimu_dt += draw(0.01);
    for (int i = 0; i < p.num_cameras; i++) {
      double *d = p.camera_intrinsics[(size_t)i].d;
      for (int r = 0; r < 4; r++)
        d[r] += draw(1.0);
      for (int r = 4; r < 8; r++)
        d[r] += draw(0.005);
      rotate(p.camera_extrinsics[(size_t)i].first, 0.005);
      for (auto &x : p.camera_extrinsics[(size_t)i].second)
        x += draw(0.015);
    }
    for (int j = 0; j < 6; j++) {
      p.vec_dw[j] += draw(0.005);
      p.vec_da[j] += draw(0.008);
    }
    rotate(p.q_GYROtoIMU, 0.005);
    for (int j = 0; j < 9; j++)
      p.vec_tg[j] += draw(0.005);
  }
  std::mt19937 gen_state_init, gen_state_perturb, gen_meas_imu;
  std::vector<std::mt19937> gen_meas_cams;
  bool is_running = false;
  double timestamp = 0, timestamp_last_imu = 0, timestamp_last_cam = 0;
  Vec3 true_bias_accel{0, 0, 0}, true_bias_gyro{0, 0, 0};
  bool has_skipped_first_bias = false;
  std::vector<double> hist_true_bias_time;
  std::vector<Vec3> hist_true_bias_accel, hist_true_bias_gyro;

  // Simulator::project_pointcloud (:453-499)
  std::vector<SimFeat> project_pointcloud(const Mat3 &R_GtoI, const Vec3 &p_IinG, int camid) const {
    const Mat3 R_ItoC = quat_2_Rot(params.camera_extrinsics[(size_t)camid].first);
    const Vec3 p_IinC = params.camera_extrinsics[(size_t)camid].second;
    const SimCamera &camera = params.camera_intrinsics[(size_t)camid];
    std::vector<SimFeat> uvs;
    for (const auto &feat : featmap) {
      const Vec3 p_FinI = R_GtoI * (feat.second - p_IinG);
      const Vec3 p_FinC = R_ItoC * p_FinI + p_IinC;
      if (p_FinC[2] > params.sim_max_feature_gen_distance || p_FinC[2] < 0.1)
        continue;
      const float xn = (float)(p_FinC[0] / p_FinC[2]), yn = (float)(p_FinC[1] / p_FinC[2]);
      float u, v;
      camera.distort_f(xn, yn, u, v);
      if (u < 0 || u > camera.w || v < 0 || v > camera.h)
        continue;
      uvs.push_back({feat.first, u, v});
    }
    return uvs;
  }

  // Simulator::generate_points (:501-547)
  void generate_points(const Mat3 &R_GtoI, const Vec3 &p_IinG, int camid, int numpts) {
    const Mat3 R_ItoC = quat_2_Rot(params.camera_extrinsics[(size_t)camid].first);
    const Vec3 p_IinC = params.camera_extrinsics[(size_t)camid].second;
    const SimCamera &camera = params.camera_intrinsics[(size_t)camid];
    for (int i = 0; i < numpts; i++) {
      std::uniform_real_distribution<double> gen_u(0, camera.w);
      std::uniform_real_distribution<double> gen_v(0, camera.h);
      const double u_dist = gen_u(gen_state_init);
      const double v_dist = gen_v(gen_state_init);
      float xn, yn;
      camera.undistort_f((float)u_dist, (float)v_dist, xn, yn);
      std::uniform_real_distribution<double> gen_depth(params.sim_min_feature_gen_distance, params.sim_max_feature_gen_distance);
      const double depth = gen_depth(gen_state_init);
      const Vec3 p_FinC = depth * Vec3{(double)xn, (double)yn, 1.0};
      const Vec3 p_FinI = transpose(R_ItoC) * (p_FinC - p_IinC);
      const Vec3 p_FinG = transpose(R_GtoI) * p_FinI + p_IinG;
      featmap.insert({id_map, p_FinG});
      id_map++;
    }
  }
};

} // namespace ovb200
#endif
