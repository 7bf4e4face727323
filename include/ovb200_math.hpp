// ovb200_math.hpp — small fixed-size linear algebra and JPL-quaternion / SO(3) / SE(3) helpers for the host layer.
// Restates ov_core/src/utils/quat_ops.h (formulas and branch thresholds kept: rot_2_quat :88-133, skew_x :135-139,
// quat_2_Rot :152-157, quat_multiply :180-194, exp_so3 :231-262, log_so3 :273-315, exp_se3 :343-380, log_se3 :402-426,
// hat_se3 :445-450, Inv_se3 :457-462, Omega :482-489, quatnorm :496-501, Jl_so3 :515-527, Jr_so3 :537) without Eigen.
// Matrices are row-major std::array; quaternions are JPL [x y z w]; R = quat_2_Rot(q) rotates global -> local.
// The mean update of JPLQuat::update (quatnorm, quat_multiply, quat_2_Rot and what they call) is also device code: the engine
// moves its copy of the window with it between the landmarks of ovb_slam_delayed_init_batch, in a unit built without FMA
// contraction, so both sides round every product and sum on its own and agree bit for bit.
#ifndef OVB200_MATH_HPP
#define OVB200_MATH_HPP

#include <array>
#include <cmath>

#ifdef __CUDACC__
#define OVB_MATH_HD __host__ __device__
#else
#define OVB_MATH_HD
#endif

namespace ovb200 {

using Vec3 = std::array<double, 3>;
using Vec4 = std::array<double, 4>;
using Vec6 = std::array<double, 6>;
using Mat3 = std::array<double, 9>;  // row-major
using Mat4 = std::array<double, 16>; // row-major

OVB_MATH_HD inline Mat3 eye3() { return {1, 0, 0, 0, 1, 0, 0, 0, 1}; }
inline Mat3 zero3() { return {0, 0, 0, 0, 0, 0, 0, 0, 0}; }
inline Mat4 eye4() { return {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; }
inline Vec3 operator+(const Vec3 &a, const Vec3 &b) { return {a[0] + b[0], a[1] + b[1], a[2] + b[2]}; }
inline Vec3 operator-(const Vec3 &a, const Vec3 &b) { return {a[0] - b[0], a[1] - b[1], a[2] - b[2]}; }
inline Vec3 operator-(const Vec3 &a) { return {-a[0], -a[1], -a[2]}; }
inline Vec3 operator*(double s, const Vec3 &a) { return {s * a[0], s * a[1], s * a[2]}; }
inline Vec3 operator*(const Vec3 &a, double s) { return {s * a[0], s * a[1], s * a[2]}; }
inline Vec3 &operator+=(Vec3 &a, const Vec3 &b) {
  a[0] += b[0], a[1] += b[1], a[2] += b[2];
  return a;
}
inline double dot(const Vec3 &a, const Vec3 &b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
inline double norm(const Vec3 &a) { return std::sqrt(dot(a, a)); }
inline Mat3 operator*(const Mat3 &A, const Mat3 &B) {
  Mat3 C;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
  return C;
}
inline Vec3 operator*(const Mat3 &A, const Vec3 &v) {
  return {A[0] * v[0] + A[1] * v[1] + A[2] * v[2], A[3] * v[0] + A[4] * v[1] + A[5] * v[2], A[6] * v[0] + A[7] * v[1] + A[8] * v[2]};
}
OVB_MATH_HD inline Mat3 operator*(double s, const Mat3 &A) {
  Mat3 C;
  for (int i = 0; i < 9; i++)
    C[i] = s * A[i];
  return C;
}
OVB_MATH_HD inline Mat3 operator+(const Mat3 &A, const Mat3 &B) {
  Mat3 C;
  for (int i = 0; i < 9; i++)
    C[i] = A[i] + B[i];
  return C;
}
OVB_MATH_HD inline Mat3 operator-(const Mat3 &A, const Mat3 &B) {
  Mat3 C;
  for (int i = 0; i < 9; i++)
    C[i] = A[i] - B[i];
  return C;
}
inline Mat3 operator-(const Mat3 &A) { return -1.0 * A; }
inline Mat3 transpose(const Mat3 &A) { return {A[0], A[3], A[6], A[1], A[4], A[7], A[2], A[5], A[8]}; }
inline double trace(const Mat3 &A) { return A[0] + A[4] + A[8]; }
OVB_MATH_HD inline Mat3 outer(const Vec3 &a, const Vec3 &b) { return {a[0] * b[0], a[0] * b[1], a[0] * b[2], a[1] * b[0], a[1] * b[1], a[1] * b[2], a[2] * b[0], a[2] * b[1], a[2] * b[2]}; }
inline Mat4 operator*(const Mat4 &A, const Mat4 &B) {
  Mat4 C;
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) {
      double s = 0;
      for (int k = 0; k < 4; k++)
        s += A[i * 4 + k] * B[k * 4 + j];
      C[i * 4 + j] = s;
    }
  return C;
}
inline Mat4 operator*(double s, const Mat4 &A) {
  Mat4 C;
  for (int i = 0; i < 16; i++)
    C[i] = s * A[i];
  return C;
}
inline Mat4 operator+(const Mat4 &A, const Mat4 &B) {
  Mat4 C;
  for (int i = 0; i < 16; i++)
    C[i] = A[i] + B[i];
  return C;
}
inline Mat3 rot_of(const Mat4 &T) { return {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}; }
inline Vec3 pos_of(const Mat4 &T) { return {T[3], T[7], T[11]}; }
inline Mat4 make_T(const Mat3 &R, const Vec3 &p) { return {R[0], R[1], R[2], p[0], R[3], R[4], R[5], p[1], R[6], R[7], R[8], p[2], 0, 0, 0, 1}; }

OVB_MATH_HD inline Mat3 skew_x(const Vec3 &w) { return {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0}; } // quat_ops.h:135
inline Vec3 vee(const Mat3 &W) { return {W[7], W[2], W[3]}; }                                   // quat_ops.h:203

// quat_ops.h:88-133
inline Vec4 rot_2_quat(const Mat3 &rot) {
  Vec4 q;
  const double T = trace(rot);
  const double r00 = rot[0], r11 = rot[4], r22 = rot[8];
  if ((r00 >= T) && (r00 >= r11) && (r00 >= r22)) {
    q[0] = std::sqrt((1 + (2 * r00) - T) / 4);
    q[1] = (1 / (4 * q[0])) * (rot[1] + rot[3]);
    q[2] = (1 / (4 * q[0])) * (rot[2] + rot[6]);
    q[3] = (1 / (4 * q[0])) * (rot[5] - rot[7]);
  } else if ((r11 >= T) && (r11 >= r00) && (r11 >= r22)) {
    q[1] = std::sqrt((1 + (2 * r11) - T) / 4);
    q[0] = (1 / (4 * q[1])) * (rot[1] + rot[3]);
    q[2] = (1 / (4 * q[1])) * (rot[5] + rot[7]);
    q[3] = (1 / (4 * q[1])) * (rot[6] - rot[2]);
  } else if ((r22 >= T) && (r22 >= r00) && (r22 >= r11)) {
    q[2] = std::sqrt((1 + (2 * r22) - T) / 4);
    q[0] = (1 / (4 * q[2])) * (rot[2] + rot[6]);
    q[1] = (1 / (4 * q[2])) * (rot[5] + rot[7]);
    q[3] = (1 / (4 * q[2])) * (rot[1] - rot[3]);
  } else {
    q[3] = std::sqrt((1 + T) / 4);
    q[0] = (1 / (4 * q[3])) * (rot[5] - rot[7]);
    q[1] = (1 / (4 * q[3])) * (rot[6] - rot[2]);
    q[2] = (1 / (4 * q[3])) * (rot[1] - rot[3]);
  }
  if (q[3] < 0)
    for (auto &v : q)
      v = -v;
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (auto &v : q)
    v /= n;
  return q;
}

// quat_ops.h:152-157
OVB_MATH_HD inline Mat3 quat_2_Rot(const Vec4 &q) {
  const Vec3 v{q[0], q[1], q[2]};
  return (2 * q[3] * q[3] - 1) * eye3() - (2 * q[3]) * skew_x(v) + 2.0 * outer(v, v);
}

// quat_ops.h:180-194 (q ⊗ p, JPL)
OVB_MATH_HD inline Vec4 quat_multiply(const Vec4 &q, const Vec4 &p) {
  const Mat3 S = skew_x({q[0], q[1], q[2]});
  Vec4 t;
  for (int i = 0; i < 3; i++)
    t[i] = (q[3] * (i == 0) - S[i * 3]) * p[0] + (q[3] * (i == 1) - S[i * 3 + 1]) * p[1] + (q[3] * (i == 2) - S[i * 3 + 2]) * p[2] + q[i] * p[3];
  t[3] = -q[0] * p[0] - q[1] * p[1] - q[2] * p[2] + q[3] * p[3];
  if (t[3] < 0)
    for (auto &v : t)
      v = -v;
  const double n = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2] + t[3] * t[3]);
  for (auto &v : t)
    v /= n;
  return t;
}

// quat_ops.h:496-501
OVB_MATH_HD inline Vec4 quatnorm(Vec4 q) {
  if (q[3] < 0)
    for (auto &v : q)
      v = -v;
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (auto &v : q)
    v /= n;
  return q;
}

// quat_ops.h:482-489: 4x4 Omega(w) applied to a quaternion: Omega(w) q
inline Vec4 Omega_times(const Vec3 &w, const Vec4 &q) {
  const Mat3 S = skew_x(w);
  Vec4 r;
  for (int i = 0; i < 3; i++)
    r[i] = -(S[i * 3] * q[0] + S[i * 3 + 1] * q[1] + S[i * 3 + 2] * q[2]) + w[i] * q[3];
  r[3] = -(w[0] * q[0] + w[1] * q[1] + w[2] * q[2]);
  return r;
}

// quat_ops.h:231-262
inline Mat3 exp_so3(const Vec3 &w) {
  const Mat3 wx = skew_x(w);
  const double theta = norm(w);
  double A, B;
  if (theta < 1e-7) {
    A = 1;
    B = 0.5;
  } else {
    A = std::sin(theta) / theta;
    B = (1 - std::cos(theta)) / (theta * theta);
  }
  if (theta == 0)
    return eye3();
  return eye3() + A * wx + B * (wx * wx);
}

// quat_ops.h:273-315
inline Vec3 log_so3(const Mat3 &R) {
  const double R11 = R[0], R12 = R[1], R13 = R[2], R21 = R[3], R22 = R[4], R23 = R[5], R31 = R[6], R32 = R[7], R33 = R[8];
  const double tr = trace(R);
  if (tr + 1.0 < 1e-10) {
    if (std::abs(R33 + 1.0) > 1e-5)
      return (M_PI / std::sqrt(2.0 + 2.0 * R33)) * Vec3{R13, R23, 1.0 + R33};
    else if (std::abs(R22 + 1.0) > 1e-5)
      return (M_PI / std::sqrt(2.0 + 2.0 * R22)) * Vec3{R12, 1.0 + R22, R32};
    else
      return (M_PI / std::sqrt(2.0 + 2.0 * R11)) * Vec3{1.0 + R11, R21, R31};
  }
  double magnitude;
  const double tr_3 = tr - 3.0;
  if (tr_3 < -1e-7) {
    const double theta = std::acos((tr - 1.0) / 2.0);
    magnitude = theta / (2.0 * std::sin(theta));
  } else {
    magnitude = 0.5 - tr_3 / 12.0;
  }
  return magnitude * Vec3{R32 - R23, R13 - R31, R21 - R12};
}

// quat_ops.h:343-380
inline Mat4 exp_se3(const Vec6 &vec) {
  const Vec3 w{vec[0], vec[1], vec[2]}, u{vec[3], vec[4], vec[5]};
  const double theta = std::sqrt(dot(w, w));
  const Mat3 wskew = skew_x(w);
  double A, B, C;
  if (theta < 1e-7) {
    A = 1;
    B = 0.5;
    C = 1.0 / 6.0;
  } else {
    A = std::sin(theta) / theta;
    B = (1 - std::cos(theta)) / (theta * theta);
    C = (1 - A) / (theta * theta);
  }
  const Mat3 w2 = wskew * wskew;
  const Mat3 V = eye3() + B * wskew + C * w2;
  return make_T(eye3() + A * wskew + B * w2, V * u);
}

// quat_ops.h:402-426
inline Vec6 log_se3(const Mat4 &mat) {
  const Vec3 w = log_so3(rot_of(mat));
  const Vec3 T = pos_of(mat);
  const double t = norm(w);
  if (t < 1e-10)
    return {w[0], w[1], w[2], T[0], T[1], T[2]};
  const Mat3 W = skew_x((1.0 / t) * w);
  const double Tan = std::tan(0.5 * t);
  const Vec3 WT = W * T;
  const Vec3 u = T - (0.5 * t) * WT + (1 - t / (2. * Tan)) * (W * WT);
  return {w[0], w[1], w[2], u[0], u[1], u[2]};
}

// quat_ops.h:445-450
inline Mat4 hat_se3(const Vec6 &v) {
  const Mat3 S = skew_x({v[0], v[1], v[2]});
  return {S[0], S[1], S[2], v[3], S[3], S[4], S[5], v[4], S[6], S[7], S[8], v[5], 0, 0, 0, 0};
}
// quat_ops.h:457-462
inline Mat4 Inv_se3(const Mat4 &T) {
  const Mat3 Rt = transpose(rot_of(T));
  return make_T(Rt, -(Rt * pos_of(T)));
}
inline Vec6 operator*(double s, const Vec6 &v) { return {s * v[0], s * v[1], s * v[2], s * v[3], s * v[4], s * v[5]}; }

// quat_ops.h:515-527, :537
inline Mat3 Jl_so3(const Vec3 &w) {
  const double theta = norm(w);
  if (theta < 1e-6)
    return eye3();
  const Vec3 a = (1.0 / theta) * w;
  return (std::sin(theta) / theta) * eye3() + (1 - std::sin(theta) / theta) * outer(a, a) + ((1 - std::cos(theta)) / theta) * skew_x(a);
}
inline Mat3 Jr_so3(const Vec3 &w) { return Jl_so3(-w); }

} // namespace ovb200
#endif
