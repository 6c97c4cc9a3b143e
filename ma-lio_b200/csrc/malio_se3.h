// malio_se3.h — the library's quaternion and SE(3) algebra, one source for the host and the device: the kernels (through
// malio_device.cuh), the compounding (malio_compound.h), the host IESKF's manifold (malio_manifold.h) and the host code that
// builds guesses for the device.  Every function keeps the operation order of the Eigen or quat_ops.h expression it restates;
// the device build has -fmad=false and the host build has no FMA, so the host and the device return the same bits for the
// same inputs.  No CUDA header: g++ compiles it as it is.  Quaternions are (w, x, y, z), matrices row-major.
//
// Reference interface mirrored (paths relative to the MA_LIO source tree):
//   Eigen Quaternion * Vector3, Quaternion * Quaternion, toRotationMatrix, operator=(Matrix3)
//   log_so3, exp_se3, log_se3, Inv_se3              include/quat_ops.h:150-257
#ifndef MALIO_SE3_H_
#define MALIO_SE3_H_

#include <cmath>

// MALIO_CHD: callable from host and device code.  MALIO_CHD_FI: the same, always inlined (the per-point rotations of the
// hot kernels)
#ifdef __CUDACC__
#define MALIO_CHD __host__ __device__
#define MALIO_CHD_FI __host__ __device__ __forceinline__
#else
#define MALIO_CHD
#define MALIO_CHD_FI inline
#endif

namespace malio_se3 {

MALIO_CHD_FI void cross3(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
// Quaternion * vector as Eigen's _transformVector: v + w*uv + qv x uv, uv = 2 (qv x v)
MALIO_CHD_FI void q_rot(const double q[4], const double v[3], double o[3]) {
  const double qv[3] = {q[1], q[2], q[3]};
  double uv[3], c2[3];
  cross3(qv, v, uv);
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  cross3(qv, uv, c2);
  o[0] = v[0] + q[0] * uv[0] + c2[0];
  o[1] = v[1] + q[0] * uv[1] + c2[1];
  o[2] = v[2] + q[0] * uv[2] + c2[2];
}
MALIO_CHD_FI void q_rot_conj(const double q[4], const double v[3], double o[3]) {
  const double qc[4] = {q[0], -q[1], -q[2], -q[3]};
  q_rot(qc, v, o);
}
// Eigen's quaternion product a * b; o may alias a or b
MALIO_CHD inline void q_mul(const double a[4], const double b[4], double o[4]) {
  const double w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  const double x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  const double y = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  const double z = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
  o[0] = w; o[1] = x; o[2] = y; o[3] = z;
}
// Eigen's toRotationMatrix
MALIO_CHD inline void q_to_R(const double q[4], double R[9]) {
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x,
               tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
// q_yaw(theta) * q, q_yaw(theta) = (cos(theta/2), 0, 0, sin(theta/2)): the candidate rotations of malio_relocalize (malio_b200.h,
// step 1).  Host only: cos and sin are the C library's, so that the device searches the rotations the caller computes
inline void q_yaw_mul(double theta, const double q[4], double o[4]) {
  const double c = std::cos(theta / 2.0), s = std::sin(theta / 2.0);
  const double w0 = q[0], x0 = q[1], y0 = q[2], z0 = q[3];
  o[0] = c * w0 - s * z0;
  o[1] = c * x0 - s * y0;
  o[2] = c * y0 + s * x0;
  o[3] = c * z0 + s * w0;
}

// ------------------------------------------------------------------ quat_ops.h
MALIO_CHD inline void mul3(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
// 4x4 homogeneous product in Eigen's coefficient order (k ascending, the bottom row 0 0 0 1 included)
MALIO_CHD inline void mul4(const double* A, const double* B, double* C) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = A[4 * i] * B[j];
      for (int k = 1; k < 4; ++k) s += A[4 * i + k] * B[4 * k + j];
      C[4 * i + j] = s;
    }
}
// quat_ops.h:150-187
MALIO_CHD inline void log_so3(const double R[9], double omega[3]) {
  const double R11 = R[0], R12 = R[1], R13 = R[2], R21 = R[3], R22 = R[4], R23 = R[5], R31 = R[6], R32 = R[7], R33 = R[8];
  const double tr = R11 + R22 + R33;
  const double PI = 3.14159265358979323846;
  if (tr + 1.0 < 1e-10) {
    if (fabs(R33 + 1.0) > 1e-5) {
      const double f = PI / sqrt(2.0 + 2.0 * R33);
      omega[0] = f * R13; omega[1] = f * R23; omega[2] = f * (1.0 + R33);
    } else if (fabs(R22 + 1.0) > 1e-5) {
      const double f = PI / sqrt(2.0 + 2.0 * R22);
      omega[0] = f * R12; omega[1] = f * (1.0 + R22); omega[2] = f * R32;
    } else {
      const double f = PI / sqrt(2.0 + 2.0 * R11);
      omega[0] = f * (1.0 + R11); omega[1] = f * R21; omega[2] = f * R31;
    }
  } else {
    double magnitude;
    const double tr_3 = tr - 3.0;
    if (tr_3 < -1e-7) {
      const double theta = acos((tr - 1.0) / 2.0);
      magnitude = theta / (2.0 * sin(theta));
    } else {
      magnitude = 0.5 - tr_3 / 12.0;
    }
    omega[0] = magnitude * (R32 - R23); omega[1] = magnitude * (R13 - R31); omega[2] = magnitude * (R21 - R12);
  }
}
// quat_ops.h:190-220
MALIO_CHD inline void exp_se3(const double vec[6], double mat[16]) {
  const double w0 = vec[0], w1 = vec[1], w2 = vec[2];
  const double theta = sqrt(w0 * w0 + w1 * w1 + w2 * w2);
  const double K[9] = {0, -w2, w1, w2, 0, -w0, -w1, w0, 0};
  double A, B, Cc;
  if (theta < 1e-7) { A = 1; B = 0.5; Cc = 1.0 / 6.0; }
  else { A = sin(theta) / theta; B = (1 - cos(theta)) / (theta * theta); Cc = (1 - A) / (theta * theta); }
  double K2[9];
  mul3(K, K, K2);
  double V[9];
  for (int i = 0; i < 9; ++i) {
    const double I = (i % 4 == 0) ? 1.0 : 0.0;
    V[i] = I + B * K[i] + Cc * K2[i];
    const double r = I + A * K[i] + B * K2[i];
    mat[4 * (i / 3) + (i % 3)] = r;
  }
  for (int i = 0; i < 3; ++i) mat[4 * i + 3] = V[3 * i] * vec[3] + V[3 * i + 1] * vec[4] + V[3 * i + 2] * vec[5];
  mat[12] = 0; mat[13] = 0; mat[14] = 0; mat[15] = 1;
}
// quat_ops.h:223-243
MALIO_CHD inline void log_se3(const double mat[16], double out[6]) {
  const double R[9] = {mat[0], mat[1], mat[2], mat[4], mat[5], mat[6], mat[8], mat[9], mat[10]};
  double w[3];
  log_so3(R, w);
  const double T[3] = {mat[3], mat[7], mat[11]};
  const double t = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  out[0] = w[0]; out[1] = w[1]; out[2] = w[2];
  if (t < 1e-10) { out[3] = T[0]; out[4] = T[1]; out[5] = T[2]; return; }
  const double a[3] = {w[0] / t, w[1] / t, w[2] / t};
  const double W[9] = {0, -a[2], a[1], a[2], 0, -a[0], -a[1], a[0], 0};
  const double Tan = tan(0.5 * t);
  double WT[3], WWT[3];
  for (int i = 0; i < 3; ++i) WT[i] = W[3 * i] * T[0] + W[3 * i + 1] * T[1] + W[3 * i + 2] * T[2];
  for (int i = 0; i < 3; ++i) WWT[i] = W[3 * i] * WT[0] + W[3 * i + 1] * WT[1] + W[3 * i + 2] * WT[2];
  for (int i = 0; i < 3; ++i) out[3 + i] = T[i] - (0.5 * t) * WT[i] + (1 - t / (2. * Tan)) * WWT[i];
}
// quat_ops.h:252-257
MALIO_CHD inline void inv_se3(const double T[16], double Ti[16]) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Ti[4 * i + j] = T[4 * j + i];
  for (int i = 0; i < 3; ++i) Ti[4 * i + 3] = -(Ti[4 * i] * T[3] + Ti[4 * i + 1] * T[7] + Ti[4 * i + 2] * T[11]);
  Ti[12] = 0; Ti[13] = 0; Ti[14] = 0; Ti[15] = 1;
}
// Eigen 3.3 QuaternionBase::operator=(rotation matrix); m row-major 3x3
MALIO_CHD inline void quat_from_R(const double m[9], double q[4]) {
  double t = m[0] + m[4] + m[8];
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (m[7] - m[5]) * t;
    q[2] = (m[2] - m[6]) * t;
    q[3] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m[4 * i] - m[4 * j] - m[4 * k] + 1.0);
    double qv[3];
    qv[i] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[3 * k + j] - m[3 * j + k]) * t;
    qv[j] = (m[3 * j + i] + m[3 * i + j]) * t;
    qv[k] = (m[3 * k + i] + m[3 * i + k]) * t;
    q[1] = qv[0]; q[2] = qv[1]; q[3] = qv[2];
  }
}

}  // namespace malio_se3

#endif  // MALIO_SE3_H_
