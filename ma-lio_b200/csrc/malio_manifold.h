// malio_manifold.h — the state manifold of the filter (MTK SO3 / S2 / vect operators, A_matrix) used by the host IESKF
// (malio_host.cpp).
//
// Reference interface mirrored (paths relative to /root/reference/MA_LIO):
//   state_ikfom manifold                        src/use-ikfom.hpp:14-27
//   MTK SO3 / S2 / vect boxplus, boxminus       include/IKFoM_toolkit/mtk/types/{SOn,S2,vect}.hpp
//   MTK::A_matrix, exp, log                     include/IKFoM_toolkit/mtk/src/mtkmath.hpp:235-289
#ifndef MALIO_MANIFOLD_H_
#define MALIO_MANIFOLD_H_

#include <cmath>
#include <limits>

#include "malio_b200.h"

namespace malio_manifold {

// ---------------------------------------------------------------- rotations
struct Quat { double w, x, y, z; };
inline Quat qload(const double* q) { return Quat{q[0], q[1], q[2], q[3]}; }
inline void qstore(const Quat& q, double* o) { o[0] = q.w; o[1] = q.x; o[2] = q.y; o[3] = q.z; }
inline Quat qconj(const Quat& q) { return Quat{q.w, -q.x, -q.y, -q.z}; }
inline Quat qmul(const Quat& a, const Quat& b) {
  return Quat{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
              a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
struct M3 { double m[3][3]; };
inline M3 hat3(const double v[3]) { return M3{{{0, -v[2], v[1]}, {v[2], 0, -v[0]}, {-v[1], v[0], 0}}}; }
inline M3 mul3(const M3& A, const M3& B) {
  M3 C{};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C.m[i][j] = A.m[i][0] * B.m[0][j] + A.m[i][1] * B.m[1][j] + A.m[i][2] * B.m[2][j];
  return C;
}
inline M3 rotmat(const Quat& q) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  return M3{{{1 - (tyy + tzz), txy - twz, txz + twy}, {txy + twz, 1 - (txx + tzz), tyz - twx}, {txz - twy, tyz + twx, 1 - (txx + tyy)}}};
}

constexpr double kTol = 1e-11;                    // MTK::tolerance<double>() (mtkmath.hpp:122)
constexpr double kGrav = 98090.0 / 10000.0;       // S2<double,98090,10000,1> (use-ikfom.hpp:8)

// cos(sqrt(x2)), sinc(sqrt(x2))  (mtkmath.hpp:141-171)
inline void cos_sinc_sqrt(double x2, double& c, double& sc) {
  const double b0 = std::numeric_limits<double>::epsilon();
  const double bn = std::sqrt(std::sqrt(b0));
  if (x2 >= bn) {
    const double x = std::sqrt(x2);
    c = std::cos(x);
    sc = std::sin(x) / x;
    return;
  }
  const double inv[] = {1 / 3., 1 / 4., 1 / 5., 1 / 6., 1 / 7., 1 / 8., 1 / 9.};
  double ci = 1., si = 1., term = -1 / 2. * x2;
  for (int i = 0; i < 3; ++i) {
    ci += term;
    term *= inv[2 * i];
    si += term;
    term *= -inv[2 * i + 1] * x2;
  }
  c = ci;
  sc = si;
}
// quaternion of MTK::exp(vec, scale) (mtkmath.hpp:249-256)
inline Quat exp_quat(const double v[3], double scale) {
  double c, sc;
  cos_sinc_sqrt(scale * scale * (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]), c, sc);
  const double m = sc * scale;
  return Quat{c, m * v[0], m * v[1], m * v[2]};
}
// SO3::log (SOn.hpp:341-345 -> mtkmath.hpp:268-289, scale 2, +-periodic)
inline void so3_log(const Quat& q, double out[3]) {
  double nv = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
  if (nv < kTol) nv = kTol;
  const double s = 2.0 / nv * std::atan(nv / q.w);
  out[0] = s * q.x; out[1] = s * q.y; out[2] = s * q.z;
}
// MTK::A_matrix (mtkmath.hpp:235-247)
inline M3 A_matrix(const double v[3]) {
  const double sq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], nrm = std::sqrt(sq);
  M3 R{{{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}};
  if (nrm < kTol) return R;
  const M3 H = hat3(v), HH = mul3(H, H);
  const double a = (1 - std::cos(nrm)) / sq, b = (1 - std::sin(nrm) / nrm) / sq;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R.m[i][j] += a * H.m[i][j] + b * HH.m[i][j];
  return R;
}
inline M3 transpose3(const M3& A) {
  M3 T{};
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) T.m[i][j] = A.m[j][i];
  return T;
}

// S2 chart with the x axis as pole (S2_typ == 1, S2.hpp:225-243): Bx is 3x2
inline void S2_Bx(const double v[3], double B[3][2]) {
  const double L = kGrav;
  if (v[0] + L > kTol) {
    const double d = L + v[0];
    B[0][0] = -v[1];              B[0][1] = -v[2];
    B[1][0] = L - v[1] * v[1] / d; B[1][1] = -v[2] * v[1] / d;
    B[2][0] = -v[2] * v[1] / d;    B[2][1] = L - v[2] * v[2] / d;
    for (int i = 0; i < 3; ++i) { B[i][0] /= L; B[i][1] /= L; }
  } else {
    for (int i = 0; i < 3; ++i) B[i][0] = B[i][1] = 0;
    B[1][1] = -1;
    B[2][0] = 1;
  }
}
inline void S2_boxplus(double v[3], const double d[2]) {   // S2.hpp:136-142
  double B[3][2];
  S2_Bx(v, B);
  const double Bu[3] = {B[0][0] * d[0] + B[0][1] * d[1], B[1][0] * d[0] + B[1][1] * d[1], B[2][0] * d[0] + B[2][1] * d[1]};
  const M3 R = rotmat(exp_quat(Bu, 0.5));
  const double o[3] = {R.m[0][0] * v[0] + R.m[0][1] * v[1] + R.m[0][2] * v[2], R.m[1][0] * v[0] + R.m[1][1] * v[1] + R.m[1][2] * v[2],
                       R.m[2][0] * v[0] + R.m[2][1] * v[1] + R.m[2][2] * v[2]};
  v[0] = o[0]; v[1] = o[1]; v[2] = o[2];
}
inline void S2_boxminus(const double v[3], const double o[3], double res[2]) {   // S2.hpp:144-168
  const double cr[3] = {v[1] * o[2] - v[2] * o[1], v[2] * o[0] - v[0] * o[2], v[0] * o[1] - v[1] * o[0]};
  const double v_sin = std::sqrt(cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2]);
  const double v_cos = v[0] * o[0] + v[1] * o[1] + v[2] * o[2];
  const double theta = std::atan2(v_sin, v_cos);
  if (v_sin < kTol) {
    res[0] = (std::fabs(theta) > kTol) ? 3.1415926 : 0.0;
    res[1] = 0.0;
    return;
  }
  double B[3][2];
  S2_Bx(o, B);
  const double u[3] = {o[1] * v[2] - o[2] * v[1], o[2] * v[0] - o[0] * v[2], o[0] * v[1] - o[1] * v[0]};   // hat(o) v
  const double f = theta / v_sin;
  res[0] = f * (B[0][0] * u[0] + B[1][0] * u[1] + B[2][0] * u[2]);
  res[1] = f * (B[0][1] * u[0] + B[1][1] * u[1] + B[2][1] * u[2]);
}
// J = Nx(x) * Mx(x0, delta), the 2x2 projection of the S2 block (esekfom.hpp:560-564; S2.hpp:269-291).
// Mx's exp_delta uses scalar(1/2) == 0 in the reference, i.e. the identity rotation.
inline void S2_projection(const double x[3], const double x0[3], const double delta[2], double J[2][2]) {
  double Bx[3][2], B0[3][2];
  S2_Bx(x, Bx);
  S2_Bx(x0, B0);
  const M3 Hx = hat3(x), H0 = hat3(x0);
  double Nx[2][3];
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 3; ++j) Nx[i][j] = (Bx[0][i] * Hx.m[0][j] + Bx[1][i] * Hx.m[1][j] + Bx[2][i] * Hx.m[2][j]) / kGrav / kGrav;
  double Mx[3][2];
  if (std::sqrt(delta[0] * delta[0] + delta[1] * delta[1]) < kTol) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 2; ++j) Mx[i][j] = -(H0.m[i][0] * B0[0][j] + H0.m[i][1] * B0[1][j] + H0.m[i][2] * B0[2][j]);
  } else {
    const double Bu[3] = {B0[0][0] * delta[0] + B0[0][1] * delta[1], B0[1][0] * delta[0] + B0[1][1] * delta[1],
                          B0[2][0] * delta[0] + B0[2][1] * delta[1]};
    const M3 HA = mul3(H0, transpose3(A_matrix(Bu)));
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 2; ++j) Mx[i][j] = -(HA.m[i][0] * B0[0][j] + HA.m[i][1] * B0[1][j] + HA.m[i][2] * B0[2][j]);
  }
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) J[i][j] = Nx[i][0] * Mx[0][j] + Nx[i][1] * Mx[1][j] + Nx[i][2] * Mx[2][j];
}

// ---------------------------------------------------------------- state manifold
struct StateLayout {
  int L, n, c, rot, vel, bg, ba, grav;
  int offR[MALIO_MAX_LIDAR], offT[MALIO_MAX_LIDAR];
  int so3[1 + MALIO_MAX_LIDAR];
  explicit StateLayout(int L_) : L(L_) {
    n = 17 + 6 * L; c = 6 * (L + 1); rot = 3;
    so3[0] = rot;
    for (int l = 0; l < L; ++l) { offR[l] = 6 + 3 * l; offT[l] = 6 + 3 * L + 3 * l; so3[1 + l] = offR[l]; }
    vel = 6 + 6 * L; bg = vel + 3; ba = bg + 3; grav = ba + 3;
  }
};
inline void boxminus(const StateLayout& ly, const malio_state& x, const malio_state& x0, double* d) {
  for (int k = 0; k < 3; ++k) d[k] = x.pos[k] - x0.pos[k];
  so3_log(qmul(qconj(qload(x0.rot)), qload(x.rot)), d + ly.rot);
  for (int l = 0; l < ly.L; ++l) {
    so3_log(qmul(qconj(qload(x0.ext[l].q)), qload(x.ext[l].q)), d + ly.offR[l]);
    for (int k = 0; k < 3; ++k) d[ly.offT[l] + k] = x.ext[l].t[k] - x0.ext[l].t[k];
  }
  for (int k = 0; k < 3; ++k) {
    d[ly.vel + k] = x.vel[k] - x0.vel[k];
    d[ly.bg + k] = x.bg[k] - x0.bg[k];
    d[ly.ba + k] = x.ba[k] - x0.ba[k];
  }
  S2_boxminus(x.grav, x0.grav, d + ly.grav);
}
inline void boxplus(const StateLayout& ly, malio_state& x, const double* d) {
  for (int k = 0; k < 3; ++k) x.pos[k] += d[k];
  qstore(qmul(qload(x.rot), exp_quat(d + ly.rot, 0.5)), x.rot);
  for (int l = 0; l < ly.L; ++l) {
    qstore(qmul(qload(x.ext[l].q), exp_quat(d + ly.offR[l], 0.5)), x.ext[l].q);
    for (int k = 0; k < 3; ++k) x.ext[l].t[k] += d[ly.offT[l] + k];
  }
  for (int k = 0; k < 3; ++k) {
    x.vel[k] += d[ly.vel + k];
    x.bg[k] += d[ly.bg + k];
    x.ba[k] += d[ly.ba + k];
  }
  S2_boxplus(x.grav, d + ly.grav);
}

// singular values of the N x 3 matrix whose Gram matrix is S (descending) = sqrt(eig(S)): cyclic Jacobi on the 3x3
inline void sym3_singular_values(const double S[6], double sv[3]) {
  double A[3][3] = {{S[0], S[1], S[2]}, {S[1], S[3], S[4]}, {S[2], S[4], S[5]}};
  for (int sweep = 0; sweep < 50; ++sweep) {
    const double off = std::fabs(A[0][1]) + std::fabs(A[0][2]) + std::fabs(A[1][2]);
    // converged: the off-diagonal mass is below 1e-22 of the diagonal's (eigenvalue error ~ off^2 / gap: far below one ulp)
    if (off <= 1e-22 * (std::fabs(A[0][0]) + std::fabs(A[1][1]) + std::fabs(A[2][2]))) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (A[p][q] == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2 * A[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
        const double c = 1 / std::sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < 3; ++k) { const double a = A[k][p], b = A[k][q]; A[k][p] = c * a - s * b; A[k][q] = s * a + c * b; }
        for (int k = 0; k < 3; ++k) { const double a = A[p][k], b = A[q][k]; A[p][k] = c * a - s * b; A[q][k] = s * a + c * b; }
      }
  }
  double e[3] = {A[0][0], A[1][1], A[2][2]};
  if (e[0] > e[1]) { const double t_ = e[0]; e[0] = e[1]; e[1] = t_; }
  if (e[1] > e[2]) { const double t_ = e[1]; e[1] = e[2]; e[2] = t_; }
  if (e[0] > e[1]) { const double t_ = e[0]; e[0] = e[1]; e[1] = t_; }
  sv[0] = std::sqrt((e[2] > 0.0 ? e[2] : 0.0));
  sv[1] = std::sqrt((e[1] > 0.0 ? e[1] : 0.0));
  sv[2] = std::sqrt((e[0] > 0.0 ? e[0] : 0.0));
}

}  // namespace malio_manifold

#endif  // MALIO_MANIFOLD_H_
