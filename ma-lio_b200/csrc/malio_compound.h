// malio_compound.h — struct Pose and Barfoot's 4th-order SE(3) covariance compounding, shared by the host C-ABI
// (malio_host.cpp: malio_pose_initial, malio_compound_*, malio_build_pose_unc) and the device's per-scan uncertainty build
// (malio_preproc.cu: malio_scan_uncertainty).  One source for both: __host__ __device__ inline, and with -fmad=false on the
// device (the host build has no FMA) the two return the same bits for the same inputs.
//
// Reference interface mirrored (paths relative to the MA_LIO source tree):
//   PoseInitial                                 include/common_lib.h:129-142
//   adjointMatrix, covop1, covop2               include/associate_uct.hpp:8-27
//   compoundInvPoseWithCov / compoundPoseWithCov, method 2   include/associate_uct.hpp:29-142
//   pose_unc of one scan                        src/laserMapping.cpp:1028-1048
#ifndef MALIO_COMPOUND_H_
#define MALIO_COMPOUND_H_

#include "malio_b200.h"
#include "malio_se3.h"

namespace malio_compound {

struct M6 { double a[6][6]; };
struct M3s { double a[3][3]; };
MALIO_CHD inline M3s blk(const M6& m, int r, int c) { M3s o; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) o.a[i][j] = m.a[r + i][c + j]; return o; }
MALIO_CHD inline void set_blk(M6& m, int r, int c, const M3s& b) { for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) m.a[r + i][c + j] = b.a[i][j]; }
MALIO_CHD inline M3s mul(const M3s& x, const M3s& y) { M3s o; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += x.a[i][k] * y.a[k][j]; o.a[i][j] = s; } return o; }
MALIO_CHD inline M3s add(const M3s& x, const M3s& y) { M3s o; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) o.a[i][j] = x.a[i][j] + y.a[i][j]; return o; }
MALIO_CHD inline M3s tr(const M3s& x) { M3s o; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) o.a[i][j] = x.a[j][i]; return o; }
MALIO_CHD inline M3s covop1(const M3s& B) {   // -tr(B) I + B   (:17-21)
  const double t = B.a[0][0] + B.a[1][1] + B.a[2][2];
  M3s o = B;
  for (int i = 0; i < 3; ++i) o.a[i][i] += -t;
  return o;
}
MALIO_CHD inline M3s covop2(const M3s& B, const M3s& C) { return add(mul(covop1(B), covop1(C)), covop1(mul(C, B))); }   // :23-27
MALIO_CHD inline M6 mul6(const M6& x, const M6& y) { M6 o; for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) { double s = 0; for (int k = 0; k < 6; ++k) s += x.a[i][k] * y.a[k][j]; o.a[i][j] = s; } return o; }
MALIO_CHD inline M6 tr6(const M6& x) { M6 o; for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) o.a[i][j] = x.a[j][i]; return o; }
MALIO_CHD inline M6 load6(const double* p) { M6 o; for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) o.a[i][j] = p[6 * i + j]; return o; }
MALIO_CHD inline void copy_n(double* dst, const double* src, int n) { for (int k = 0; k < n; ++k) dst[k] = src[k]; }
MALIO_CHD inline void set_T(malio_pose* p) {   // T_ from q_, t_ (bottom row 0 0 0 1)
  double R[9];
  malio_se3::q_to_R(p->q, R);
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) p->T[4 * i + j] = R[3 * i + j]; p->T[4 * i + 3] = p->t[i]; }
  p->T[12] = 0; p->T[13] = 0; p->T[14] = 0; p->T[15] = 1;
}
// adjointMatrix(T.inverse()) (:8-15, :44, :99); T is a rigid transform [R t; 0 1]: inverse = [R^T, -R^T t]
MALIO_CHD inline M6 adjoint_of_inverse(const double T[16]) {
  double Ri[3][3], ti[3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Ri[i][j] = T[4 * j + i];
  for (int i = 0; i < 3; ++i) ti[i] = -(Ri[i][0] * T[3] + Ri[i][1] * T[7] + Ri[i][2] * T[11]);
  M6 Ad{};
  const double S[3][3] = {{0, -ti[2], ti[1]}, {ti[2], 0, -ti[0]}, {-ti[1], ti[0], 0}};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      Ad.a[i][j] = Ri[i][j];
      Ad.a[3 + i][3 + j] = Ri[i][j];
      double sum = 0;
      for (int k = 0; k < 3; ++k) sum += S[i][k] * Ri[k][j];
      Ad.a[i][3 + j] = sum;
    }
  return Ad;
}
// the shared 4th-order part (:52-85 and :107-134): cov_cp = c1' + c2 + (A1 c2 + c2 A1^T + A2 c1' + c1' A2^T)/12 + B/4
MALIO_CHD inline void compound_cov(const M6& c1p, const M6& c2, double* out) {
  const M3s c1rr = blk(c1p, 0, 0), c1rp = blk(c1p, 0, 3), c1pp = blk(c1p, 3, 3);
  const M3s c2rr = blk(c2, 0, 0), c2rp = blk(c2, 0, 3), c2pp = blk(c2, 3, 3);
  M6 A1{}, A2{}, B{};
  set_blk(A1, 0, 0, covop1(c1pp)); set_blk(A1, 0, 3, covop1(add(c1rp, tr(c1rp)))); set_blk(A1, 3, 3, covop1(c1pp));
  set_blk(A2, 0, 0, covop1(c2pp)); set_blk(A2, 0, 3, covop1(add(c2rp, tr(c2rp)))); set_blk(A2, 3, 3, covop1(c2pp));
  const M3s Brr = add(add(covop2(c1pp, c2rr), covop2(tr(c1rp), c2rp)), add(covop2(c1rp, tr(c2rp)), covop2(c1rr, c2pp)));
  const M3s Brp = add(covop2(c1pp, tr(c2rp)), covop2(tr(c1rp), c2pp));
  const M3s Bpp = covop2(c1pp, c2pp);
  set_blk(B, 0, 0, Brr); set_blk(B, 0, 3, Brp); set_blk(B, 3, 0, tr(Brp)); set_blk(B, 3, 3, Bpp);
  const M6 t1 = mul6(A1, c2), t2 = mul6(c2, tr6(A1)), t3 = mul6(A2, c1p), t4 = mul6(c1p, tr6(A2));
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j)
      out[6 * i + j] = c1p.a[i][j] + c2.a[i][j] + (t1.a[i][j] + t2.a[i][j] + t3.a[i][j] + t4.a[i][j]) / 12 + B.a[i][j] / 4;
}

// PoseInitial (common_lib.h:129-142); cov may alias pose->cov
MALIO_CHD inline void pose_initial(malio_pose* pose, const double t[3], const double q[4], const double cov[36]) {
  for (int k = 0; k < 3; ++k) pose->t[k] = t[k];
  for (int k = 0; k < 4; ++k) pose->q[k] = q[k];
  set_T(pose);
  if (cov != pose->cov) copy_n(pose->cov, cov, 36);
}
// compoundPoseWithCov, method 2.  Field order of associate_uct.hpp:93-100 — pose_cp may be pose_2
MALIO_CHD inline void compound_pose_with_cov(const malio_pose* pose_1, const double* cov_1, const malio_pose* pose_2, const double* cov_2,
                                             malio_pose* pose_cp, double* cov_cp) {
  double q[4], t[3];
  malio_se3::q_mul(pose_1->q, pose_2->q, q);
  for (int k = 0; k < 4; ++k) pose_cp->q[k] = q[k];                       // :93
  malio_se3::q_rot(pose_1->q, pose_2->t, t);
  for (int k = 0; k < 3; ++k) pose_cp->t[k] = t[k] + pose_1->t[k];        // :94
  set_T(pose_cp);                                                         // :96-98
  const M6 Ad = adjoint_of_inverse(pose_2->T);                            // :99 (the new T_ when pose_cp aliases pose_2)
  const M6 c1p = mul6(mul6(Ad, load6(cov_1)), tr6(Ad));                   // :100
  const M6 c2 = load6(cov_2);
  double out[36];
  compound_cov(c1p, c2, out);
  copy_n(cov_cp, out, 36);                                                // :133
  copy_n(pose_cp->cov, out, 36);                                          // :134
}
// compoundInvPoseWithCov, method 2 (associate_uct.hpp:29-86); pose_cp->cov is written only through cov_cp
MALIO_CHD inline void compound_inv_pose_with_cov(const malio_pose* pose_1, const double* cov_1, const malio_pose* pose_2, const double* cov_2,
                                                 malio_pose* pose_cp, double* cov_cp) {
  const double qc[4] = {pose_1->q[0], -pose_1->q[1], -pose_1->q[2], -pose_1->q[3]};
  double q[4], d[3], t[3];
  malio_se3::q_mul(qc, pose_2->q, q);
  for (int k = 0; k < 3; ++k) d[k] = pose_2->t[k] - pose_1->t[k];
  malio_se3::q_rot(qc, d, t);
  for (int k = 0; k < 4; ++k) pose_cp->q[k] = q[k];                       // :36
  for (int k = 0; k < 3; ++k) pose_cp->t[k] = t[k];                       // :37
  set_T(pose_cp);                                                         // :41-43
  const M6 Ad = adjoint_of_inverse(pose_cp->T);                           // :44
  const M6 c1p = mul6(mul6(Ad, load6(cov_1)), tr6(Ad));                   // :45
  const M6 c2 = load6(cov_2);
  double out[36];
  compound_cov(c1p, c2, out);
  copy_n(cov_cp, out, 36);                                                // :85
}
// one entry of pose_unc[num] from kf.lidar_uncertainty[num][i] (laserMapping.cpp:1036, :1042-1045): LiDAR 0's entries are
// taken as they are; the others go through LiDAR 0's frame, the last two compoundings with their output aliasing the 2nd input
// tcomp = kf.temporal_comp[num - 1] (not read for num == 0)
MALIO_CHD inline void pose_unc_entry(int num, const malio_pose* extrinsic, const malio_pose* tcomp, const malio_pose* lu,
                                     malio_pose_entry* out) {
  if (num == 0) {
    copy_n(out->T, lu->T, 16);
    copy_n(out->cov, lu->cov, 36);
    return;
  }
  malio_pose pose_point{};
  compound_pose_with_cov(&extrinsic[num], extrinsic[num].cov, lu, lu->cov, &pose_point, pose_point.cov);
  compound_pose_with_cov(tcomp, tcomp->cov, &pose_point, pose_point.cov, &pose_point, pose_point.cov);
  compound_inv_pose_with_cov(&extrinsic[0], extrinsic[0].cov, &pose_point, pose_point.cov, &pose_point, pose_point.cov);
  copy_n(out->T, pose_point.T, 16);
  copy_n(out->cov, pose_point.cov, 36);
}

}  // namespace malio_compound

#endif  // MALIO_COMPOUND_H_
