// malio_pass.cu — the measurement pass of libmalio_b200.so, sm_90a (DESIGN.md has the data layout and rooflines):
//   K2 fit/tau/gate    h_share_model S1 + esti_plane (once per search) + evalPointUncertainty (once per scan)
//                      (laserMapping.cpp:559-612, 725-743; common_lib.h:144-190; associate_uct.hpp:153-175)
//   K3 reduce_kernel   h_share_model S3-S4 rows fused with esekfom.hpp:622-635 (H^T R^-1 H, H^T R^-1 h)
// both fused into one cooperative pass_kernel per pass, its in-kernel multi-GPU exchange, the NCCL path between separate
// kernels, and measure(), which runs one pass: search (malio_knn.cu), pass kernels, host epilogue.
// Compiled with -fmad=false: every float/double expression below is evaluated with the same IEEE operations,
// in the same order, as the reference's x86-64 build (no FMA, CMakeLists.txt:8) so that the selection gates do not
// flip; explicit fma() is used only in the FP64 accumulation of K3.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "malio_internal.h"
#include "malio_device.cuh"

using namespace malio_devstate;
namespace {

__device__ __forceinline__ void mat3_mul(const double R[9], const double v[3], double o[3]) {
  o[0] = fma(R[2], v[2], fma(R[1], v[1], R[0] * v[0]));
  o[1] = fma(R[5], v[2], fma(R[4], v[1], R[3] * v[0]));
  o[2] = fma(R[8], v[2], fma(R[7], v[1], R[6] * v[0]));
}
__device__ __forceinline__ void cross3_fma(const double a[3], const double b[3], double o[3]) {
  o[0] = fma(a[1], b[2], -(a[2] * b[1]));
  o[1] = fma(a[2], b[0], -(a[0] * b[2]));
  o[2] = fma(a[0], b[1], -(a[1] * b[0]));
}

// ------------------------------------------------------------------ K2: plane fit, gates, point-wise uncertainty
// Eigen::ColPivHouseholderQR<Matrix<float,5,3>>::solve(b) with b = -1 (common_lib.h:156-157,174), float, no FMA.
__device__ __forceinline__ void qr_solve_5x3(float A[5][3], float x[3]) {
  const float eps = 1.1920928955078125e-07f;   // FLT_EPSILON
  float hC[3] = {0.f, 0.f, 0.f};
  int perm[3] = {0, 1, 2};
  float nU[3], nD[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) s += A[i][k] * A[i][k];
    nD[k] = sqrtf(s);
    nU[k] = nD[k];
  }
  const float maxn = fmaxf(nU[0], fmaxf(nU[1], nU[2]));
  const float threshold_helper = (maxn * eps) * (maxn * eps) / 5.0f;
  const float downdate_thr = sqrtf(eps);
  int nonzero = 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int biggest = k;
#pragma unroll
    for (int j = k + 1; j < 3; ++j) {
      float cur = nU[k];
#pragma unroll
      for (int jj = k + 1; jj < 3; ++jj) if (biggest == jj) cur = nU[jj];
      if (nU[j] > cur) biggest = j;
    }
    float bn = nU[k];
#pragma unroll
    for (int jj = k + 1; jj < 3; ++jj) if (biggest == jj) bn = nU[jj];
    if (nonzero == 3 && bn * bn < threshold_helper * (float)(5 - k)) nonzero = k;
#pragma unroll
    for (int j = k + 1; j < 3; ++j) {
      if (biggest == j) {
#pragma unroll
        for (int i = 0; i < 5; ++i) { float t = A[i][k]; A[i][k] = A[i][j]; A[i][j] = t; }
        float t = nU[k]; nU[k] = nU[j]; nU[j] = t;
        t = nD[k]; nD[k] = nD[j]; nD[j] = t;
        int ti = perm[k]; perm[k] = perm[j]; perm[j] = ti;
      }
    }
    float tailSq = 0.f;
#pragma unroll
    for (int i = k + 1; i < 5; ++i) tailSq += A[i][k] * A[i][k];
    const float c0 = A[k][k];
    float beta, tau;
    if (tailSq <= 1.17549435e-38f) {   // numeric_limits<float>::min()
      tau = 0.f; beta = c0;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) A[i][k] = 0.f;
    } else {
      beta = sqrtf(c0 * c0 + tailSq);
      if (c0 >= 0.f) beta = -beta;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) A[i][k] = A[i][k] / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    A[k][k] = beta;
    hC[k] = tau;
    if (tau != 0.f) {
#pragma unroll
      for (int j = k + 1; j < 3; ++j) {
        float tmp = 0.f;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) tmp += A[i][k] * A[i][j];
        tmp += A[k][j];
        A[k][j] -= tau * tmp;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) A[i][j] -= tau * A[i][k] * tmp;
      }
    }
#pragma unroll
    for (int j = k + 1; j < 3; ++j) {
      if (nU[j] != 0.f) {
        float temp = fabsf(A[k][j]) / nU[j];
        temp = (1.f + temp) * (1.f - temp);
        temp = temp < 0.f ? 0.f : temp;
        const float r = nU[j] / nD[j];
        const float temp2 = temp * r * r;
        if (temp2 <= downdate_thr) {
          float s = 0.f;
#pragma unroll
          for (int i = k + 1; i < 5; ++i) s += A[i][j] * A[i][j];
          nD[j] = sqrtf(s);
          nU[j] = nD[j];
        } else {
          nU[j] *= sqrtf(temp);
        }
      }
    }
  }
  float c[5] = {-1.f, -1.f, -1.f, -1.f, -1.f};
  x[0] = x[1] = x[2] = 0.f;
  if (nonzero == 0) return;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (k < nonzero && hC[k] != 0.f) {
      float tmp = 0.f;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) tmp += A[i][k] * c[i];
      tmp += c[k];
      c[k] -= hC[k] * tmp;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) c[i] -= hC[k] * A[i][k] * tmp;
    }
  }
#pragma unroll
  for (int i = 2; i >= 0; --i) {
    if (i < nonzero) {
      float s = c[i];
#pragma unroll
      for (int j = i + 1; j < 3; ++j) if (j < nonzero) s -= A[i][j] * c[j];
      c[i] = s / A[i][i];
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < nonzero) {
#pragma unroll
      for (int q = 0; q < 3; ++q) if (perm[i] == q) x[q] = c[i];
    }
  }
}

// trace of evalPointUncertainty's 3x3 (associate_uct.hpp:153-175) in closed form:
//   G = [ q_w I | -[q]x | T(0:3,0:3) ], q = T (0.05 p, 1);  Sigma_in = blkdiag(1e4 cov, 0.1 I)
//   trace = sum_{i<3} (F (1e4 cov) F^T)_ii + 0.1 |T(0:3,0:3)|_F^2,  F = [ q_w I | -[q]x ]
// Row i of F has three non-zeros, so (F S F^T)_ii is a 3x3 quadratic form: 27 terms instead of the dense 9x9
// product.  `e` is one table entry as uploaded: T (16) then cov (36).
__device__ __forceinline__ double point_cov_trace(float px, float py, float pz, const double* __restrict__ e) {
  const double pc0 = px * 0.05, pc1 = py * 0.05, pc2 = pz * 0.05;
  double q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = e[4 * i] * pc0 + e[4 * i + 1] * pc1 + e[4 * i + 2] * pc2 + e[4 * i + 3] * 1.0;
  const double* cov = e + 16;
  // non-zero columns / values of the rows of F = [q3 I | -skew(q)]
  const int col[3][3] = {{0, 4, 5}, {1, 3, 5}, {2, 3, 4}};
  const double val[3][3] = {{q[3], q[2], -q[1]}, {q[3], -q[2], q[0]}, {q[3], q[1], -q[0]}};
  double tr = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      double m = 0.0;
#pragma unroll
      for (int b = 0; b < 3; ++b) m += val[i][b] * (cov[6 * col[i][b] + col[i][a]] * 10000.0);
      tr += m * val[i][a];
    }
  }
  double fro = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) fro += (e[4 * i + j] * 0.1) * e[4 * i + j];
  return tr + fro;
}

struct MinMax4 { double umin, umax, tmin, tmax; uint32_t cnt; };

__device__ __forceinline__ MinMax4 warp_reduce(MinMax4 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.umin = fmin(v.umin, __shfl_xor_sync(0xffffffffu, v.umin, o));
    v.umax = fmax(v.umax, __shfl_xor_sync(0xffffffffu, v.umax, o));
    v.tmin = fmin(v.tmin, __shfl_xor_sync(0xffffffffu, v.tmin, o));
    v.tmax = fmax(v.tmax, __shfl_xor_sync(0xffffffffu, v.tmax, o));
    v.cnt += __shfl_xor_sync(0xffffffffu, v.cnt, o);
  }
  return v;
}

// ---- K2a (search passes only): plane fit of the 5 neighbours.  esti_plane depends on the neighbours alone, not on
// the state, so its result is computed once per search and reused by the passes that re-use Nearest_Points
// (the reference recomputes it every pass, laserMapping.cpp:596, with the same outcome).
//   plane[p] = (n_x, n_y, n_z, d) ;  ucov[p] = plane_cov ;  sel[p] &= plane ok
__device__ __forceinline__ void fit_point(const float4* __restrict__ nodes, const float* __restrict__ node_cov, uint32_t N,
                                          const ParamConst& prm, const uint32_t* __restrict__ nn_idx,
                                          uint8_t* __restrict__ sel, float4* __restrict__ plane,
                                          double* __restrict__ ucov, uint32_t p) {
  float A[5][3], W[5];
#pragma unroll
  for (int j = 0; j < MALIO_K; ++j) {
    const uint32_t idx = nn_idx[(size_t)j * N + p];
    const float4 a = __ldg(nodes + idx);   // compact mirror of the snapshot: 16 B stride
    A[j][0] = a.x; A[j][1] = a.y; A[j][2] = a.z;
    W[j] = __ldg(node_cov + idx);
  }
  // esti_plane (common_lib.h:144-190)
  double cov_sum = 0.0, unit_cov = 0.0;
#pragma unroll
  for (int j = 0; j < MALIO_K; ++j) cov_sum += fabs(prm.cov_threshold - (double)W[j]);
  if ((double)W[0] > 0.00001) {
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j)
      unit_cov += ((prm.cov_threshold - (double)W[j]) / cov_sum) * ((prm.cov_threshold - (double)W[j]) / cov_sum) * (double)W[j];
  }
  float Aq[5][3];
#pragma unroll
  for (int j = 0; j < 5; ++j) { Aq[j][0] = A[j][0]; Aq[j][1] = A[j][1]; Aq[j][2] = A[j][2]; }
  float nv[3];
  qr_solve_5x3(Aq, nv);
  const float n = sqrtf(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
  const float pa = nv[0] / n, pb = nv[1] / n, pcn = nv[2] / n;
  const float pd = (float)(1.0 / (double)n);
  bool ok = true;
#pragma unroll
  for (int j = 0; j < MALIO_K; ++j)
    if (fabsf(pa * A[j][0] + pb * A[j][1] + pcn * A[j][2] + pd) > prm.plane_th) ok = false;
  plane[p] = make_float4(pa, pb, pcn, pd);
  ucov[p] = unit_cov;
  if (!ok) sel[p] = 0;
}
__global__ void __launch_bounds__(PLANE_THREADS)
fit_kernel(const float4* __restrict__ nodes, const float* __restrict__ node_cov, uint32_t N, ParamConst prm,
           const uint32_t* __restrict__ nn_idx, uint8_t* __restrict__ sel, float4* __restrict__ plane,
           double* __restrict__ ucov) {
  const uint32_t p = blockIdx.x * PLANE_THREADS + threadIdx.x;
  if (p >= N || !sel[p]) return;
  fit_point(nodes, node_cov, N, prm, nn_idx, sel, plane, ucov, p);
}

// ---- K2b (once per scan): point-wise uncertainty.  evalPointUncertainty depends on the point and its table entry
// only; the entry index is clamped differently for selected (:694-696) and non-selected (:737-739) points, so both
// traces are kept:  tau2[p] = (tau_selected, tau_not_selected).
__device__ __forceinline__ void tau_point(const malio_scan_pt& pt, const PassConst& pc, const double* __restrict__ table,
                                          double2* __restrict__ tau2, uint32_t p) {
  const int lid = pt.lidar;
  const int tsize = (int)(pc.table_off[lid + 1] - pc.table_off[lid]);
  const int ti = (int)pt.table_idx;
  const int ti_sel = (ti >= tsize) ? tsize - 2 : ti;
  const int ti_non = (ti >= tsize - 1) ? tsize - 2 : ti;
  const double t_sel = point_cov_trace(pt.x, pt.y, pt.z, table + (size_t)(pc.table_off[lid] + ti_sel) * TABLE_DOUBLES);
  const double t_non = (ti_non == ti_sel) ? t_sel
                       : point_cov_trace(pt.x, pt.y, pt.z, table + (size_t)(pc.table_off[lid] + ti_non) * TABLE_DOUBLES);
  tau2[p] = make_double2(t_sel, t_non);
}
__global__ void __launch_bounds__(PLANE_THREADS)
tau_kernel(const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm, uint32_t N, PassConst pc,
           const double* __restrict__ table, double2* __restrict__ tau2) {
  const uint32_t p = blockIdx.x * PLANE_THREADS + threadIdx.x;
  if (p >= N) return;
  const malio_scan_pt pt = pts[perm ? perm[p] : p];
  tau_point(pt, pc, table, tau2, p);
}

// ---- K2c (every pass): transform, point-to-plane residual, residual gate, min/max of the two weights.
// d_mmkey layout: dkey of {min_u, -max_u, min_tau, -max_tau}: one (integer) MIN all-reduce serves all four
struct GateOut { double u, tau; float pd2; int lid; bool selected; };
// one point of the gate: returns its contribution to the min/max of the two weights in mm
__device__ __forceinline__ void gate_point(const malio_scan_pt& pt, uint32_t p, const PassConst& pc,
                                           const float4* __restrict__ plane, const double* __restrict__ ucov,
                                           const double2* __restrict__ tau2, uint8_t* __restrict__ sel,
                                           float4* __restrict__ world, float* __restrict__ pd2_out, double* __restrict__ tau,
                                           float* __restrict__ normal_y, double* __restrict__ rows12,
                                           uint8_t* __restrict__ lid8, MinMax4& mm, double* __restrict__ srow = nullptr,
                                           GateOut* __restrict__ go = nullptr) {
  double b[3], m[3], g[3];
  transform_point(pc, pt.x, pt.y, pt.z, pt.lidar, b, m, g);
  const float wx = (float)g[0], wy = (float)g[1], wz = (float)g[2];
  world[p] = make_float4(wx, wy, wz, 0.f);
  bool selected = sel[p] != 0;
  if (selected) {
    const float4 pl = plane[p];
    const float pd2 = pl.x * wx + pl.y * wy + pl.z * wz + pl.w;                  // laserMapping.cpp:598
    const double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
    const float s = (float)(1 - 0.9 * (double)fabsf(pd2) / sqrt(nb));           // :599
    selected = (double)s > 0.1;
    pd2_out[p] = pd2;
    if (!selected) sel[p] = 0;
    if (selected) {
      // un-weighted Jacobian row, compact: [ n | A | B | C ]  (laserMapping.cpp:665-693)
      const int lid = pt.lidar;
      const double nvec[3] = {(double)pl.x, (double)pl.y, (double)pl.z};
      // C0 = R(s.rot)^T n (:676);  A = [m]x C0 (:677);  l = 0: C = C0, B = [b]x R(qE0)^T C (:683-684);
      // l != 0: C = R(qC_l)^T C0, B = [p]x R(qE_l)^T C (:687-690).  [v]x (R C) = v x (R C): evaluated as matrix-vector
      // products and cross products with FMAs — equal to the reference's (skew * R) * C to rounding (bar: 1e-9 on the system)
      double C[3], A[3], B[3] = {0.0, 0.0, 0.0};
      mat3_mul(pc.RsT, nvec, C);
      cross3_fma(m, C, A);
      double Cc[3] = {0.0, 0.0, 0.0};
      if (pc.ext_en) {
        double w[3];
        if (lid == 0) {
          mat3_mul(pc.ReT[0], C, w);
          cross3_fma(b, w, B);
        } else {
          double C2[3];
          mat3_mul(pc.RcT[lid], C, C2);
          C[0] = C2[0]; C[1] = C2[1]; C[2] = C2[2];
          mat3_mul(pc.ReT[lid], C, w);
          const double v[3] = {(double)pt.x, (double)pt.y, (double)pt.z};
          cross3_fma(v, w, B);
        }
        Cc[0] = C[0]; Cc[1] = C[1]; Cc[2] = C[2];
      }
      double2* dst = reinterpret_cast<double2*>(rows12 + (size_t)p * 12);
      dst[0] = make_double2(nvec[0], nvec[1]); dst[1] = make_double2(nvec[2], A[0]); dst[2] = make_double2(A[1], A[2]);
      dst[3] = make_double2(B[0], B[1]);       dst[4] = make_double2(B[2], Cc[0]);   dst[5] = make_double2(Cc[1], Cc[2]);
      lid8[p] = (uint8_t)lid;
      if (srow) {   // the fused pass keeps the row on chip across the min/max barrier
        srow[0] = nvec[0]; srow[1] = nvec[1]; srow[2] = nvec[2]; srow[3] = A[0]; srow[4] = A[1]; srow[5] = A[2];
        srow[6] = B[0]; srow[7] = B[1]; srow[8] = B[2]; srow[9] = Cc[0]; srow[10] = Cc[1]; srow[11] = Cc[2];
      }
      if (go) go->pd2 = pd2;
    }
  }
  const double2 t2 = tau2[p];
  if (go) { go->selected = selected; go->lid = pt.lidar; go->u = selected ? ucov[p] : 0.0; go->tau = t2.x; }
  if (selected) {
    const double u = ucov[p];
    mm.umin = fmin(mm.umin, u); mm.umax = fmax(mm.umax, u); mm.cnt += 1;
    if (pc.ext_en) {   // :694-703; with extrinsic_est_en == false R and normal_y are left untouched
      tau[p] = t2.x;
      normal_y[p] = (float)t2.x;
      mm.tmin = fmin(mm.tmin, t2.x); mm.tmax = fmax(mm.tmax, t2.x);
    }
  } else {
    normal_y[p] = (float)t2.y;   // :735-741
  }
}
// block-level min/max, then one integer atomicMin per quantity and block on the order-preserving keys:
// min/max are exact under any ordering, so this is deterministic without a serial fold.
template <int THREADS>
__device__ __forceinline__ void minmax_block_commit(MinMax4 mm, unsigned long long* __restrict__ d_mmkey) {
  __shared__ MinMax4 s_w[THREADS / 32];
  mm = warp_reduce(mm);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = mm;
  __syncthreads();
  if (threadIdx.x == 0) {
    MinMax4 r = s_w[0];
    for (int w = 1; w < THREADS / 32; ++w) {
      r.umin = fmin(r.umin, s_w[w].umin); r.umax = fmax(r.umax, s_w[w].umax);
      r.tmin = fmin(r.tmin, s_w[w].tmin); r.tmax = fmax(r.tmax, s_w[w].tmax);
      r.cnt += s_w[w].cnt;
    }
    if (r.cnt) {
      atomicMin(d_mmkey + 0, dkey(r.umin)); atomicMin(d_mmkey + 1, dkey(-r.umax));
      atomicMin(d_mmkey + 2, dkey(r.tmin)); atomicMin(d_mmkey + 3, dkey(-r.tmax));
    }
  }
}
__global__ void __launch_bounds__(GATE_THREADS)
gate_kernel(const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm, uint32_t N, PassConst pc,
            const float4* __restrict__ plane, const double* __restrict__ ucov, const double2* __restrict__ tau2,
            uint8_t* __restrict__ sel, float4* __restrict__ world, float* __restrict__ pd2_out,
            double* __restrict__ tau, float* __restrict__ normal_y, double* __restrict__ rows12,
            uint8_t* __restrict__ lid8, unsigned long long* __restrict__ d_mmkey) {
  const uint32_t p = blockIdx.x * GATE_THREADS + threadIdx.x;
  MinMax4 mm{1000.0, 0.0, 9999.0, 0.0, 0u};   // laserMapping.cpp:615-616, 646-647
  if (p < N) {
    const malio_scan_pt pt = pts[perm ? perm[p] : p];
    gate_point(pt, p, pc, plane, ucov, tau2, sel, world, pd2_out, tau, normal_y, rows12, lid8, mm);
  }
  minmax_block_commit<GATE_THREADS>(mm, d_mmkey);
}

// ------------------------------------------------------------------ K3: weights + fused H^T R^-1 [H | h] reduction
// The gate kernel leaves, per selected point, the un-weighted Jacobian row in compact form
//   J12 = [ n | [m]x C0 | B | C ]     (laserMapping.cpp:665-693; 12 of the 24 columns are non-zero)
// and the LiDAR id that says where B and C sit (columns 6+3l and 6+3(L+l)).  Here each row gets its plane weight
// a_i (:651-656) and noise rho_i (:716-721, clamp esekfom.hpp:624-626) and the block accumulates, per LiDAR l,
//     Gc_l = sum_{i in l} (a J12 / rho^)_a * [ a J12 | z | rho^ a J12_0..2 ]_b          (12 x 16, upper 4x4 blocks)
// i.e. esekfom.hpp:622-635 restricted to the non-zero columns (3.7x fewer FP64 operations than the dense 24 x 28
// form; FP64 issue is the limiter of this kernel).  The host scatters the three compact systems into the c x c one.
// The localization weight (a scalar, :745-759) factors out and is applied on the host.
__device__ __forceinline__ void point_weights(const ParamConst& prm, double u, double tau_i, int ext_en,
                                              double umin, double umax, double tmin, double tmax,
                                              double& a, double& rho) {
  // :651-656
  a = u;
  if (a == 0) a = 1;
  else if (umax == umin) a = (prm.plane_cov_max + prm.plane_cov_min) / 2;
  else a = 1 / ((prm.plane_cov_max - prm.plane_cov_min) * (a - umin) / (umax - umin) + prm.plane_cov_min);
  // :716-721 (FIC).  Degenerate 0/0 defined as mid-range (the reference yields NaN; SURVEY.md quirk 8)
  double R = ext_en ? tau_i : 0.0;
  if (R < tmin + (tmax - tmin) * prm.range_min) R = prm.point_cov_min;
  else if (R > tmin + (tmax - tmin) * prm.range_max) R = prm.point_cov_max;
  else {
    const double den = (prm.range_max - prm.range_min) * (tmax - tmin);
    if (den == 0.0) R = (prm.point_cov_max + prm.point_cov_min) / 2;
    else R = (prm.point_cov_max - prm.point_cov_min) * (R - (tmin + (tmax - tmin) * prm.range_min)) / den + prm.point_cov_min;
  }
  if (R < 0.0001) R = 0.001;   // esekfom.hpp:624-626
  rho = R;
}

// task t (0..8) -> upper-triangular 4x4 block (row group gi < 3, col group gj >= gi, gj < 4) of a 12 x 16 system
__device__ __forceinline__ void red_task(int t, int& gi, int& gj) {
  gi = (t >= 4) + (t >= 7);
  gj = t - (gi == 0 ? 0 : (gi == 1 ? 3 : 5));
}

// The body of the reduction for one block: tiles [tile_begin, tile_end) (contiguous, so that with the LiDAR-major
// internal order a block sees one LiDAR for many tiles), result in the block's slot.  Each of the 126 worker threads
// owns one 4x4 block (task) of the compact 12 x 16 system and every RED_KS-th row; its 16 accumulators stay in
// registers for as long as the LiDAR does not change and are folded over the row-splits (fixed order) into the slot
// only then.
__device__ __forceinline__ void reduce_flush(const double acc[16], bool worker, int l, double* __restrict__ s_flush,
                                             double* __restrict__ slot) {
  if (worker) {
#pragma unroll
    for (int k = 0; k < 16; ++k) s_flush[k * (RED_TASKS * RED_KS) + threadIdx.x] = acc[k];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < RED_TASKS * 16; e += RED_THREADS) {
    const int tk = e / 16, k = e % 16;
    double sum = 0.0;
#pragma unroll
    for (int q = 0; q < RED_KS; ++q) sum += s_flush[k * (RED_TASKS * RED_KS) + tk * RED_KS + q];
    slot[(l * RED_TASKS + tk) * 16 + k] += sum;
  }
  __syncthreads();
}
__device__ __forceinline__ void reduce_block(uint32_t N, const ParamConst& prm, int ext_en, const uint8_t* __restrict__ sel,
                                             const uint8_t* __restrict__ lid8, const double* __restrict__ rows12,
                                             const float* __restrict__ pd2v, const double* __restrict__ ucov,
                                             const double* __restrict__ tau, const unsigned long long* __restrict__ d_mm,
                                             uint32_t tile_begin, uint32_t tile_end, double* __restrict__ slot) {
  extern __shared__ double smem[];
  double* s_hs = smem;                                       // [128][RED_HS_STRIDE]  a J12 / rho^
  double* s_hx = s_hs + RED_THREADS * RED_HS_STRIDE;         // [128][RED_HX_STRIDE]  [a J12 | z | rho^ a J12_0..2]
  double* s_flush = s_hx + RED_THREADS * RED_HX_STRIDE;      // [16][RED_TASKS * RED_KS]  (entry-major: conflict-free)
  __shared__ uint32_t s_wcnt[MALIO_MAX_LIDAR][RED_THREADS / 32];
  __shared__ uint32_t s_seg[MALIO_MAX_LIDAR + 1];
  const int task = threadIdx.x / RED_KS, ks = threadIdx.x % RED_KS;
  const bool worker = task < RED_TASKS;
  int gi = 0, gj = 0;
  if (worker) red_task(task, gi, gj);
  for (int e = threadIdx.x; e < MALIO_RED_DOUBLES; e += RED_THREADS) slot[e] = 0.0;
  const double umin = dkey_inv(d_mm[0]), umax = -dkey_inv(d_mm[1]), tmin = dkey_inv(d_mm[2]), tmax = -dkey_inv(d_mm[3]);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t cnt_total = 0;
  int cur_l = -1;            // block-uniform: every thread derives it from s_seg
  double acc[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) acc[k] = 0.0;
  __syncthreads();
  for (uint32_t tile = tile_begin; tile < tile_end; ++tile) {
    // ---- phase A: weight this thread's row, then place it in the tile's LiDAR-sorted order
    const uint32_t p = tile * RED_THREADS + threadIdx.x;
    const bool ok = (p < N) && sel[p];
    const int l = ok ? (int)lid8[p] : -1;
    double h[12], z = 0.0, rho = 1.0, a = 0.0;
    if (ok) {
      point_weights(prm, ucov[p], ext_en ? tau[p] : 0.0, ext_en, umin, umax, tmin, tmax, a, rho);
      const double2* src = reinterpret_cast<const double2*>(rows12 + (size_t)p * 12);
#pragma unroll
      for (int k = 0; k < 6; ++k) { const double2 v = src[k]; h[2 * k] = v.x * a; h[2 * k + 1] = v.y * a; }   // :714
      z = ((-1) * (double)pd2v[p]) * a;                                                                  // :707,715
    }
    const uint32_t b0 = __ballot_sync(0xffffffffu, l == 0), b1 = __ballot_sync(0xffffffffu, l == 1),
                   b2 = __ballot_sync(0xffffffffu, l == 2);
    if (lane == 0) { s_wcnt[0][wid] = __popc(b0); s_wcnt[1][wid] = __popc(b1); s_wcnt[2][wid] = __popc(b2); }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t run = 0;
      for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
        s_seg[ll] = run;
        for (int w = 0; w < RED_THREADS / 32; ++w) { const uint32_t c = s_wcnt[ll][w]; s_wcnt[ll][w] = run; run += c; }
      }
      s_seg[MALIO_MAX_LIDAR] = run;
    }
    __syncthreads();
    if (ok) {
      const uint32_t bal = l == 0 ? b0 : (l == 1 ? b1 : b2);
      const uint32_t dst = s_wcnt[l][wid] + __popc(bal & ((1u << lane) - 1u));
      double* hs = s_hs + dst * RED_HS_STRIDE;
      double* hx = s_hx + dst * RED_HX_STRIDE;
      const double inv_rho = 1.0 / rho;   // HT(:,i) / R_i (esekfom.hpp:627) as a multiply: <= 1 ulp per term
#pragma unroll
      for (int k = 0; k < 12; ++k) { hs[k] = h[k] * inv_rho; hx[k] = h[k]; }
      hx[12] = z; hx[13] = rho * h[0]; hx[14] = rho * h[1]; hx[15] = rho * h[2];
    }
    __syncthreads();
    cnt_total += s_seg[MALIO_MAX_LIDAR];
    // ---- phase B: per LiDAR segment, 9 block tasks x RED_KS row-splits
#pragma unroll 1
    for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
      const uint32_t beg = s_seg[ll], end = s_seg[ll + 1];
      if (beg == end) continue;
      if (ll != cur_l) {
        if (cur_l >= 0) reduce_flush(acc, worker, cur_l, s_flush, slot);
        cur_l = ll;
#pragma unroll
        for (int k = 0; k < 16; ++k) acc[k] = 0.0;
      }
      if (worker) {
        for (uint32_t q = beg + ks; q < end; q += RED_KS) {
          const double* aa = s_hs + q * RED_HS_STRIDE + 4 * gi;
          const double* bb = s_hx + q * RED_HX_STRIDE + 4 * gj;
          const double a0 = aa[0], a1 = aa[1], a2 = aa[2], a3 = aa[3];
          const double c0 = bb[0], c1 = bb[1], c2 = bb[2], c3 = bb[3];
          acc[0] = fma(a0, c0, acc[0]);   acc[1] = fma(a0, c1, acc[1]);   acc[2] = fma(a0, c2, acc[2]);   acc[3] = fma(a0, c3, acc[3]);
          acc[4] = fma(a1, c0, acc[4]);   acc[5] = fma(a1, c1, acc[5]);   acc[6] = fma(a1, c2, acc[6]);   acc[7] = fma(a1, c3, acc[7]);
          acc[8] = fma(a2, c0, acc[8]);   acc[9] = fma(a2, c1, acc[9]);   acc[10] = fma(a2, c2, acc[10]); acc[11] = fma(a2, c3, acc[11]);
          acc[12] = fma(a3, c0, acc[12]); acc[13] = fma(a3, c1, acc[13]); acc[14] = fma(a3, c2, acc[14]); acc[15] = fma(a3, c3, acc[15]);
        }
      }
    }
    __syncthreads();   // the staging area is rewritten by the next tile
  }
  if (cur_l >= 0) reduce_flush(acc, worker, cur_l, s_flush, slot);
  if (threadIdx.x == 0) { slot[MALIO_RED_BLOCKS * 16] = (double)cnt_total; slot[MALIO_RED_BLOCKS * 16 + 1] = 0.0; }
}
// contiguous tile range of block b when n_tiles are dealt to `grid` blocks (the host picks grid = ceil(n_tiles / per_block))
__device__ __forceinline__ void block_tiles(uint32_t n_tiles, uint32_t& t0, uint32_t& t1) {
  const uint32_t per_block = (n_tiles + gridDim.x - 1) / gridDim.x;
  t0 = blockIdx.x * per_block;
  t1 = t0 + per_block < n_tiles ? t0 + per_block : n_tiles;
  if (t0 > n_tiles) t0 = n_tiles;
}
__global__ void __launch_bounds__(RED_THREADS)
reduce_kernel(uint32_t N, ParamConst prm, int ext_en, const uint8_t* __restrict__ sel, const uint8_t* __restrict__ lid8,
              const double* __restrict__ rows12, const float* __restrict__ pd2v, const double* __restrict__ ucov,
              const double* __restrict__ tau, const unsigned long long* __restrict__ d_mm, uint32_t n_tiles,
              double* __restrict__ block_red) {
  uint32_t t0, t1;
  block_tiles(n_tiles, t0, t1);
  reduce_block(N, prm, ext_en, sel, lid8, rows12, pd2v, ucov, tau, d_mm, t0, t1, block_red + (size_t)blockIdx.x * MALIO_RED_DOUBLES);
}

// ------------------------------------------------------------------ one measurement pass in ONE cooperative launch
// K2 + K3 fused (single-GPU path):  [tau once per scan] [plane fit once per search] gate -> grid barrier -> weights +
// H^T R^-1 [H|h] accumulation -> grid barrier -> distributed fixed-order fold, written both to device memory and straight
// into pinned, mapped host memory, followed by a sequence flag the host spins on.  Compared with the three launches +
// D2H copy + stream synchronisation it replaces, this removes every launch gap and the copy/sync latency from the
// per-pass critical path; arithmetic and summation order are unchanged (bit-identical results).
// The kernel is launched with cudaLaunchCooperativeKernel (all blocks co-resident), the barriers are plain
// device-scope counters that only ever grow (the host passes the value they had before the launch).
// Multi-GPU: the two exchanges of a pass (MIN of the four min/max keys before the weights, SUM of the reduced system at
// the end) go through per-rank mailboxes in device memory that every peer maps with CUDA IPC and writes over
// NVLink/NVSwitch from inside pass_kernel — no NCCL call, no extra launch, the cross-GPU latency of a pass is two
// one-way store + flag hops.  Layout of one rank's mailbox: [parity 2][kind: MIN 64 B | SUM 3584 B][source rank 8].
struct PeerArgs {
  unsigned char* mail[MAIL_MAX_WORLD];   // mail[r] = rank r's mailbox as mapped into THIS process (mail[rank] is local)
  int rank, world;
};
__device__ __forceinline__ unsigned char* mail_min_slot(unsigned char* box, uint32_t seq, int src) {
  return box + (seq & 1u) * MAIL_PARITY_BYTES + src * MAIL_MIN_BYTES;
}
__device__ __forceinline__ unsigned char* mail_sum_slot(unsigned char* box, uint32_t seq, int src) {
  return box + (seq & 1u) * MAIL_PARITY_BYTES + MAIL_MAX_WORLD * MAIL_MIN_BYTES + src * MAIL_SUM_BYTES;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// spin until *p == want; gives up after ~2 s (a peer that never launched) and reports it
__device__ __forceinline__ bool wait_seq_sys(const uint32_t* p, uint32_t want) {
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (uint32_t it = 0;; ++it) {
    if (ld_acquire_sys_u32(p) == want) return true;
    if ((it & 0xFFFu) == 0xFFFu) {
      unsigned long long t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > 2000000000ull) return false;
    }
  }
}
struct PassArgs {
  const malio_scan_pt* pts; const uint32_t* perm; uint32_t N;
  const double* table; const float4* nodes; const float* node_cov; const uint32_t* nn_idx;
  uint8_t* sel; float4* world; float4* plane; double* ucov; double2* tau2; float* pd2; double* tau; float* normal_y;
  double* rows12; uint8_t* lid8;
  int do_tau, do_fit;
  unsigned long long *mmkey, *mmkey_next; uint32_t* gstats;
  uint32_t* bar;           // [0] barrier 1 arrivals, [1] barrier 2 arrivals, [2] folded entries  (monotone), [3] release flag of barrier 1 (multi-GPU)
  PeerArgs peer;
  uint32_t bar_base[3];
  uint32_t n_tiles;
  double* block_red; double* d_res;
  double* h_res;           // mapped host memory: MALIO_RED_DOUBLES result | 4 min/max keys | flag
  uint32_t seq;
  unsigned long long* dbg; // optional [grid][8] %globaltimer stamps at the phase boundaries (MALIO_PASS_TRACE=1)
  unsigned long long* xwait;   // multi-GPU: [0] ns spent in the MIN exchange (push + wait for every peer), [1] same for the SUM exchange, [2] passes
};
__device__ __forceinline__ void pass_stamp(const PassArgs& a, int k) {
  if (a.dbg && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    a.dbg[(size_t)blockIdx.x * 8 + k] = t;
  }
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// all threads of all blocks call this; returns when `expected` arrivals have been counted
// Gives up after ~2 s (a block of the grid that never became resident) and raises the fault word of the mapped result buffer,
// which measure() reports.
__device__ __forceinline__ void grid_barrier(uint32_t* counter, uint32_t target, uint32_t* fault) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned long long t0 = 0;
    for (uint32_t it = 0; (int32_t)(ld_acquire_u32(counter) - target) < 0; ++it) {
      if ((it & 0x3FFFu) == 0x3FFFu) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t0 == 0) t0 = t1;
        else if (t1 - t0 > 2000000000ull) { *reinterpret_cast<volatile uint32_t*>(fault) = 2u; break; }
      }
    }
  }
  __syncthreads();
}
// FAST: every block owns at most PASS_FAST_TILES tiles and keeps their Jacobian rows in shared memory from the gate to
// the accumulation (no global round trip, no staging pass); rows stay in their own positions and the workers pick the
// rows of the LiDAR they are accumulating by a per-row tag, so no prefix sums or compaction barriers are needed.
// !FAST: any number of tiles per block, rows go through global memory (reduce_block).
#ifndef MALIO_PASS_TILES
#define MALIO_PASS_TILES 2
#endif
#ifndef MALIO_PASS_MINB
#define MALIO_PASS_MINB 4
#endif
constexpr int PASS_FAST_TILES = MALIO_PASS_TILES;   // tiles of 128 points a block keeps on chip (fast path)
constexpr int PASS_MIN_BLOCKS = MALIO_PASS_MINB;    // co-resident blocks per SM the kernel is compiled for
constexpr int PASS_ROW_STRIDE = 15;        // doubles per staged row: a*J12 (12) | 1/rho^ | z | rho^   (odd: conflict-free)
constexpr int PASS_FAST_SMEM_DOUBLES = PASS_FAST_TILES * RED_THREADS * PASS_ROW_STRIDE + RED_TASKS * RED_KS * 16;
static_assert(PASS_FAST_SMEM_DOUBLES <= RED_SMEM_DOUBLES, "the fast path must fit the generic path's shared memory");
template <bool FAST>
__global__ void __launch_bounds__(RED_THREADS, FAST ? PASS_MIN_BLOCKS : 4)
pass_kernel(PassArgs a, PassConst pc, ParamConst prm) {
  uint32_t t0, t1;
  block_tiles(a.n_tiles, t0, t1);
  extern __shared__ double smem[];
  // FAST: rows stay in their own slots; per (tile, LiDAR) the slots that hold a row are listed (compacted) so that the
  // accumulation loop runs over rows of one LiDAR only, every lane busy
  __shared__ uint8_t s_list[PASS_FAST_TILES * RED_THREADS];
  __shared__ uint16_t s_wc[PASS_FAST_TILES][MALIO_MAX_LIDAR][RED_THREADS / 32];   // selected rows per tile, LiDAR, warp
  GateOut go[PASS_FAST_TILES];
  uint32_t bal[PASS_FAST_TILES];   // ballot of this thread's LiDAR within its warp (FAST)
  pass_stamp(a, 0);
  // ---- phase 1: per point, same tile -> block mapping as the accumulation below
  {
    MinMax4 mm{1000.0, 0.0, 9999.0, 0.0, 0u};   // laserMapping.cpp:615-616, 646-647
#pragma unroll
    for (int k = 0; k < (FAST ? PASS_FAST_TILES : 1); ++k) go[k].selected = false;
    if (FAST) {
#pragma unroll
      for (int k = 0; k < PASS_FAST_TILES; ++k) {
        const uint32_t tile = t0 + k;
        const uint32_t p = tile * RED_THREADS + threadIdx.x;
        if (tile < t1 && p < a.N) {
          const malio_scan_pt pt = a.pts[a.perm ? a.perm[p] : p];
          if (a.do_tau) tau_point(pt, pc, a.table, a.tau2, p);
          if (a.do_fit && a.sel[p]) fit_point(a.nodes, a.node_cov, a.N, prm, a.nn_idx, a.sel, a.plane, a.ucov, p);
          gate_point(pt, p, pc, a.plane, a.ucov, a.tau2, a.sel, a.world, a.pd2, a.tau, a.normal_y, a.rows12, a.lid8, mm,
                     smem + (size_t)(k * RED_THREADS + threadIdx.x) * PASS_ROW_STRIDE, &go[k]);
        }
        const int l = go[k].selected ? go[k].lid : -1;
        const uint32_t b0 = __ballot_sync(0xffffffffu, l == 0), b1 = __ballot_sync(0xffffffffu, l == 1),
                       b2 = __ballot_sync(0xffffffffu, l == 2);
        bal[k] = l == 0 ? b0 : (l == 1 ? b1 : b2);
        if ((threadIdx.x & 31) == 0) {
          s_wc[k][0][threadIdx.x >> 5] = (uint16_t)__popc(b0); s_wc[k][1][threadIdx.x >> 5] = (uint16_t)__popc(b1);
          s_wc[k][2][threadIdx.x >> 5] = (uint16_t)__popc(b2);
        }
      }
    } else {
      for (uint32_t tile = t0; tile < t1; ++tile) {
        const uint32_t p = tile * RED_THREADS + threadIdx.x;
        if (p < a.N) {
          const malio_scan_pt pt = a.pts[a.perm ? a.perm[p] : p];
          if (a.do_tau) tau_point(pt, pc, a.table, a.tau2, p);
          if (a.do_fit && a.sel[p]) fit_point(a.nodes, a.node_cov, a.N, prm, a.nn_idx, a.sel, a.plane, a.ucov, p);
          gate_point(pt, p, pc, a.plane, a.ucov, a.tau2, a.sel, a.world, a.pd2, a.tau, a.normal_y, a.rows12, a.lid8, mm);
        }
      }
    }
    minmax_block_commit<RED_THREADS>(mm, a.mmkey);
  }
  pass_stamp(a, 1);
  if (a.peer.world <= 1) {
    grid_barrier(a.bar + 0, a.bar_base[0] + gridDim.x, reinterpret_cast<uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9));
  } else {
    // barrier 1 fused with the cross-GPU MIN: every block arrives; warp 0 of block 0 waits for the local arrivals, pushes
    // this GPU's four keys into every peer's mailbox, waits for the peers' keys, writes the global minima into the local
    // key cell and only then releases the local blocks
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); atomicAdd(a.bar + 0, 1u); }
    if (blockIdx.x == 0 && threadIdx.x < 32) {
      const int lane = threadIdx.x, me = a.peer.rank, W = a.peer.world;
      if (lane == 0) while ((int32_t)(ld_acquire_u32(a.bar + 0) - (a.bar_base[0] + gridDim.x)) < 0) { }
      __syncwarp();
      unsigned long long xw0 = 0;
      if (lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xw0));
      unsigned long long k[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) k[c] = __ldcg(a.mmkey + c);
      bool ok = true;
      if (lane < W && lane != me) {
        unsigned char* dst = mail_min_slot(a.peer.mail[lane], a.seq, me);
        volatile unsigned long long* dk = reinterpret_cast<volatile unsigned long long*>(dst);
#pragma unroll
        for (int c = 0; c < 4; ++c) dk[c] = k[c];
        st_release_sys_u32(reinterpret_cast<uint32_t*>(dst + 40), a.seq);
        const unsigned char* src = mail_min_slot(a.peer.mail[me], a.seq, lane);
        ok = wait_seq_sys(reinterpret_cast<const uint32_t*>(src + 40), a.seq);
        const volatile unsigned long long* sk = reinterpret_cast<const volatile unsigned long long*>(src);
#pragma unroll
        for (int c = 0; c < 4; ++c) k[c] = sk[c];
      } else if (lane >= W) {
#pragma unroll
        for (int c = 0; c < 4; ++c) k[c] = ~0ull;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int c = 0; c < 4; ++c) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, k[c], o); k[c] = v < k[c] ? v : k[c]; }
      }
      const bool all_ok = __all_sync(0xffffffffu, ok);
      if (lane == 0) {
        unsigned long long xw1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xw1));
        a.xwait[0] += xw1 - xw0;      // only this thread of this GPU ever writes these words
        a.xwait[2] += 1;
#pragma unroll
        for (int c = 0; c < 4; ++c) a.mmkey[c] = k[c];
        if (!all_ok) *reinterpret_cast<volatile uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9) = 1u;   // peer timeout
        __threadfence();
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.bar + 3), "r"(a.seq) : "memory");
      }
    }
    if (threadIdx.x == 0) while (ld_acquire_u32(a.bar + 3) != a.seq) { }
    __syncthreads();
  }
  pass_stamp(a, 2);
  if (blockIdx.x == 0 && threadIdx.x == 0) {   // arm the other parity's min/max cell for the next pass
    a.mmkey_next[0] = dkey(1000.0); a.mmkey_next[1] = dkey(-0.0);
    a.mmkey_next[2] = dkey(9999.0); a.mmkey_next[3] = dkey(-0.0);
    a.gstats[2] = 0; a.gstats[4] = 0;
  }
  // ---- phase 2: weights + accumulation into this block's slot
  double* slot = a.block_red + (size_t)blockIdx.x * MALIO_RED_DOUBLES;
  if (FAST) {
    double* s_flush = smem + PASS_FAST_TILES * RED_THREADS * PASS_ROW_STRIDE;
    const double umin = dkey_inv(a.mmkey[0]), umax = -dkey_inv(a.mmkey[1]), tmin = dkey_inv(a.mmkey[2]), tmax = -dkey_inv(a.mmkey[3]);
    uint32_t mine = 0;
    // segment table of the block: seg[k][l] = [beg, end) inside tile k's list (every thread derives it from s_wc)
    uint32_t seg_beg[PASS_FAST_TILES][MALIO_MAX_LIDAR], seg_end[PASS_FAST_TILES][MALIO_MAX_LIDAR];
#pragma unroll
    for (int k = 0; k < PASS_FAST_TILES; ++k) {
      uint32_t run = 0;
#pragma unroll
      for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
        seg_beg[k][l] = run;
#pragma unroll
        for (int w = 0; w < RED_THREADS / 32; ++w) run += s_wc[k][l][w];
        seg_end[k][l] = run;
      }
    }
#pragma unroll
    for (int k = 0; k < PASS_FAST_TILES; ++k) {
      if (go[k].selected) {
        double aw, rho;
        point_weights(prm, go[k].u, pc.ext_en ? go[k].tau : 0.0, pc.ext_en, umin, umax, tmin, tmax, aw, rho);
        double* row = smem + (size_t)(k * RED_THREADS + threadIdx.x) * PASS_ROW_STRIDE;
#pragma unroll
        for (int c = 0; c < 12; ++c) row[c] = row[c] * aw;                       // laserMapping.cpp:714
        row[12] = 1.0 / rho;   // HT(:,i) / R_i (esekfom.hpp:627) as a multiply: <= 1 ulp per term
        row[13] = ((-1) * (double)go[k].pd2) * aw;                               // :707,715
        row[14] = rho;
        // compacted position of this row among the tile's rows of its LiDAR
        const int l = go[k].lid, wid = threadIdx.x >> 5;
        uint32_t pos = l == 0 ? seg_beg[k][0] : (l == 1 ? seg_beg[k][1] : seg_beg[k][2]);
        for (int w = 0; w < wid; ++w) pos += s_wc[k][l][w];
        pos += __popc(bal[k] & ((1u << (threadIdx.x & 31)) - 1u));
        s_list[k * RED_THREADS + pos] = (uint8_t)threadIdx.x;
        ++mine;
      }
    }
    __shared__ uint32_t s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    if (mine) atomicAdd(&s_cnt, mine);
    const int task = threadIdx.x / RED_KS, ks = threadIdx.x % RED_KS;
    const bool worker = task < RED_TASKS;
    int gi = 0, gj = 0;
    if (worker) red_task(task, gi, gj);
    // thread e < 144 ends up holding entry (task e / 16, element e % 16) of each LiDAR's compact system, e >= 128 wraps
    // onto threads 0..15 as a second entry: two result registers per LiDAR and thread
    double res0[MALIO_MAX_LIDAR], res1[MALIO_MAX_LIDAR];
#pragma unroll
    for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
      res0[ll] = 0.0; res1[ll] = 0.0;
      if (ll < pc.L) {
        double acc[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) acc[k] = 0.0;
        if (worker) {
#pragma unroll
          for (int k = 0; k < PASS_FAST_TILES; ++k) {
            for (uint32_t i = seg_beg[k][ll] + ks; i < seg_end[k][ll]; i += RED_KS) {
              const uint32_t q = k * RED_THREADS + s_list[k * RED_THREADS + i];
              const double* row = smem + (size_t)q * PASS_ROW_STRIDE;
              const double ir = row[12];
              const double a0 = row[4 * gi] * ir, a1 = row[4 * gi + 1] * ir, a2 = row[4 * gi + 2] * ir, a3 = row[4 * gi + 3] * ir;
              double c0, c1, c2, c3;
              if (gj < 3) { c0 = row[4 * gj]; c1 = row[4 * gj + 1]; c2 = row[4 * gj + 2]; c3 = row[4 * gj + 3]; }
              else { const double rho = row[14]; c0 = row[13]; c1 = rho * row[0]; c2 = rho * row[1]; c3 = rho * row[2]; }
              acc[0] = fma(a0, c0, acc[0]);   acc[1] = fma(a0, c1, acc[1]);   acc[2] = fma(a0, c2, acc[2]);   acc[3] = fma(a0, c3, acc[3]);
              acc[4] = fma(a1, c0, acc[4]);   acc[5] = fma(a1, c1, acc[5]);   acc[6] = fma(a1, c2, acc[6]);   acc[7] = fma(a1, c3, acc[7]);
              acc[8] = fma(a2, c0, acc[8]);   acc[9] = fma(a2, c1, acc[9]);   acc[10] = fma(a2, c2, acc[10]); acc[11] = fma(a2, c3, acc[11]);
              acc[12] = fma(a3, c0, acc[12]); acc[13] = fma(a3, c1, acc[13]); acc[14] = fma(a3, c2, acc[14]); acc[15] = fma(a3, c3, acc[15]);
            }
          }
#pragma unroll
          for (int k = 0; k < 16; ++k) s_flush[k * (RED_TASKS * RED_KS) + threadIdx.x] = acc[k];
        }
        __syncthreads();
        {   // fold the RED_KS row-splits in a fixed order
          const int e0 = threadIdx.x, e1 = threadIdx.x + RED_THREADS;
          double sum = 0.0;
#pragma unroll
          for (int q = 0; q < RED_KS; ++q) sum += s_flush[(e0 % 16) * (RED_TASKS * RED_KS) + (e0 / 16) * RED_KS + q];
          res0[ll] = sum;
          if (e1 < RED_TASKS * 16) {
            sum = 0.0;
#pragma unroll
            for (int q = 0; q < RED_KS; ++q) sum += s_flush[(e1 % 16) * (RED_TASKS * RED_KS) + (e1 / 16) * RED_KS + q];
            res1[ll] = sum;
          }
        }
        __syncthreads();
      }
    }
#pragma unroll
    for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
      slot[ll * RED_TASKS * 16 + threadIdx.x] = res0[ll];
      if (threadIdx.x + RED_THREADS < RED_TASKS * 16) slot[ll * RED_TASKS * 16 + threadIdx.x + RED_THREADS] = res1[ll];
    }
    if (threadIdx.x == 0) { slot[MALIO_RED_BLOCKS * 16] = (double)s_cnt; slot[MALIO_RED_BLOCKS * 16 + 1] = 0.0; }
  } else {
    reduce_block(a.N, prm, pc.ext_en, a.sel, a.lid8, a.rows12, a.pd2, a.ucov, a.tau, a.mmkey, t0, t1, slot);
  }
  pass_stamp(a, 3);
  grid_barrier(a.bar + 1, a.bar_base[1] + gridDim.x, reinterpret_cast<uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9));
  pass_stamp(a, 4);
  // ---- phase 3: fold the slots, one warp per entry, in fold_kernel's order
  const uint32_t lane = threadIdx.x & 31u, wpb = RED_THREADS / 32;
  uint32_t folded = 0;
  for (uint32_t e = blockIdx.x * wpb + (threadIdx.x >> 5); e < MALIO_RED_DOUBLES; e += gridDim.x * wpb) {
    double sum = 0.0;
    for (uint32_t bk = lane; bk < gridDim.x; bk += 32) sum += a.block_red[(size_t)bk * MALIO_RED_DOUBLES + e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) a.d_res[e] = sum;
    ++folded;
  }
  if (folded) {   // warp-uniform
    uint32_t done = 0;
    if (lane == 0) {
      __threadfence();
      done = atomicAdd(a.bar + 2, folded) + folded;
    }
    done = __shfl_sync(0xffffffffu, done, 0);
    if (done == a.bar_base[2] + MALIO_RED_DOUBLES) {
      // this warp folded the last entry: ship result + min/max keys to the mapped host buffer (posted PCIe writes, one
      // system-scope fence), then the sequence flag the host is spinning on
      __threadfence();
      if (a.peer.world > 1) {
        // cross-GPU SUM: this GPU's folded system goes into slot [me] of every mailbox (its own included), then the
        // slots of all ranks are added in rank order — the same order on every GPU, so all ranks hold identical bits
        const int me = a.peer.rank, W = a.peer.world;
        unsigned long long xs0 = 0;
        if (lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xs0));
        // payload with ordinary (weak) stores: they pipeline over NVLink; the system-scope fence + the release flag below publish
        // them.  (volatile = strong system-scope stores cost ~0.5 us EACH here: 17 us per pass at N = 2, ~60 us at N = 8.)
        {
          double v[(MALIO_RED_DOUBLES + 31) / 32];
#pragma unroll
          for (uint32_t j = 0; j < (MALIO_RED_DOUBLES + 31) / 32; ++j) { const uint32_t e = lane + 32 * j; v[j] = e < MALIO_RED_DOUBLES ? __ldcg(a.d_res + e) : 0.0; }
          for (int r = 0; r < W; ++r) {
            double* dst = reinterpret_cast<double*>(mail_sum_slot(a.peer.mail[r], a.seq, me));
#pragma unroll
            for (uint32_t j = 0; j < (MALIO_RED_DOUBLES + 31) / 32; ++j) { const uint32_t e = lane + 32 * j; if (e < MALIO_RED_DOUBLES) dst[e] = v[j]; }
          }
        }
        __threadfence_system();
        __syncwarp();
        bool ok = true;
        if ((int)lane < W && (int)lane != me) {
          st_release_sys_u32(reinterpret_cast<uint32_t*>(mail_sum_slot(a.peer.mail[lane], a.seq, me) + MAIL_SUM_SEQ_OFF), a.seq);
          ok = wait_seq_sys(reinterpret_cast<const uint32_t*>(mail_sum_slot(a.peer.mail[me], a.seq, (int)lane) + MAIL_SUM_SEQ_OFF), a.seq);
        }
        if (!__all_sync(0xffffffffu, ok) && lane == 0) *reinterpret_cast<volatile uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9) = 1u;
        if (lane == 0) {
          unsigned long long xs1;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xs1));
          a.xwait[1] += xs1 - xs0;    // the last-folding warp of the grid: one writer per pass
        }
        __syncwarp();     // every lane's peer has published (acquire loads above); L2 is the coherence point for the peers' writes
        for (uint32_t e = lane; e < MALIO_RED_DOUBLES; e += 32) {
          double sum = 0.0;
          for (int r = 0; r < W; ++r) sum += __ldcg(reinterpret_cast<const double*>(mail_sum_slot(a.peer.mail[me], a.seq, r)) + e);
          a.d_res[e] = sum;
          a.h_res[e] = sum;
        }
      } else {
        for (uint32_t e = lane; e < MALIO_RED_DOUBLES; e += 32) a.h_res[e] = __ldcg(a.d_res + e);
      }
      if (lane < 4) reinterpret_cast<unsigned long long*>(a.h_res + MALIO_RED_DOUBLES)[lane] = a.mmkey[lane];
      // k-NN list statistics of the last search as knn_list_kernel published them ([3] traversal list, [5] 5x5x5 retries),
      // the traversal fault bits and the tie count
      if (lane == 4) { uint32_t* hg = reinterpret_cast<uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 4); hg[3] = a.gstats[3]; hg[5] = a.gstats[5]; hg[6] = a.gstats[6]; hg[7] = a.gstats[7]; }
      __threadfence_system();
      __syncwarp();
      if (lane == 0) *reinterpret_cast<volatile uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 8) = a.seq;
    }
  }
  pass_stamp(a, 5);
}

// second stage: one warp per entry of the reduced system folds the per-block slots in a fixed order
// (lane-strided partial sums, then a shuffle tree) -> bit-reproducible result, no FP64 atomics
__global__ void __launch_bounds__(256)
fold_kernel(const double* __restrict__ block_red, uint32_t n_slots, double* __restrict__ d_res,
            unsigned long long* __restrict__ next_mmkey, uint32_t* __restrict__ gstats) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {   // arm the other parity's min/max cell for the next pass
    gstats[2] = 0; gstats[4] = 0;              // and the k-NN fast path's unsettled / ring-2 counters
    next_mmkey[0] = dkey(1000.0); next_mmkey[1] = dkey(-0.0);    // laserMapping.cpp:615-616
    next_mmkey[2] = dkey(9999.0); next_mmkey[3] = dkey(-0.0);    // :646-647
  }
  const uint32_t e = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (e >= MALIO_RED_DOUBLES) return;
  double s = 0.0;
  for (uint32_t bk = lane; bk < n_slots; bk += 32) s += block_red[(size_t)bk * MALIO_RED_DOUBLES + e];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) d_res[e] = s;
}

// rows for the degenerate branch (esekfom.hpp:574-582): the first `cap` selected points in position order, one
// block; rows are written in the padded 24-column layout + z, un-weighted by the localization weight
__global__ void rows_kernel(uint32_t N, ParamConst prm, int ext_en, const uint8_t* __restrict__ sel,
                            const uint8_t* __restrict__ lid8, const double* __restrict__ rows12,
                            const float* __restrict__ pd2v, const double* __restrict__ ucov,
                            const double* __restrict__ tau, const unsigned long long* __restrict__ d_mm, uint32_t cap,
                            double* __restrict__ rows /* cap x 25 */, uint32_t* __restrict__ n_rows) {
  __shared__ uint32_t s_base;
  __shared__ uint32_t s_wcnt[32];
  if (threadIdx.x == 0) s_base = 0;
  const double umin = dkey_inv(d_mm[0]), umax = -dkey_inv(d_mm[1]), tmin = dkey_inv(d_mm[2]), tmax = -dkey_inv(d_mm[3]);
  __syncthreads();
  for (uint32_t start = 0; start < N; start += blockDim.x) {
    const uint32_t p = start + threadIdx.x;
    const bool ok = (p < N) && sel[p];
    const uint32_t bal = __ballot_sync(0xffffffffu, ok);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) s_wcnt[w] = __popc(bal);
    __syncthreads();
    uint32_t off = s_base;
    for (int k = 0; k < w; ++k) off += s_wcnt[k];
    off += __popc(bal & ((1u << lane) - 1u));
    if (ok && off < cap) {
      double a, rho;
      point_weights(prm, ucov[p], ext_en ? tau[p] : 0.0, ext_en, umin, umax, tmin, tmax, a, rho);
      const int l = lid8[p];
      double* o = rows + (size_t)off * 25;
      for (int k = 0; k < 24; ++k) o[k] = 0.0;
      const double* j = rows12 + (size_t)p * 12;
      for (int k = 0; k < 6; ++k) o[k] = j[k] * a;
      for (int k = 0; k < 3; ++k) { o[6 + 3 * l + k] = j[6 + k] * a; o[15 + 3 * l + k] = j[9 + k] * a; }
      o[24] = ((-1) * (double)pd2v[p]) * a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t tot = 0;
      for (int k = 0; k < (int)(blockDim.x >> 5); ++k) tot += s_wcnt[k];
      s_base += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *n_rows = s_base;
    rows[(size_t)MALIO_MAX_DOF * 25] = (double)(s_base < cap ? s_base : cap);   // count travels with the rows (multi-rank gather)
  }
}

// ------------------------------------------------------------------ NCCL through dlopen (no link-time dependency)
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool load(std::string& err) {
    if (lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
    if (!lib) { err = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return false; }
    GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
    AllReduce = (decltype(AllReduce))dlsym(lib, "ncclAllReduce");
    AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
    CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
    GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllReduce || !CommDestroy) { err = "NCCL symbols missing"; return false; }
    return true;
  }
};
NcclApi g_nccl;

ParamConst make_param_const(const malio_params& p) {
  ParamConst c{};
  c.plane_th = p.plane_th; c.knn_max_sqdist = p.knn_max_sqdist;
  c.cov_threshold = p.cov_threshold; c.point_cov_max = p.point_cov_max; c.point_cov_min = p.point_cov_min;
  c.plane_cov_max = p.plane_cov_max; c.plane_cov_min = p.plane_cov_min; c.range_min = p.range_min; c.range_max = p.range_max;
  return c;
}

// blocks in one wave of the fused pass's FAST variant: its co-resident blocks, capped at the slots for the per-block
// systems (red_grid).  measure() and the sort's LiDAR-major switch derive the launch from it.
static uint32_t fast_wave(const DeviceState* D) {
  return (D->pass_max_blocks > 0 && (uint32_t)D->pass_max_blocks < D->red_grid) ? (uint32_t)D->pass_max_blocks : D->red_grid;
}

// padded (L=3 positions) -> compact c columns: 0-5 | 6+3l | 6+3L+3l
void compact_columns(int L, int map[MALIO_MAX_COLS]) {
  for (int k = 0; k < 6; ++k) map[k] = k;
  for (int l = 0; l < L; ++l)
    for (int k = 0; k < 3; ++k) { map[6 + 3 * l + k] = 6 + 3 * l + k; map[6 + 3 * L + 3 * l + k] = 15 + 3 * l + k; }
}

// ---- measure() in pieces, all enqueued on D->stream: search, then the fused pass or the separate kernels, then the host
// epilogue.  Events: ev[0] start | ev[5] sorted | ev[6] k-NN done | ev[1] pass start | ev[2] gate done | ev[3] reduced |
// ev[4] result on the host.

// the search of a pass: the scan sort (once per scan), evalPointUncertainty's traces (once per scan), the k-NN (search
// passes)
int pass_search(malio_handle* h, DeviceState* D, const PassConst& pc, int redo_knn, bool fused_now,
                const malio_scan_pt* pts_k, bool& sorted_now, bool& knn_now) {
  cudaStream_t st = D->stream;
  const uint32_t N = D->N;
  bool tau_async = false;
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[0], st));
  if (N > 0) {
    if (h->cfg.sort_queries && !D->perm_valid) {
      // LiDAR-major keys exactly where the fused pass leaves its FAST variant (more than PASS_FAST_TILES tiles per block)
      const int lid_major = (uint64_t)N > (uint64_t)PASS_FAST_TILES * RED_THREADS * (uint64_t)fast_wave(D) ? 1 : 0;
      if (int rc = sort_queries<0>(h, D, N, pc, lid_major)) return rc;
      D->perm_valid = true;
      sorted_now = true;
    }
    if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[5], st));
    // once per scan: evalPointUncertainty's trace depends on the point and its table entry only.  On the first pass of
    // a scan that is a search pass it runs on the second stream beside the k-NN kernels (which leave most of the SMs'
    // warp slots empty) instead of inside the pass kernel.
    if (!D->tau_valid && redo_knn && D->fused) {
      CUDA_TRY(cudaEventRecord(D->ev_sorted, st));
      CUDA_TRY(cudaStreamWaitEvent(D->stream2, D->ev_sorted, 0));
      tau_kernel<<<(N + PLANE_THREADS - 1) / PLANE_THREADS, PLANE_THREADS, 0, D->stream2>>>(pts_k, nullptr, N, pc, D->d_table, D->d_tau2);
      CUDA_TRY(cudaEventRecord(D->ev_tau, D->stream2));
      D->tau_valid = true;
      D->ctr.kernel_launches += 1;
      tau_async = true;
    }
    if (redo_knn) {
      knn_now = true;
      if (int rc = run_knn<0>(h, D, N, pts_k, nullptr, pc, h->cfg.params.knn_max_sqdist)) return rc;
      if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[6], st));
      // list statistics of this search: the fused pass kernel ships them with its result; the separate-kernel path copies
      if (!fused_now) { if (int rc = fetch_knn_stats(h, D, st)) return rc; }
    }
  }
  if (tau_async) CUDA_TRY(cudaStreamWaitEvent(st, D->ev_tau, 0));
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[1], st));
  return MALIO_OK;
}

// launch geometry of a pass (tests/reduce_ref.py restates it): one resident wave, every block the same number of tiles (+-1),
// no straggler blocks
struct PassGeom { uint32_t n_tiles, per_block, grid; };
PassGeom pass_geometry(const DeviceState* D, bool fused_now) {
  PassGeom g;
  g.n_tiles = (D->N + RED_THREADS - 1) / RED_THREADS;
  uint32_t wave = fused_now ? fast_wave(D) : D->red_grid;
  g.per_block = g.n_tiles ? (g.n_tiles + wave - 1) / wave : 1;
  if (fused_now && g.per_block > (uint32_t)PASS_FAST_TILES) {   // rows through global memory: that variant's own co-residency limit
    wave = (uint32_t)D->pass_max_blocks_generic < D->red_grid ? (uint32_t)D->pass_max_blocks_generic : D->red_grid;
    g.per_block = (g.n_tiles + wave - 1) / wave;
  }
  g.grid = g.n_tiles ? (g.n_tiles + g.per_block - 1) / g.per_block : 1;
  return g;
}

// the whole pass in one cooperative launch; the result arrives in mapped host memory.  With several GPUs the two
// exchanges of the pass happen inside the kernel through the peers' mailboxes (CUDA IPC over NVLink).  hp1: host clock
// once the launch is enqueued.
int pass_fused(malio_handle* h, DeviceState* D, const PassConst& pc, const ParamConst& prm, int redo_knn,
               const malio_scan_pt* pts_k, const PassGeom& g, std::chrono::steady_clock::time_point& hp1) {
  cudaStream_t st = D->stream;
  const uint32_t N = D->N, grid = g.grid;
  PassArgs a{};
  a.pts = pts_k; a.perm = nullptr; a.N = N; a.table = D->d_table; a.nodes = D->d_mpts; a.node_cov = D->d_cov;
  a.nn_idx = D->d_nn_idx; a.sel = D->d_sel; a.world = D->d_world; a.plane = D->d_plane; a.ucov = D->d_ucov;
  a.tau2 = D->d_tau2; a.pd2 = D->d_pd2; a.tau = D->d_tau; a.normal_y = D->d_normal_y; a.rows12 = D->d_rows12; a.lid8 = D->d_lid8;
  a.do_tau = (N > 0 && !D->tau_valid) ? 1 : 0;
  a.do_fit = (N > 0 && redo_knn) ? 1 : 0;
  a.mmkey = D->d_mmkey + 4 * D->parity; a.mmkey_next = D->d_mmkey + 4 * (1 - D->parity); a.gstats = D->d_gstats;
  a.bar = D->d_bar;
  for (int k = 0; k < 3; ++k) a.bar_base[k] = D->bar_base[k];
  D->bar_base[0] += grid; D->bar_base[1] += grid; D->bar_base[2] += MALIO_RED_DOUBLES;
  a.n_tiles = g.n_tiles; a.block_red = D->d_block_red; a.d_res = D->d_res; a.h_res = D->h_res_dev;
  a.seq = ++D->seq;
  a.peer.rank = D->rank; a.peer.world = D->p2p ? D->world : 1;
  for (int r = 0; r < MAIL_MAX_WORLD; ++r) a.peer.mail[r] = D->mail_peer[r];
  *reinterpret_cast<volatile uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 9) = 0u;
  a.dbg = nullptr;
  a.xwait = D->d_cand + 1;
  if (D->trace_passes > 0) {
    if (!D->d_dbg) { if (int rc = D->d_dbg.allocate(h, D->stream, (size_t)4096 * 8)) return rc; D->trace_left = D->trace_passes; }
    if (D->trace_left > 0 && grid <= 4096) a.dbg = D->d_dbg;
  }
  PassConst pc_arg = pc;
  ParamConst prm_arg = prm;
  void* kargs[] = {&a, &pc_arg, &prm_arg};
  const bool fast = g.per_block <= (uint32_t)PASS_FAST_TILES;
  const size_t pass_smem = (fast ? PASS_FAST_SMEM_DOUBLES : RED_SMEM_DOUBLES) * sizeof(double);
  CUDA_TRY(cudaLaunchCooperativeKernel(fast ? (const void*)pass_kernel<true> : (const void*)pass_kernel<false>, dim3(grid),
                                       dim3(RED_THREADS), kargs, pass_smem, st));
  D->ctr.kernel_launches += 1;
  D->tau_valid = D->tau_valid || N > 0;
  if (D->timing) { CUDA_TRY(cudaEventRecord(D->ev[2], st)); CUDA_TRY(cudaEventRecord(D->ev[3], st)); CUDA_TRY(cudaEventRecord(D->ev[4], st)); }
  D->last_parity = D->parity;
  D->parity = 1 - D->parity;
  hp1 = std::chrono::steady_clock::now();
  // the host needs the 3.5 KB system to take the IESKF step: spin on the sequence flag the kernel writes last
  volatile uint32_t* flag = reinterpret_cast<volatile uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 8);
  for (uint64_t spins = 1; *flag != D->seq; ++spins) {
    __builtin_ia32_pause();
    if ((spins & 0x3FFF) == 0) {
      const cudaError_t q = cudaStreamQuery(st);
      if (q == cudaErrorNotReady) {
        if (std::chrono::duration<double>(std::chrono::steady_clock::now() - hp1).count() > 20.0) {
          h->err = "pass_kernel: no result after 20 s";
          return MALIO_ERR_CUDA;
        }
        continue;
      }
      if (q != cudaSuccess) { h->err = std::string("pass_kernel: ") + cudaGetErrorString(q); return MALIO_ERR_CUDA; }
      if (*flag != D->seq) { h->err = "pass_kernel finished without publishing its result"; return MALIO_ERR_CUDA; }
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  if (const uint32_t fault = *reinterpret_cast<volatile uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 9)) {
    if (fault == 2u) { h->err = "pass_kernel: a grid barrier did not complete within 2 s (blocks not co-resident)"; return MALIO_ERR_CUDA; }
    h->err = "pass_kernel: a peer GPU did not answer the in-kernel exchange within 2 s";
    return MALIO_ERR_NCCL;
  }
  if (a.dbg) {
    CUDA_TRY(cudaStreamSynchronize(st));
    std::vector<unsigned long long> t((size_t)grid * 8);
    CUDA_TRY(cudaMemcpy(t.data(), D->d_dbg, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    unsigned long long t00 = ~0ull;
    for (uint32_t b = 0; b < grid; ++b) if (t[b * 8] < t00) t00 = t[b * 8];
    const char* nm[6] = {"start", "phase1 done", "barrier1 passed", "phase2 done", "barrier2 passed", "end"};
    fprintf(stderr, "[malio] pass trace: grid %u fast %d fit %d tau %d (us from first block start: min / mean / max over blocks)\n",
            grid, g.per_block <= (uint32_t)PASS_FAST_TILES, a.do_fit, a.do_tau);
    for (int k = 0; k < 6; ++k) {
      double mn = 1e30, mx = 0, sm = 0;
      for (uint32_t b = 0; b < grid; ++b) { const double v = (double)(t[b * 8 + k] - t00) * 1e-3; mn = v < mn ? v : mn; mx = v > mx ? v : mx; sm += v; }
      fprintf(stderr, "[malio]   %-16s %8.2f %8.2f %8.2f\n", nm[k], mn, sm / grid, mx);
    }
    D->trace_left--;
  }
  if (D->timing) CUDA_TRY(cudaEventSynchronize(D->ev[4]));
  return MALIO_OK;
}

// the pass as separate kernels (no cooperative launch, or several GPUs without peer mailboxes: NCCL between the kernels).
// hp1: host clock once everything is enqueued.
int pass_separate(malio_handle* h, DeviceState* D, const PassConst& pc, const ParamConst& prm, int redo_knn,
                  const malio_scan_pt* pts_k, const PassGeom& g, std::chrono::steady_clock::time_point& hp1) {
  cudaStream_t st = D->stream;
  const uint32_t N = D->N;
  unsigned long long* mmkey = D->d_mmkey + 4 * D->parity;
  unsigned long long* mmkey_next = D->d_mmkey + 4 * (1 - D->parity);
  const uint32_t pblocks = N > 0 ? (N + PLANE_THREADS - 1) / PLANE_THREADS : 1;
  if (N > 0 && !D->tau_valid) {   // once per scan
    tau_kernel<<<pblocks, PLANE_THREADS, 0, st>>>(pts_k, nullptr, N, pc, D->d_table, D->d_tau2);
    D->tau_valid = true;
    D->ctr.kernel_launches += 1;
  }
  if (N > 0 && redo_knn) {         // once per search
    fit_kernel<<<pblocks, PLANE_THREADS, 0, st>>>(D->d_mpts, D->d_cov, N, prm, D->d_nn_idx, D->d_sel, D->d_plane, D->d_ucov);
    D->ctr.kernel_launches += 1;
  }
  D->ctr.kernel_launches += 3;     // gate, reduce, fold
  const uint32_t gblocks = N > 0 ? (N + GATE_THREADS - 1) / GATE_THREADS : 1;
  gate_kernel<<<gblocks, GATE_THREADS, 0, st>>>(pts_k, nullptr, N, pc, D->d_plane, D->d_ucov, D->d_tau2, D->d_sel,
                                                D->d_world, D->d_pd2, D->d_tau, D->d_normal_y, D->d_rows12, D->d_lid8, mmkey);
  if (D->comm)   // keys of {min_u, -max_u, min_tau, -max_tau}: one MIN all-reduce (laserMapping.cpp:615-628, 700-703)
    if (g_nccl.AllReduce(mmkey, mmkey, 4, ncclUint64, ncclMin, D->comm, st) != ncclSuccess) { h->err = "ncclAllReduce(min) failed"; return MALIO_ERR_NCCL; }
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[2], st));
  reduce_kernel<<<g.grid, RED_THREADS, RED_SMEM_DOUBLES * sizeof(double), st>>>(
      N, prm, pc.ext_en, D->d_sel, D->d_lid8, D->d_rows12, D->d_pd2, D->d_ucov, D->d_tau, mmkey, g.n_tiles, D->d_block_red);
  fold_kernel<<<(MALIO_RED_DOUBLES * 32 + 255) / 256, 256, 0, st>>>(D->d_block_red, g.grid, D->d_res, mmkey_next, D->d_gstats);
  if (D->comm)   // the reduced system + n_eff: one SUM all-reduce
    if (g_nccl.AllReduce(D->d_res, D->d_res, MALIO_RED_DOUBLES, ncclDouble, ncclSum, D->comm, st) != ncclSuccess) { h->err = "ncclAllReduce(sum) failed"; return MALIO_ERR_NCCL; }
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[3], st));
  CUDA_TRY(cudaMemcpyAsync(D->h_res, D->d_res, MALIO_RED_DOUBLES * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(D->h_res + MALIO_RED_DOUBLES, mmkey, 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
  D->last_parity = D->parity;
  D->parity = 1 - D->parity;
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[4], st));
  hp1 = std::chrono::steady_clock::now();
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}

// host epilogue: un-block, localization weight (laserMapping.cpp:745-759), compact to c x c; pass statistics and counters
int pass_epilogue(malio_handle* h, DeviceState* D, int redo_knn, bool sorted_now, bool knn_now, double* HtRinvH,
                  double* HtRinvh, malio_pass_stats* st) {
  const malio_params& P = h->cfg.params;
  const int L = P.n_lidar, c = 6 * (L + 1);
  const uint32_t N = D->N;
  const double* res = D->h_res;
  double mm[4];
  for (int k = 0; k < 4; ++k) { unsigned long long key; std::memcpy(&key, D->h_res + MALIO_RED_DOUBLES + k, 8); mm[k] = dkey_inv(key); }
  // res holds, per LiDAR l, the 9 upper-triangular 4x4 blocks of the compact 12 x 16 system Gc_l; scatter into the
  // padded 24 x 28 one (columns at their L=3 positions: 0-5 | 6+3l | 15+3l ; 24 = residual ; 25-27 = normal scatter)
  double G[MALIO_RED_ROWS][MALIO_RED_COLS];
  std::memset(G, 0, sizeof(G));
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
    double Gc[12][16];
    std::memset(Gc, 0, sizeof(Gc));
    int t = 0;
    for (int gi = 0; gi < 3; ++gi)
      for (int gj = gi; gj < 4; ++gj, ++t)
        for (int a = 0; a < 4; ++a)
          for (int b = 0; b < 4; ++b) Gc[4 * gi + a][4 * gj + b] = res[(l * 9 + t) * 16 + a * 4 + b];
    for (int a = 0; a < 12; ++a) for (int b = 0; b < a; ++b) Gc[a][b] = Gc[b][a];
    int col[16];
    for (int k = 0; k < 6; ++k) col[k] = k;
    for (int k = 0; k < 3; ++k) { col[6 + k] = 6 + 3 * l + k; col[9 + k] = 15 + 3 * l + k; }
    col[12] = 24; col[13] = 25; col[14] = 26; col[15] = 27;
    for (int a = 0; a < 12; ++a)
      for (int b = 0; b < 16; ++b) G[col[a]][col[b]] += Gc[a][b];
  }
  const uint32_t n_eff = (uint32_t)(res[MALIO_RED_BLOCKS * 16] + 0.5);
  malio_pass_stats S{};
  S.n_points = N; S.n_eff = n_eff; S.searched = redo_knn ? 1 : 0;
  S.u_min = mm[0]; S.u_max = -mm[1]; S.tau_min = mm[2]; S.tau_max = -mm[3];
  float ms = 0.f;
  if (knn_now && D->grid_on) { D->ctr.knn_fallback_queries += D->h_gstats[3]; D->ctr.knn_ring2_queries += D->h_gstats[5]; }
  if (D->timing) {
    if (N > 0 && sorted_now) { cudaEventElapsedTime(&ms, D->ev[0], D->ev[5]); S.ms_sort = ms; }
    if (knn_now) {
      cudaEventElapsedTime(&ms, D->ev[5], D->ev[6]); S.ms_knn = ms;
      D->ctr.knn_launches += 1; D->ctr.knn_queries += N; D->ctr.knn_ms += ms;
    }
    D->ctr.d2h_bytes += (MALIO_RED_DOUBLES + 4) * sizeof(double);
    cudaEventElapsedTime(&ms, D->ev[1], D->ev[2]); S.ms_plane = ms;
    cudaEventElapsedTime(&ms, D->ev[2], D->ev[3]); S.ms_reduce = ms;
    cudaEventElapsedTime(&ms, D->ev[0], D->ev[4]); S.ms_total = ms;
    cudaEventElapsedTime(&ms, D->ev[1], D->ev[4]);
    D->ctr.pass_launches += 1; D->ctr.pass_points += N; D->ctr.pass_ms += ms; D->ctr.pass_fit_launches += redo_knn ? 1 : 0;
  }
  if (n_eff < 1) {
    S.valid = 0;
    if (st) *st = S;
    return MALIO_ERR_NO_EFFECTIVE_POINTS;
  }
  S.valid = 1;
  const double Ssym[6] = {G[0][25], G[0][26], G[0][27], G[1][26], G[1][27], G[2][27]};
  malio_host::sym3_singular_values(Ssym, S.sigma);
  double weight = S.sigma[2] / S.sigma[0];
  if (weight > P.localize_thresh_max) weight = P.localize_cov_max;
  else if (weight < P.localize_thresh_min) weight = P.localize_cov_min;
  else weight = (P.localize_cov_max - P.localize_cov_min) * (weight - P.localize_thresh_min) / (P.localize_thresh_max - P.localize_thresh_min) + P.localize_cov_min;
  S.loc_weight = weight;
  const double w2 = weight * weight;
  int map[MALIO_MAX_COLS];
  compact_columns(L, map);
  for (int a = 0; a < c; ++a) {
    for (int b = 0; b < c; ++b) HtRinvH[a * c + b] = w2 * G[map[a]][map[b]];
    HtRinvh[a] = w2 * G[map[a]][24];
  }
  if (st) *st = S;
  return MALIO_OK;
}
}  // namespace

namespace malio_devstate {

PassConst make_pass_const(const malio_handle* h, const DeviceState* D, const malio_pass_state* s) {
  PassConst pc{};
  std::memcpy(pc.rot, s->rot, sizeof(pc.rot));
  std::memcpy(pc.pos, s->pos, sizeof(pc.pos));
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
    std::memcpy(pc.eq[l], s->ext[l].q, sizeof(pc.eq[l]));
    std::memcpy(pc.et[l], s->ext[l].t, sizeof(pc.et[l]));
    std::memcpy(pc.cq[l], D->tcomp[l].q, sizeof(pc.cq[l]));
    std::memcpy(pc.ct[l], D->tcomp[l].t, sizeof(pc.ct[l]));
  }
  for (int l = 0; l <= MALIO_MAX_LIDAR; ++l) pc.table_off[l] = D->table_off[l];
  auto conj_R = [](const double q[4], double R[9]) {   // Eigen's toRotationMatrix of the conjugate, row-major
    const double w = q[0], x = -q[1], y = -q[2], z = -q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
  };
  conj_R(pc.rot, pc.RsT);
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) { conj_R(pc.eq[l], pc.ReT[l]); conj_R(pc.cq[l], pc.RcT[l]); }
  pc.L = h->cfg.params.n_lidar;
  pc.ext_en = h->cfg.params.extrinsic_est_en;
  return pc;
}

int pass_init(malio_handle* h, DeviceState* D) {
  D->red_grid = (uint32_t)D->sm_count * (PASS_MIN_BLOCKS > 4 ? PASS_MIN_BLOCKS : 4);   // slots for the per-block partial systems
  if (int rc = D->d_block_red.allocate(h, D->stream, (size_t)D->red_grid * MALIO_RED_DOUBLES)) return rc;
  if (int rc = D->d_bar.allocate(h, D->stream, 4)) return rc;
  CUDA_TRY(cudaMemset(D->d_bar, 0, 4 * sizeof(uint32_t)));
  CUDA_TRY(cudaFuncSetAttribute(pass_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RED_SMEM_DOUBLES * (int)sizeof(double)));
  CUDA_TRY(cudaFuncSetAttribute(pass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, RED_SMEM_DOUBLES * (int)sizeof(double)));
  int per_sm = 0, per_sm2 = 0;
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pass_kernel<true>, RED_THREADS, PASS_FAST_SMEM_DOUBLES * sizeof(double)));
  CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, pass_kernel<false>, RED_THREADS, RED_SMEM_DOUBLES * sizeof(double)));
  D->pass_max_blocks_generic = per_sm2 * D->sm_count;
  int coop = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, D->device));
  D->pass_max_blocks = per_sm * D->sm_count;
  D->fused = coop && per_sm > 0;
  if (const char* e = getenv("MALIO_FUSED_PASS")) D->fused = D->fused && atoi(e) != 0;
  if (const char* e = getenv("MALIO_PASS_TRACE")) D->trace_passes = atoi(e);
  CUDA_TRY(cudaFuncSetAttribute(reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                RED_SMEM_DOUBLES * (int)sizeof(double)));
  return MALIO_OK;
}

void comm_destroy(DeviceState* D) {
  if (D->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(D->comm);
  for (unsigned char*& p : D->mail_peer) {   // the peers' mailboxes; this rank's own is D->d_mail
    if (p && p != D->d_mail.data()) cudaIpcCloseMemHandle(p);
    p = nullptr;
  }
}
}  // namespace malio_devstate

namespace malio_dev {

int measure(malio_handle* h, const malio_pass_state* s, int redo_knn, double* HtRinvH, double* HtRinvh,
            malio_pass_stats* st) {
  DeviceState* D = h->dev.get();
  if (h->mapst) { if (int rc = malio_map::commit(h)) return rc; }   // device-resident map: pending deltas -> index
  if (!D->map_ready || !D->scan_ready) { h->err = "measure before upload_map/upload_scan"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const auto hp0 = std::chrono::steady_clock::now();
  const PassConst pc = make_pass_const(h, D, s);
  const ParamConst prm = make_param_const(h->cfg.params);
  D->last_pc = pc;
  const bool fused_now = D->fused && (!D->comm || D->p2p);
  // the per-pass kernels read the scan in position order: the sorted copy when the scan was sorted, else the upload itself
  const malio_scan_pt* pts_k = (h->cfg.sort_queries && D->N > 0) ? D->d_pts_sorted : D->d_pts;
  bool sorted_now = false, knn_now = false;
  if (int rc = pass_search(h, D, pc, redo_knn, fused_now, pts_k, sorted_now, knn_now)) return rc;
  const PassGeom g = pass_geometry(D, fused_now);
  std::chrono::steady_clock::time_point hp1;
  if (int rc = fused_now ? pass_fused(h, D, pc, prm, redo_knn, pts_k, g, hp1) : pass_separate(h, D, pc, prm, redo_knn, pts_k, g, hp1))
    return rc;
  const auto hp2 = std::chrono::steady_clock::now();
  D->pass_done = true;
  if (int rc = knn_fault(h, D)) return rc;
  D->host_launch_us += std::chrono::duration<double, std::micro>(hp1 - hp0).count();
  D->host_wait_us += std::chrono::duration<double, std::micro>(hp2 - hp1).count();
  D->host_passes += 1;
  return pass_epilogue(h, D, redo_knn, sorted_now, knn_now, HtRinvH, HtRinvh, st);
}

int download_rows(malio_handle* h, double* h_x, double* hvec, uint32_t cap, uint32_t* n_rows) {
  DeviceState* D = h->dev.get();
  if (!D->pass_done) { h->err = "download_rows before measure"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const malio_params& P = h->cfg.params;
  const int L = P.n_lidar, c = 6 * (L + 1);
  if (cap > MALIO_MAX_DOF) cap = MALIO_MAX_DOF;
  rows_kernel<<<1, 256, 0, D->stream>>>(D->N, make_param_const(P), D->last_pc.ext_en, D->d_sel, D->d_lid8, D->d_rows12,
                                          D->d_pd2, D->d_ucov, D->d_tau, D->d_mmkey + 4 * D->last_parity, cap, D->d_rows,
                                          D->d_counters + 3);
  double* hr = D->h_res + MALIO_RED_DOUBLES + 16;
  uint32_t nr = 0;
  std::vector<double> gathered;
  if (D->comm && D->world > 1) {
    // stats->n_eff is summed over the ranks, the rows are not: gather every rank's (at most cap) rows and concatenate them in
    // rank order, so that every rank forms the same H and takes the same step (esekfom.hpp:574-582 needs all N_eff rows)
    if (!g_nccl.AllGather) { h->err = "ncclAllGather unavailable: cannot gather the rows of the degenerate branch"; return MALIO_ERR_NCCL; }
    double* d_all = D->d_rows + ROWS_DOUBLES;
    if (g_nccl.AllGather(D->d_rows, d_all, ROWS_DOUBLES, ncclDouble, D->comm, D->stream) != ncclSuccess) { h->err = "ncclAllGather(rows) failed"; return MALIO_ERR_NCCL; }
    gathered.resize((size_t)ROWS_DOUBLES * D->world);
    CUDA_TRY(cudaMemcpyAsync(gathered.data(), d_all, gathered.size() * sizeof(double), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    D->ctr.kernel_launches += 1;
    for (int r = 0; r < D->world && nr < cap; ++r) {
      const double* src = gathered.data() + (size_t)r * ROWS_DOUBLES;
      const uint32_t cnt = (uint32_t)(src[(size_t)MALIO_MAX_DOF * 25] + 0.5);
      for (uint32_t k = 0; k < cnt && nr < cap; ++k, ++nr) std::memcpy(hr + (size_t)nr * 25, src + (size_t)k * 25, 25 * sizeof(double));
    }
  } else {
    CUDA_TRY(cudaMemcpyAsync(hr, D->d_rows, (size_t)cap * 25 * sizeof(double), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaMemcpyAsync(&nr, D->d_counters + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    if (nr > cap) nr = cap;
  }
  int map[MALIO_MAX_COLS];
  compact_columns(L, map);
  for (uint32_t r = 0; r < nr; ++r) {
    for (int k = 0; k < c; ++k) h_x[(size_t)r * c + k] = hr[(size_t)r * 25 + map[k]];
    hvec[r] = hr[(size_t)r * 25 + 24];
  }
  *n_rows = nr;
  return MALIO_OK;
}

int get_unique_id(uint8_t* id) {
  std::string err;
  if (!g_nccl.load(err)) return MALIO_ERR_NCCL;
  ncclUniqueId uid;
  if (g_nccl.GetUniqueId(&uid) != ncclSuccess) return MALIO_ERR_NCCL;
  static_assert(sizeof(ncclUniqueId) == MALIO_NCCL_UNIQUE_ID_BYTES, "ncclUniqueId size");
  std::memcpy(id, &uid, sizeof(uid));
  return MALIO_OK;
}

int comm_init(malio_handle* h, const uint8_t* id, int rank, int world) {
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  if (!g_nccl.load(h->err)) return MALIO_ERR_NCCL;
  ncclUniqueId uid;
  std::memcpy(&uid, id, sizeof(uid));
  ncclResult_t r = g_nccl.CommInitRank(&D->comm, world, uid, rank);
  if (r != ncclSuccess) {
    h->err = std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    D->comm = nullptr;
    return MALIO_ERR_NCCL;
  }
  D->rank = rank; D->world = world;
  // ---- peer mailboxes for the in-kernel exchanges (CUDA IPC; NCCL only carries the 64-byte handles).  Falls back to the
  // NCCL all-reduce path between separate kernels unless EVERY rank succeeded.
  D->p2p = false;
  const char* env = getenv("MALIO_P2P");
  int ok = (world > 1 && world <= MAIL_MAX_WORLD && D->fused && g_nccl.AllGather && !(env && atoi(env) == 0)) ? 1 : 0;
  cudaIpcMemHandle_t mine{};
  DeviceBuffer<unsigned char> d_h;
  std::vector<cudaIpcMemHandle_t> all((size_t)world);
  if (ok) {
    if (D->d_mail.allocate_empty(MAIL_BYTES) != cudaSuccess || cudaMemset(D->d_mail, 0, MAIL_BYTES) != cudaSuccess ||
        cudaIpcGetMemHandle(&mine, D->d_mail) != cudaSuccess) { ok = 0; cudaGetLastError(); }
  }
  // every rank takes part in the two collectives below whatever its own outcome
  if (world > 1 && g_nccl.AllGather) {
    if (int rc = d_h.allocate(h, D->stream, (size_t)(world + 1) * sizeof(mine) + 2 * sizeof(int))) return rc;
    CUDA_TRY(cudaMemcpy(d_h + (size_t)world * sizeof(mine), &mine, sizeof(mine), cudaMemcpyHostToDevice));
    if (g_nccl.AllGather(d_h + (size_t)world * sizeof(mine), d_h, sizeof(mine), ncclChar, D->comm, D->stream) != ncclSuccess) ok = 0;
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    CUDA_TRY(cudaMemcpy(all.data(), d_h, (size_t)world * sizeof(mine), cudaMemcpyDeviceToHost));
    if (ok) {
      for (int r = 0; r < world && ok; ++r) {
        if (r == rank) { D->mail_peer[r] = D->d_mail; continue; }
        void* ptr = nullptr;
        if (cudaIpcOpenMemHandle(&ptr, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); }
        D->mail_peer[r] = (unsigned char*)ptr;
      }
    }
    int* d_ok = reinterpret_cast<int*>(d_h + (size_t)(world + 1) * sizeof(mine));
    CUDA_TRY(cudaMemcpy(d_ok, &ok, sizeof(int), cudaMemcpyHostToDevice));
    if (g_nccl.AllReduce(d_ok, d_ok + 1, 1, ncclInt, ncclMin, D->comm, D->stream) != ncclSuccess) ok = 0;
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    int all_ok = 0;
    CUDA_TRY(cudaMemcpy(&all_ok, d_ok + 1, sizeof(int), cudaMemcpyDeviceToHost));
    D->p2p = ok && all_ok;
  }
  if (D->host_prof) fprintf(stderr, "[malio] rank %d/%d: in-kernel peer exchange %s\n", rank, world, D->p2p ? "ON" : "off (NCCL path)");
  return MALIO_OK;
}

}  // namespace malio_dev
