// malio_solve.cu — the IESKF step on the device (sm_90a): esekf::update_iterated_dyn_share_modified's per-pass algebra
// (esekfom.hpp:521-718) as a one-block kernel that runs after every measurement pass, so that a whole iterated update is ONE
// enqueued kernel sequence without a host round trip per pass.
//
// What the host loop (malio_host.cpp: malio_ieskf_update) did between two pass kernels — wait for the 3.5 KB system over
// PCIe, ~10 us of 35 x 35 algebra, a ~15 us cooperative launch — is replaced by: solve_kernel reads the folded system from
// device memory, takes the step (same algebra: one c x c LU of (I + G P_cc)^T, two right-hand sides, the n x c block only
// in the pass that updates the covariance), writes the next pass's constants (state, rotation matrices) and the
// "repeat the search" / "done" flags into the ScanCtl block the already-enqueued kernels of the following passes read.
// The degenerate branch n > N_eff (esekfom.hpp:574-582) needs the dense rows: it is flagged and the host finishes that
// (rare) scan through its own loop.  Manifold operators: malio_manifold.h (shared with the host code).
#include <cuda_runtime.h>

#include <cstring>

#include "malio_device.cuh"
#include "malio_manifold.h"

using namespace malio_devstate;
using namespace malio_manifold;

namespace {

constexpr int SV_T = 256;
constexpr int ND = MALIO_MAX_DOF, NC = MALIO_MAX_COLS;

__device__ __forceinline__ void conj_R(const double q[4], double R[9]) {   // toRotationMatrix of the conjugate, row-major
  const double w = q[0], x = -q[1], y = -q[2], z = -q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
// pass constants of the next pass from the state sx (shared memory): make_pass_const of malio_b200.cu on the device; called by
// all threads of the block (7 of them build one rotation matrix each)
__device__ void build_pc(ScanCtl* c, const malio_state& sx) {
  PassConst& pc = c->pc;
  const int tid = threadIdx.x;
  if (tid < 4) pc.rot[tid] = sx.rot[tid];
  if (tid < 3) pc.pos[tid] = sx.pos[tid];
  if (tid >= 32 && tid < 32 + MALIO_MAX_LIDAR) {
    const int l = tid - 32;
    for (int k = 0; k < 4; ++k) { pc.eq[l][k] = sx.ext[l].q[k]; pc.cq[l][k] = c->tcomp[l].q[k]; }
    for (int k = 0; k < 3; ++k) { pc.et[l][k] = sx.ext[l].t[k]; pc.ct[l][k] = c->tcomp[l].t[k]; }
  }
  if (tid >= 64 && tid < 64 + MALIO_MAX_LIDAR) { double R[9]; conj_R(sx.ext[tid - 64].q, R); for (int k = 0; k < 9; ++k) pc.ReT[tid - 64][k] = R[k]; }
  if (tid >= 96 && tid < 96 + MALIO_MAX_LIDAR) { double R[9]; conj_R(c->tcomp[tid - 96].q, R); for (int k = 0; k < 9; ++k) pc.RcT[tid - 96][k] = R[k]; }
  if (tid == 128) { double R[9]; conj_R(sx.rot, R); for (int k = 0; k < 9; ++k) pc.RsT[k] = R[k]; }
  if (tid == 160) {
    for (int l = 0; l <= MALIO_MAX_LIDAR; ++l) pc.table_off[l] = c->table_off[l];
    pc.L = c->L;
    pc.ext_en = c->ext_en;
  }
}

__global__ void __launch_bounds__(SV_T) init_ctl_kernel(ScanCtl* c, uint32_t seq0, int parity, uint32_t* bar) {
  __shared__ malio_state sx;
  const int tid = threadIdx.x;
  {
    const double* src = reinterpret_cast<const double*>(&c->x_prop);
    double* dst = reinterpret_cast<double*>(&sx);
    double* gx = reinterpret_cast<double*>(&c->x);
    for (int k = tid; k < (int)(sizeof(malio_state) / sizeof(double)); k += SV_T) { const double v = src[k]; dst[k] = v; gx[k] = v; }
  }
  __syncthreads();
  build_pc(c, sx);
  const int nn = c->n * c->n;
  for (int k = tid; k < nn; k += SV_T) c->P_cur[k] = c->P_prop[k];
  for (int k = tid; k < ND; k += SV_T) c->dx_last[k] = 0.0;
  if (tid == 0) {
    c->it = -1; c->redo = 1; c->active = 1; c->t = 0; c->parity = parity; c->seq = seq0;
    c->passes = 0; c->searches = 0; c->status = MALIO_OK; c->need_host = 0; c->n_eff_last = 0; c->converged_count = 0; c->searched_mask = 0;
    bar[0] = 0; bar[1] = 0; bar[2] = 0;
    c->bar_base[0] = c->bar_base[1] = c->bar_base[2] = c->bar_base[3] = 0;
  }
}

// rows [idx, idx+BS) <- J * rows   /  cols <- cols * J^T   (esekfom.hpp:541-548, 563-571), one thread per column / row
template <int BS>
__device__ __forceinline__ void left_block(double* M, int ld, int idx, const double* J, int ncols) {
  for (int j = threadIdx.x; j < ncols; j += SV_T) {
    double v[BS], o[BS];
    for (int a = 0; a < BS; ++a) v[a] = M[(idx + a) * ld + j];
    for (int a = 0; a < BS; ++a) { o[a] = 0; for (int b = 0; b < BS; ++b) o[a] += J[a * BS + b] * v[b]; }
    for (int a = 0; a < BS; ++a) M[(idx + a) * ld + j] = o[a];
  }
  __syncthreads();
}
template <int BS>
__device__ __forceinline__ void right_block_T(double* M, int ld, int nrows, int idx, const double* J) {
  for (int i = threadIdx.x; i < nrows; i += SV_T) {
    double v[BS], o[BS];
    for (int a = 0; a < BS; ++a) v[a] = M[i * ld + idx + a];
    for (int a = 0; a < BS; ++a) { o[a] = 0; for (int b = 0; b < BS; ++b) o[a] += v[b] * J[a * BS + b]; }
    for (int a = 0; a < BS; ++a) M[i * ld + idx + a] = o[a];
  }
  __syncthreads();
}

// write the final report + state + covariance into mapped host memory, then the done flag
__device__ void publish(const ScanCtl* c, double* h_out, volatile uint32_t* h_flag) {
  // layout: [0, ND*ND) P_out (n x n used) | state (64 doubles reserved) | dx_last (ND) | 10 ints (5 doubles) | flag (last 8 bytes of UPD_DOUBLES)
  const int n = c->n;
  for (int k = threadIdx.x; k < n * n; k += SV_T) h_out[k] = c->P_out[k];
  double* st = h_out + ND * ND;
  const double* xs = reinterpret_cast<const double*>(&c->x);
  for (int k = threadIdx.x; k < (int)(sizeof(malio_state) / sizeof(double)); k += SV_T) st[k] = xs[k];
  double* dl = st + 64;
  for (int k = threadIdx.x; k < ND; k += SV_T) dl[k] = c->dx_last[k];
  if (threadIdx.x == 0) {
    int32_t* r = reinterpret_cast<int32_t*>(dl + ND);
    r[0] = c->passes; r[1] = c->searches; r[2] = c->status; r[3] = c->need_host; r[4] = (int32_t)c->n_eff_last; r[5] = (int32_t)c->converged_count;
    r[6] = (int32_t)c->seq; r[7] = c->parity; r[8] = (int32_t)c->searched_mask; r[9] = 0;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) *h_flag = c->scan_id;
}

__global__ void __launch_bounds__(SV_T)
solve_kernel(ScanCtl* c, const double* __restrict__ d_res, uint32_t* bar, double* h_out, uint32_t* h_flag) {
  if (!c->active) return;
  extern __shared__ double sm[];
  const int n = c->n, nc = c->c, L = c->L;
  double* P = sm;                         // n x n (ld = n)
  double* G = P + ND * ND;                // c x c
  double* LU = G + NC * NC;               // c x c
  double* Y = LU + NC * NC;               // c x n  (final pass)
  double* Kx = Y + NC * ND;               // n x c
  double* Lm = Kx + ND * NC;              // n x n
  double* Gp = Lm + ND * ND;              // padded 24 x 28 system
  double* vec = Gp + MALIO_RED_ROWS * MALIO_RED_COLS;   // g[NC] | dx[ND] | dxn[ND] | Kh[ND] | KxDx[ND] | step[ND] | z1[NC] | z2[NC] | J[9*4+4]
  double* g = vec; double* dx = g + NC; double* dxn = dx + ND; double* Kh = dxn + ND; double* KxDx = Kh + ND; double* step = KxDx + ND;
  double* z1 = step + ND; double* z2 = z1 + NC; double* Jb = z2 + NC;
  __shared__ int s_piv[NC];
  __shared__ int s_flag[4];   // [0] finished, [1] singular, [2] redo_next
  __shared__ malio_state sx, sx0;   // working copies of x_ and x_propagated (the control block lives in global memory)
  const int tid = threadIdx.x;
  const StateLayout ly(L);
  {
    const double* a = reinterpret_cast<const double*>(&c->x);
    const double* b = reinterpret_cast<const double*>(&c->x_prop);
    double* da = reinterpret_cast<double*>(&sx);
    double* db = reinterpret_cast<double*>(&sx0);
    for (int k = tid; k < (int)(sizeof(malio_state) / sizeof(double)); k += SV_T) { da[k] = a[k]; db[k] = b[k]; }
  }
  const int max_iter = c->max_iter;
  const int t_in = c->t;

  // ---- the folded system -> padded 24 x 28 (measure()'s host epilogue), localization weight, compact c x c
  const uint32_t n_eff = (uint32_t)(d_res[MALIO_RED_BLOCKS * 16] + 0.5);
  for (int k = tid; k < MALIO_RED_ROWS * MALIO_RED_COLS; k += SV_T) Gp[k] = 0.0;
  __syncthreads();
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
    for (int e = tid; e < 12 * 16; e += SV_T) {
      const int a = e / 16, b = e % 16;
      // Gc[a][b]: upper-triangular 4x4 blocks are stored, the lower part of the 12 x 12 is the transpose
      int ra = a, rb = b;
      if (b < 12 && b < a) { ra = b; rb = a; }
      const int gi = ra / 4, gj = rb / 4;
      const int t = (gi == 0 ? 0 : (gi == 1 ? 3 : 5)) + gj;   // task index of block (gi, gj >= gi): rows 0: 0-3, 1: 4-6 (gj 1..3), 2: 7-8
      const double v = d_res[(l * 9 + t) * 16 + (ra % 4) * 4 + (rb % 4)];
      int ca, cb;
      ca = a < 6 ? a : (a < 9 ? 6 + 3 * l + (a - 6) : 15 + 3 * l + (a - 9));
      cb = b < 6 ? b : (b < 9 ? 6 + 3 * l + (b - 6) : (b < 12 ? 15 + 3 * l + (b - 9) : 24 + (b - 12)));
      Gp[ca * MALIO_RED_COLS + cb] += v;
    }
    __syncthreads();
  }
  if (tid == 0) {
    if (c->redo) { c->searches += 1; c->searched_mask |= 1u << c->passes; }
    c->passes += 1;
    s_flag[0] = 0; s_flag[1] = 0; s_flag[2] = 0;
  }
  __syncthreads();
  const int it = c->it;
  bool valid = n_eff >= 1;
  if (valid && n > (int)n_eff) {   // degenerate branch (esekfom.hpp:574-582): needs the dense rows -> the host finishes this scan
    if (tid == 0) { c->need_host = 1; c->active = 0; c->n_eff_last = n_eff; }
    __syncthreads();
    publish(c, h_out, h_flag);
    return;
  }
  if (valid) {
    // localization weight (laserMapping.cpp:745-759) and the compact system
    if (tid == 0) {
      const double S6[6] = {Gp[0 * MALIO_RED_COLS + 25], Gp[0 * MALIO_RED_COLS + 26], Gp[0 * MALIO_RED_COLS + 27], Gp[1 * MALIO_RED_COLS + 26],
                            Gp[1 * MALIO_RED_COLS + 27], Gp[2 * MALIO_RED_COLS + 27]};
      double sv[3];
      sym3_singular_values(S6, sv);
      double w = sv[2] / sv[0];
      if (w > c->loc_thresh_max) w = c->loc_cov_max;
      else if (w < c->loc_thresh_min) w = c->loc_cov_min;
      else w = (c->loc_cov_max - c->loc_cov_min) * (w - c->loc_thresh_min) / (c->loc_thresh_max - c->loc_thresh_min) + c->loc_cov_min;
      Jb[40] = w * w;
      c->n_eff_last = n_eff;
      // dx = x [-] x_prop (esekfom.hpp:526)
      boxminus(ly, sx, sx0, dx);
      for (int k = 0; k < n; ++k) dxn[k] = dx[k];
    }
    for (int k = tid; k < n * n; k += SV_T) P[k] = c->P_prop[k];   // :530
    __syncthreads();
    const double w2 = Jb[40];
    for (int e = tid; e < nc * nc; e += SV_T) {
      const int a = e / nc, b = e % nc;
      const int ma = a < 6 ? a : (a < 6 + 3 * L ? a : 15 + (a - (6 + 3 * L)));
      const int mb = b < 6 ? b : (b < 6 + 3 * L ? b : 15 + (b - (6 + 3 * L)));
      G[a * nc + b] = w2 * Gp[ma * MALIO_RED_COLS + mb];
    }
    for (int a = tid; a < nc; a += SV_T) {
      const int ma = a < 6 ? a : (a < 6 + 3 * L ? a : 15 + (a - (6 + 3 * L)));
      g[a] = w2 * Gp[ma * MALIO_RED_COLS + 24];
    }
    __syncthreads();
    // ---- projections of dx and P (esekfom.hpp:532-572)
    for (int s = 0; s <= L; ++s) {
      const int idx = ly.so3[s];
      if (tid == 0) {
        const M3 Jt = transpose3(A_matrix(&dx[idx]));
        for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) Jb[a * 3 + b] = Jt.m[a][b];
        double o[3];
        for (int a = 0; a < 3; ++a) o[a] = Jt.m[a][0] * dxn[idx] + Jt.m[a][1] * dxn[idx + 1] + Jt.m[a][2] * dxn[idx + 2];
        dxn[idx] = o[0]; dxn[idx + 1] = o[1]; dxn[idx + 2] = o[2];
      }
      __syncthreads();
      left_block<3>(P, n, idx, Jb, n);
      right_block_T<3>(P, n, n, idx, Jb);
    }
    {
      if (tid == 0) {
        double J2[2][2];
        S2_projection(sx.grav, sx0.grav, &dx[ly.grav], J2);
        Jb[0] = J2[0][0]; Jb[1] = J2[0][1]; Jb[2] = J2[1][0]; Jb[3] = J2[1][1];
        const double d0 = dxn[ly.grav], d1 = dxn[ly.grav + 1];
        dxn[ly.grav] = J2[0][0] * d0 + J2[0][1] * d1;
        dxn[ly.grav + 1] = J2[1][0] * d0 + J2[1][1] * d1;
      }
      __syncthreads();
      left_block<2>(P, n, ly.grav, Jb, n);
      right_block_T<2>(P, n, n, ly.grav, Jb);
    }
    for (int k = tid; k < n * n; k += SV_T) c->P_cur[k] = P[k];
    // ---- Mt = (I + G P_cc)^T, LU with partial pivoting (malio_host.cpp: same factorisation, same pivots)
    for (int e = tid; e < nc * nc; e += SV_T) {
      const int a = e / nc, b = e % nc;
      double s = 0.0;
      for (int k = 0; k < nc; ++k) s += G[b * nc + k] * P[a * n + k];
      LU[a * nc + b] = s + ((a == b) ? 1.0 : 0.0);
    }
    __syncthreads();
    // z1 = g, z2 = G dx_new (right-hand sides of S z = rhs)
    for (int k = tid; k < nc; k += SV_T) {
      z1[k] = g[k];
      double sdx = 0.0;
      for (int b = 0; b < nc; ++b) sdx += G[k * nc + b] * dxn[b];
      z2[k] = sdx;
    }
    __syncthreads();
    // LU of Mt with partial pivoting and the two transposed triangular solves, all inside warp 0: lane i owns row i (and
    // entry i of both right-hand sides); same pivots and the same elimination arithmetic as malio_host.cpp, no block barriers
    if (tid < 32) {
      const int lane = tid;
      for (int k = 0; k < nc; ++k) {
        // pivot: largest |LU[i][k]|, i >= k, the FIRST one on ties (the host's strict '>')
        double v = (lane >= k && lane < nc) ? fabs(LU[lane * nc + k]) : -1.0;
        int who = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double ov = __shfl_xor_sync(0xffffffffu, v, o);
          const int ow = __shfl_xor_sync(0xffffffffu, who, o);
          if (ov > v || (ov == v && ow < who)) { v = ov; who = ow; }
        }
        if (lane == 0) { s_piv[k] = who; if (v == 0.0) s_flag[1] = 1; }
        if (who != k && lane < nc) { const double t_ = LU[k * nc + lane]; LU[k * nc + lane] = LU[who * nc + lane]; LU[who * nc + lane] = t_; }
        __syncwarp();
        const double inv = 1.0 / LU[k * nc + k];
        if (lane > k && lane < nc) {
          const double f = LU[lane * nc + k] * inv;
          LU[lane * nc + k] = f;
          if (f != 0.0)
            for (int j = k + 1; j < nc; ++j) LU[lane * nc + j] -= f * LU[k * nc + j];
        }
        __syncwarp();
      }
      // S = Mt^T = U^T L^T Pm:  U^T w = rhs (forward), L^T v = w (backward, unit diagonal), z = Pm^T v
      double s1 = lane < nc ? z1[lane] : 0.0, s2 = lane < nc ? z2[lane] : 0.0;
      for (int i = 0; i < nc; ++i) {
        if (lane == i) { const double inv = 1.0 / LU[i * nc + i]; s1 = s1 * inv; s2 = s2 * inv; z1[i] = s1; z2[i] = s2; }
        __syncwarp();
        if (lane > i && lane < nc) { const double u = LU[i * nc + lane]; s1 -= u * z1[i]; s2 -= u * z2[i]; }
      }
      __syncwarp();
      for (int i = nc - 1; i >= 0; --i) {
        if (lane == i) { z1[i] = s1; z2[i] = s2; }
        __syncwarp();
        if (lane < i) { const double l_ = LU[i * nc + lane]; s1 -= l_ * z1[i]; s2 -= l_ * z2[i]; }
      }
      __syncwarp();
      if (lane == 0)
        for (int k = nc - 1; k >= 0; --k)
          if (s_piv[k] != k) { double t_ = z1[k]; z1[k] = z1[s_piv[k]]; z1[s_piv[k]] = t_; t_ = z2[k]; z2[k] = z2[s_piv[k]]; z2[s_piv[k]] = t_; }
    }
    __syncthreads();
    for (int a = tid; a < n; a += SV_T) {
      double s = 0.0, u = 0.0;
      for (int k = 0; k < nc; ++k) { s += P[a * n + k] * z1[k]; u += P[a * n + k] * z2[k]; }
      Kh[a] = s; KxDx[a] = u;
      step[a] = s + u - dxn[a];                       // dx_ = K_h + (K_x - I) dx_new, :642
    }
    __syncthreads();
    for (int k = tid; k < n; k += SV_T) c->dx_last[k] = step[k];
    if (tid == 0) {
      boxplus(ly, sx, step);                          // :646
      int redo = 1;                                   // :649-657
      for (int k = 0; k < n; ++k) if (fabs(step[k]) > 0.001) { redo = 0; break; }
      int t = t_in;
      if (redo) t++;
      if (!t && it == max_iter - 2) redo = 1;         // :660-663
      c->t = t;
      s_flag[3] = t;
      s_flag[2] = redo;
      s_flag[0] = (t > 1 || it == max_iter - 1) ? 1 : 0;   // :665
    }
    __syncthreads();
    {   // the new state goes back to the control block
      const double* a = reinterpret_cast<const double*>(&sx);
      double* ga = reinterpret_cast<double*>(&c->x);
      for (int k = tid; k < (int)(sizeof(malio_state) / sizeof(double)); k += SV_T) ga[k] = a[k];
    }
    if (s_flag[0]) {
      // ---- final covariance (:665-718): Q[:,0:c]^T = Mt^-1 P[:,0:c]^T from the stored factors, K_x = Q[:,0:c] G
      for (int e = tid; e < nc * n; e += SV_T) { const int a = e / n, j = e % n; Y[a * n + j] = P[a * n + j]; }
      __syncthreads();
      for (int k = 0; k < nc; ++k) {
        const int p = s_piv[k];
        if (p != k) for (int j = tid; j < n; j += SV_T) { const double t_ = Y[k * n + j]; Y[k * n + j] = Y[p * n + j]; Y[p * n + j] = t_; }
        __syncthreads();
      }
      for (int j = tid; j < n; j += SV_T) {           // one right-hand side per thread
        for (int k = 0; k < nc; ++k)
          for (int i = k + 1; i < nc; ++i) { const double f = LU[i * nc + k]; if (f != 0.0) Y[i * n + j] -= f * Y[k * n + j]; }
        for (int i = nc - 1; i >= 0; --i) {
          for (int k = i + 1; k < nc; ++k) { const double f = LU[i * nc + k]; if (f != 0.0) Y[i * n + j] -= f * Y[k * n + j]; }
          Y[i * n + j] *= 1.0 / LU[i * nc + i];
        }
      }
      __syncthreads();
      for (int e = tid; e < n * nc; e += SV_T) {
        const int a = e / nc, b = e % nc;
        double s = 0.0;
        for (int k = 0; k < nc; ++k) s += Y[k * n + a] * G[k * nc + b];
        Kx[a * nc + b] = s;
      }
      for (int k = tid; k < n * n; k += SV_T) Lm[k] = P[k];
      __syncthreads();
      for (int s = 0; s <= L; ++s) {
        const int idx = ly.so3[s];
        if (tid == 0) {
          const M3 Jt = transpose3(A_matrix(&step[idx]));
          for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) Jb[a * 3 + b] = Jt.m[a][b];
        }
        __syncthreads();
        for (int j = tid; j < n; j += SV_T) {         // L rows from P rows
          const double v0 = P[idx * n + j], v1 = P[(idx + 1) * n + j], v2 = P[(idx + 2) * n + j];
          for (int a = 0; a < 3; ++a) Lm[(idx + a) * n + j] = Jb[a * 3] * v0 + Jb[a * 3 + 1] * v1 + Jb[a * 3 + 2] * v2;
        }
        __syncthreads();
        left_block<3>(Kx, nc, idx, Jb, nc);
        right_block_T<3>(Lm, n, n, idx, Jb);
        right_block_T<3>(P, n, n, idx, Jb);
      }
      {
        if (tid == 0) {
          double J2[2][2];
          S2_projection(sx.grav, sx0.grav, &step[ly.grav], J2);
          Jb[0] = J2[0][0]; Jb[1] = J2[0][1]; Jb[2] = J2[1][0]; Jb[3] = J2[1][1];
        }
        __syncthreads();
        for (int j = tid; j < n; j += SV_T) {
          const double v0 = P[ly.grav * n + j], v1 = P[(ly.grav + 1) * n + j];
          Lm[ly.grav * n + j] = Jb[0] * v0 + Jb[1] * v1;
          Lm[(ly.grav + 1) * n + j] = Jb[2] * v0 + Jb[3] * v1;
        }
        __syncthreads();
        left_block<2>(Kx, nc, ly.grav, Jb, nc);
        right_block_T<2>(Lm, n, n, ly.grav, Jb);
        right_block_T<2>(P, n, n, ly.grav, Jb);
      }
      for (int e = tid; e < n * n; e += SV_T) {       // P_ = L_ - K_x[:,0:c] P_[0:c,:], :714
        const int a = e / n, b = e % n;
        double s = Lm[a * n + b];
        for (int k = 0; k < nc; ++k) s -= Kx[a * nc + k] * P[k * n + b];
        c->P_out[e] = s;
      }
      if (tid == 0) { c->converged_count = (uint32_t)s_flag[3]; c->status = s_flag[1] ? MALIO_ERR_INVALID_ARG : MALIO_OK; c->active = 0; }
      __syncthreads();
      publish(c, h_out, h_flag);
      return;
    }
  }
  // ---- another pass follows, or the loop is exhausted (only when the last pass was invalid)
  __syncthreads();
  if (it + 1 >= max_iter) {
    for (int k = tid; k < n * n; k += SV_T) c->P_out[k] = c->P_cur[k];
    if (tid == 0) { c->converged_count = (uint32_t)c->t; c->status = MALIO_ERR_NO_EFFECTIVE_POINTS; c->active = 0; }
    __syncthreads();
    publish(c, h_out, h_flag);
    return;
  }
  build_pc(c, sx);
  if (tid == 0) {
    if (valid) c->redo = s_flag[2];
    c->it = it + 1;
    c->seq += 1;
    c->parity ^= 1;
    bar[0] = 0; bar[1] = 0; bar[2] = 0;
    if (s_flag[1]) { c->status = MALIO_ERR_INVALID_ARG; }
  }
}

}  // namespace

namespace malio_solve {
constexpr size_t SOLVE_SMEM = (size_t)(ND * ND * 2 + NC * NC * 2 + NC * ND * 2 + MALIO_RED_ROWS * MALIO_RED_COLS + NC * 3 + ND * 5 + 48) * sizeof(double);

int setup(malio_handle* h) {
  CUDA_TRY(cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SOLVE_SMEM));
  return MALIO_OK;
}
int launch_init(malio_handle* h, cudaStream_t st, ScanCtl* d_ctl, uint32_t seq0, int parity, uint32_t* d_bar) {
  init_ctl_kernel<<<1, SV_T, 0, st>>>(d_ctl, seq0, parity, d_bar);
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}
int launch_solve(malio_handle* h, cudaStream_t st, ScanCtl* d_ctl, const double* d_res, uint32_t* d_bar, double* h_out_dev, uint32_t* h_flag_dev) {
  solve_kernel<<<1, SV_T, SOLVE_SMEM, st>>>(d_ctl, d_res, d_bar, h_out_dev, h_flag_dev);
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}
}  // namespace malio_solve
