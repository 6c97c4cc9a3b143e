// malio_loop.cu — a stored scan registered against a submap of stored scans, sm_90a (include/malio_b200.h,
// malio_scan_store_match): the loop edges of malio_pose_graph_optimize (malio_posegraph.cpp).  Every device expression is a
// +, -, *, /, sqrt or floor on doubles and every sum has a fixed order, so tests/loop_ref.py restates the result bit for bit;
// the host part (the solve, the pose update, exp_se3) is built with -ffp-contract=off.
//   lp_key_kernel    a target row's voxel key at one level (non-finite rows: KEY_NONE; a key out of range raises the fault word)
//   lp_fit_kernel    per voxel: centroid, covariance, cyclic Jacobi, plane test (one thread per voxel, rows in row order)
//   lp_eval_kernel   per source point: correspondence, residual, the 29 sums of one inlier, a block's binary tree of them
//   lp_tree_kernel   the next levels of the binary tree over the block sums
// The rows come from malio_store's registration (the target under the stored states, the source in the body frame).
// The voxels are ordered by a CUB radix sort of (key, row) pairs (stable: each voxel's rows stay in row order) and looked up by
// binary search.  All scratch is local to the call and goes back before it returns.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

#include <chrono>
#include <cmath>
#include <cstring>
#include <string>

#include "malio_device.cuh"

using namespace malio_devstate;

namespace {

constexpr int LP_THREADS = 128;                    // one block tree over 128 entries
constexpr int NSUM = 29;                           // J^T J (21) | J^T r (6) | r^2 | 1
constexpr uint64_t KEY_NONE = ~0ull;               // a non-finite row: sorts last, never looked up
constexpr double KEY_LIM = (double)MALIO_MATCH_KEY_RANGE;
constexpr int KEY_BITS = 21;

struct Plane { double mu[3], n[3]; };

__device__ __forceinline__ uint64_t pack_key(double kx, double ky, double kz) {
  const uint64_t o = (uint64_t)MALIO_MATCH_KEY_RANGE;
  return (((uint64_t)(long long)kx + o) << (2 * KEY_BITS)) | (((uint64_t)(long long)ky + o) << KEY_BITS) | ((uint64_t)(long long)kz + o);
}
__device__ __forceinline__ bool in_range(double k) { return k >= -KEY_LIM && k < KEY_LIM; }

__global__ void __launch_bounds__(256) lp_key_kernel(const float4* __restrict__ rows, uint32_t n, double leaf, uint64_t* __restrict__ keys,
                                                     uint32_t* __restrict__ idx, uint32_t* __restrict__ fault) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n) return;
  const float4 r = rows[p];
  idx[p] = p;
  if (!(isfinite(r.x) && isfinite(r.y) && isfinite(r.z))) { keys[p] = KEY_NONE; return; }
  const double kx = floor((double)r.x / leaf), ky = floor((double)r.y / leaf), kz = floor((double)r.z / leaf);
  if (!(in_range(kx) && in_range(ky) && in_range(kz))) { keys[p] = KEY_NONE; atomicOr(fault, 1u); return; }
  keys[p] = pack_key(kx, ky, kz);
}

// the eigen-decomposition of the symmetric A (row-major, overwritten) by cyclic Jacobi: V's columns are the eigenvectors
__device__ void jacobi3(double A[9], double V[9]) {
  for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  const int P[3] = {0, 0, 1}, Q[3] = {1, 2, 2};
  for (int sweep = 0; sweep < MALIO_MATCH_JACOBI_SWEEPS; ++sweep)
    for (int e = 0; e < 3; ++e) {
      const int p = P[e], q = Q[e];
      const double apq = A[3 * p + q];
      if (apq == 0.0) continue;
      const double theta = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
      double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
      if (theta < 0.0) t = -t;
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      for (int k = 0; k < 3; ++k) {
        const double akp = A[3 * k + p], akq = A[3 * k + q];
        A[3 * k + p] = c * akp - s * akq;
        A[3 * k + q] = s * akp + c * akq;
        const double vkp = V[3 * k + p], vkq = V[3 * k + q];
        V[3 * k + p] = c * vkp - s * vkq;
        V[3 * k + q] = s * vkp + c * vkq;
      }
      for (int k = 0; k < 3; ++k) {
        const double apk = A[3 * p + k], aqk = A[3 * q + k];
        A[3 * p + k] = c * apk - s * aqk;
        A[3 * q + k] = s * apk + c * aqk;
      }
    }
}

// one thread per voxel v < *n_vox: rows row_of[off[v] .. off[v] + cnt[v]) in row order
__global__ void __launch_bounds__(128) lp_fit_kernel(const float4* __restrict__ rows, const uint32_t* __restrict__ row_of,
                                                     const uint64_t* __restrict__ keys, const uint32_t* __restrict__ cnt,
                                                     const uint32_t* __restrict__ off, const uint32_t* __restrict__ n_vox,
                                                     uint32_t min_points, double planarity, Plane* __restrict__ vox,
                                                     uint8_t* __restrict__ plane, uint32_t* __restrict__ n_plane) {
  const uint32_t v = blockIdx.x * 128u + threadIdx.x;
  if (v >= *n_vox) return;
  const uint32_t n = cnt[v], o = off[v];
  if (keys[v] == KEY_NONE || n < min_points) { plane[v] = 0; return; }
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  for (uint32_t i = 0; i < n; ++i) {
    const float4 r = rows[row_of[o + i]];
    s0 = s0 + (double)r.x; s1 = s1 + (double)r.y; s2 = s2 + (double)r.z;
  }
  const double dn = (double)n;
  const double mu[3] = {s0 / dn, s1 / dn, s2 / dn};
  double c00 = 0.0, c01 = 0.0, c02 = 0.0, c11 = 0.0, c12 = 0.0, c22 = 0.0;
  for (uint32_t i = 0; i < n; ++i) {
    const float4 r = rows[row_of[o + i]];
    const double d0 = (double)r.x - mu[0], d1 = (double)r.y - mu[1], d2 = (double)r.z - mu[2];
    c00 = c00 + d0 * d0; c01 = c01 + d0 * d1; c02 = c02 + d0 * d2;
    c11 = c11 + d1 * d1; c12 = c12 + d1 * d2; c22 = c22 + d2 * d2;
  }
  double A[9] = {c00 / dn, c01 / dn, c02 / dn, 0, c11 / dn, c12 / dn, 0, 0, c22 / dn};
  A[3] = A[1]; A[6] = A[2]; A[7] = A[5];
  double V[9];
  jacobi3(A, V);
  // order (value, index): i0 smallest, i1 middle
  const double lam[3] = {A[0], A[4], A[8]};
  int ord[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2 - a; ++b)
      if (lam[ord[b + 1]] < lam[ord[b]]) { const int t = ord[b]; ord[b] = ord[b + 1]; ord[b + 1] = t; }
  const bool ok = lam[ord[0]] <= planarity * lam[ord[1]];
  plane[v] = ok ? 1 : 0;
  if (!ok) return;
  Plane P;
  for (int k = 0; k < 3; ++k) { P.mu[k] = mu[k]; P.n[k] = V[3 * k + ord[0]]; }
  vox[v] = P;
  atomicAdd(n_plane, 1u);
}

struct Model {
  const uint64_t* keys;
  const Plane* vox;
  const uint8_t* plane;
  uint32_t n_vox;
  double leaf, leaf2, gate;
};
struct Pose { double R[9], p[3]; };

__device__ __forceinline__ int64_t find_key(const uint64_t* keys, uint32_t n, uint64_t k) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1; else hi = mid;
  }
  return (lo < n && keys[lo] == k) ? (int64_t)lo : -1;
}

// the tree over the first W (a power of two <= LP_THREADS) entries of each of the NSUM rows of sh, pairs of adjacent entries
__device__ __forceinline__ void block_tree(double (*sh)[LP_THREADS], uint32_t W, double* __restrict__ out) {
  const uint32_t t = threadIdx.x;
  for (uint32_t s = 1; s < W; s *= 2) {
    __syncthreads();
    const uint32_t i = 2 * s * t;
    if (i < W)
      for (int c = 0; c < NSUM; ++c) sh[c][i] = sh[c][i] + sh[c][i + s];
  }
  __syncthreads();
  if (t < NSUM) out[(size_t)blockIdx.x * NSUM + t] = sh[t][0];
}

__global__ void __launch_bounds__(LP_THREADS) lp_eval_kernel(const float4* __restrict__ src, uint32_t n, Model m, Pose ps, uint32_t W,
                                                             double* __restrict__ out) {
  __shared__ double sh[NSUM][LP_THREADS];
  const uint32_t t = threadIdx.x;
  const uint64_t i = (uint64_t)blockIdx.x * W + t;
  bool in = false;
  double J[6], r = 0.0;
  if (t < W && i < n) {
    const float4 bf = src[i];
    if (isfinite(bf.x) && isfinite(bf.y) && isfinite(bf.z)) {
      const double b[3] = {(double)bf.x, (double)bf.y, (double)bf.z};
      double w[3];
      for (int k = 0; k < 3; ++k) w[k] = ((ps.R[3 * k] * b[0] + ps.R[3 * k + 1] * b[1]) + ps.R[3 * k + 2] * b[2]) + ps.p[k];
      const double kb[3] = {floor(w[0] / m.leaf), floor(w[1] / m.leaf), floor(w[2] / m.leaf)};
      double best = 0.0;
      int64_t bv = -1;
      for (int dz = -1; dz <= 1; ++dz)
        for (int dy = -1; dy <= 1; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const double kx = kb[0] + dx, ky = kb[1] + dy, kz = kb[2] + dz;
            if (!(in_range(kx) && in_range(ky) && in_range(kz))) continue;
            const int64_t v = find_key(m.keys, m.n_vox, pack_key(kx, ky, kz));
            if (v < 0 || !m.plane[v]) continue;
            const Plane& P = m.vox[v];
            const double d0 = w[0] - P.mu[0], d1 = w[1] - P.mu[1], d2 = w[2] - P.mu[2];
            const double e = (d0 * d0 + d1 * d1) + d2 * d2;
            if (bv < 0 || e < best) { best = e; bv = v; }
          }
      if (bv >= 0 && best <= m.leaf2) {
        const Plane& P = m.vox[bv];
        const double d0 = w[0] - P.mu[0], d1 = w[1] - P.mu[1], d2 = w[2] - P.mu[2];
        r = (P.n[0] * d0 + P.n[1] * d1) + P.n[2] * d2;
        if (fabs(r) <= m.gate) {
          in = true;
          double mm[3];
          for (int k = 0; k < 3; ++k) mm[k] = (ps.R[k] * P.n[0] + ps.R[3 + k] * P.n[1]) + ps.R[6 + k] * P.n[2];
          malio_se3::cross3(b, mm, J);
          J[3] = mm[0]; J[4] = mm[1]; J[5] = mm[2];
        }
      }
    }
  }
  int c = 0;
  for (int a = 0; a < 6; ++a)
    for (int b = a; b < 6; ++b) sh[c++][t] = in ? J[a] * J[b] : 0.0;
  for (int a = 0; a < 6; ++a) sh[c++][t] = in ? J[a] * r : 0.0;
  sh[c++][t] = in ? r * r : 0.0;
  sh[c][t] = in ? 1.0 : 0.0;
  block_tree(sh, W, out);
}

__global__ void __launch_bounds__(LP_THREADS) lp_tree_kernel(const double* __restrict__ in, uint32_t W, double* __restrict__ out) {
  __shared__ double sh[NSUM][LP_THREADS];
  const uint32_t t = threadIdx.x;
  for (int c = 0; c < NSUM; ++c) sh[c][t] = t < W ? in[((size_t)blockIdx.x * W + t) * NSUM + c] : 0.0;
  block_tree(sh, W, out);
}

__global__ void lp_finite_kernel(const float4* __restrict__ rows, uint32_t n, unsigned long long* __restrict__ cnt) {
  uint32_t k = 0;
  for (uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (uint64_t)gridDim.x * blockDim.x) {
    const float4 r = rows[p];
    k += (isfinite(r.x) && isfinite(r.y) && isfinite(r.z)) ? 1u : 0u;
  }
  const uint32_t s = __reduce_add_sync(0xFFFFFFFFu, k);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(cnt, (unsigned long long)s);
}

// drains the handle's stream when the call's scratch goes out of scope (declared after the buffers: destroyed before them)
struct Drain {
  cudaStream_t st;
  ~Drain() { cudaStreamSynchronize(st); }
};

uint64_t pow2_at_least(uint64_t n) {
  uint64_t p = 1;
  while (p < n) p *= 2;
  return p;
}

bool finite_pos(double v) { return std::isfinite(v) && v > 0.0; }

int check_args(malio_handle* h, const malio_match_args* a) {
  if (a->n_levels == 0 || a->n_levels > MALIO_MATCH_MAX_LEVELS) {
    h->err = "malio_scan_store_match: n_levels must be 1.." + std::to_string(MALIO_MATCH_MAX_LEVELS);
    return MALIO_ERR_INVALID_ARG;
  }
  for (uint32_t l = 0; l < a->n_levels; ++l)
    if (!finite_pos(a->leaf[l]) || !finite_pos(a->gate[l])) {
      h->err = "malio_scan_store_match: every level's leaf and gate must be finite and > 0";
      return MALIO_ERR_INVALID_ARG;
    }
  if (!finite_pos(a->sigma) || !finite_pos(a->planarity)) {
    h->err = "malio_scan_store_match: sigma and planarity must be finite and > 0";
    return MALIO_ERR_INVALID_ARG;
  }
  if (a->max_iter == 0) { h->err = "malio_scan_store_match: max_iter must be > 0"; return MALIO_ERR_INVALID_ARG; }
  return MALIO_OK;
}

// LL^T of the symmetric 6 x 6 A (row-major), solving A x = b; false on a pivot <= 0 (the order of tests/loop_ref.py's cholesky_solve)
bool cholesky_solve6(const double A[36], const double b[6], double x[6]) {
  double L[36] = {0};
  for (int j = 0; j < 6; ++j) {
    double s = A[6 * j + j];
    for (int k = 0; k < j; ++k) s = s - L[6 * j + k] * L[6 * j + k];
    if (!(s > 0.0)) return false;
    const double d = std::sqrt(s);
    L[6 * j + j] = d;
    for (int i = j + 1; i < 6; ++i) {
      double t = A[6 * i + j];
      for (int k = 0; k < j; ++k) t = t - L[6 * i + k] * L[6 * j + k];
      L[6 * i + j] = t / d;
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double t = b[i];
    for (int k = 0; k < i; ++k) t = t - L[6 * i + k] * y[k];
    y[i] = t / L[6 * i + i];
  }
  for (int i = 5; i >= 0; --i) {
    double t = y[i];
    for (int k = i + 1; k < 6; ++k) t = t - L[6 * k + i] * x[k];
    x[i] = t / L[6 * i + i];
  }
  return true;
}

// the symmetric 6 x 6 of the 21 upper-triangle sums (row-major, i <= j)
void full6(const double* ut, double A[36]) {
  int c = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) { A[6 * i + j] = ut[c]; A[6 * j + i] = ut[c]; ++c; }
}

// the smallest eigenvalue of the symmetric 6 x 6 A (cyclic Jacobi to convergence; a tolerance result)
double eig_min6(const double A0[36]) {
  double A[36];
  std::memcpy(A, A0, sizeof(A));
  for (int sweep = 0; sweep < 50; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 6; ++p)
      for (int q = p + 1; q < 6; ++q) off += A[6 * p + q] * A[6 * p + q];
    if (off == 0.0) break;
    for (int p = 0; p < 6; ++p)
      for (int q = p + 1; q < 6; ++q) {
        const double apq = A[6 * p + q];
        if (apq == 0.0) continue;
        const double theta = (A[6 * q + q] - A[6 * p + p]) / (2.0 * apq);
        double t = 1.0 / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        if (theta < 0.0) t = -t;
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 6; ++k) {
          const double akp = A[6 * k + p], akq = A[6 * k + q];
          A[6 * k + p] = c * akp - s * akq;
          A[6 * k + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 6; ++k) {
          const double apk = A[6 * p + k], aqk = A[6 * q + k];
          A[6 * p + k] = c * apk - s * aqk;
          A[6 * q + k] = s * apk + c * aqk;
        }
      }
  }
  double m = A[0];
  for (int i = 1; i < 6; ++i) m = std::fmin(m, A[7 * i]);
  return m;
}

// q <- normalize(q (x) quat_from_R(R(exp_se3(delta)))), p <- p + q_rot(q_old, t(exp_se3(delta)))
void right_update(double q[4], double p[3], const double delta[6]) {
  double T[16];
  malio_se3::exp_se3(delta, T);
  const double Rm[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  double qd[4], qn[4], dp[3];
  malio_se3::quat_from_R(Rm, qd);
  malio_se3::q_mul(q, qd, qn);
  const double td[3] = {T[3], T[7], T[11]};
  malio_se3::q_rot(q, td, dp);
  const double nrm = std::sqrt(((qn[0] * qn[0] + qn[1] * qn[1]) + qn[2] * qn[2]) + qn[3] * qn[3]);
  for (int i = 0; i < 4; ++i) q[i] = qn[i] / nrm;
  for (int i = 0; i < 3; ++i) p[i] = p[i] + dp[i];
}

}  // namespace

namespace malio_loop {

int match(malio_handle* h, uint64_t source, uint64_t anchor, const malio_pass_state* guess, const malio_match_args* a,
          malio_match_report* rep) {
  if (int rc = check_args(h, a)) return rc;
  const uint64_t n_scans = malio_store::count(h);
  if (source >= n_scans || anchor >= n_scans) {
    h->err = "malio_scan_store_match: source or anchor beyond the store (" + std::to_string(n_scans) + " scans)";
    return MALIO_ERR_INVALID_ARG;
  }
  if (a->target_count == 0 || a->target_first >= n_scans || a->target_count > n_scans - a->target_first) {
    h->err = "malio_scan_store_match: the target range is empty or beyond the store";
    return MALIO_ERR_INVALID_ARG;
  }
  if (anchor < a->target_first || anchor - a->target_first >= a->target_count) {
    h->err = "malio_scan_store_match: the anchor lies outside the target range";
    return MALIO_ERR_INVALID_ARG;
  }
  const malio_store::View sv = malio_store::view(h, source);
  double q[4], p[3];
  const malio_pass_state& g0 = guess ? *guess : sv.rec->state;
  for (int i = 0; i < 4; ++i) q[i] = g0.rot[i];
  for (int i = 0; i < 3; ++i) p[i] = g0.pos[i];
  for (double v : {q[0], q[1], q[2], q[3], p[0], p[1], p[2]})
    if (!std::isfinite(v)) { h->err = "malio_scan_store_match: the guess is not finite"; return MALIO_ERR_INVALID_ARG; }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  if (D->comm) { h->err = "malio_scan_store_match: a communicator is attached (each rank stores only its block of a scan)"; return MALIO_ERR_STATE; }

  uint64_t nt64 = 0;
  for (uint64_t k = a->target_first; k < a->target_first + a->target_count; ++k) nt64 += malio_store::view(h, k).rows;
  if (nt64 >= 0x80000000ull) { h->err = "malio_scan_store_match: 2^31 or more target rows"; return MALIO_ERR_CAPACITY; }
  const uint32_t nt = (uint32_t)nt64, ns = (uint32_t)sv.rows;
  const uint64_t P = pow2_at_least(ns ? ns : 1);
  const uint32_t W0 = (uint32_t)(P < LP_THREADS ? P : LP_THREADS);
  const uint64_t blocks0 = P / W0;
  cudaStream_t st = D->stream;

  // scratch: the rows, the sort's pairs (two buffers each), the voxels, the sums
  DeviceBuffer<float4> d_t, d_s;
  DeviceBuffer<uint64_t> d_key, d_uk;
  DeviceBuffer<uint32_t> d_idx, d_cnt, d_off, d_word;
  DeviceBuffer<Plane> d_vox;
  DeviceBuffer<uint8_t> d_plane;
  DeviceBuffer<double> d_red;
  DeviceBuffer<unsigned long long> d_fin;
  const size_t nt1 = nt ? nt : 1;
  malio_buf::CubTemp cub_temp;
  uint64_t bytes = (uint64_t)nt1 * (sizeof(float4) + 2 * 8 + 8 + 2 * 4 + 4 + 4 + sizeof(Plane) + 1) + (uint64_t)(ns ? ns : 1) * sizeof(float4) +
                   2 * blocks0 * NSUM * sizeof(double) + 64;
  if (bytes > MALIO_MATCH_MAX_BYTES) {
    h->err = "malio_scan_store_match: the call needs " + std::to_string(bytes) + " bytes of scratch, above MALIO_MATCH_MAX_BYTES";
    return MALIO_ERR_CAPACITY;
  }
  if (int rc = malio_buf::allocate_group(h, st, {{d_t, nt1}, {d_s, (size_t)(ns ? ns : 1)}, {d_key, 2 * nt1}, {d_uk, nt1}, {d_idx, 2 * nt1},
                                                 {d_cnt, nt1}, {d_off, nt1}, {d_word, (size_t)4}, {d_vox, nt1}, {d_plane, nt1},
                                                 {d_red, (size_t)(2 * blocks0 * NSUM)}, {d_fin, (size_t)1}}))
    return rc;
  Drain drain{st};
  uint64_t launches = 0, d2h = 0;

  // the rows: the target under the stored states, the source in the body frame (malio_store's registration)
  uint64_t at = 0;
  for (uint64_t k = a->target_first; k < a->target_first + a->target_count; ++k) {
    const uint64_t rows = malio_store::view(h, k).rows;
    if (int rc = malio_store::enqueue_register(h, k, nullptr, rows, reinterpret_cast<float*>(d_t.data() + at))) return rc;
    at += rows;
  }
  malio_pass_state body = sv.rec->state;
  body.rot[0] = 1.0; body.rot[1] = 0.0; body.rot[2] = 0.0; body.rot[3] = 0.0;
  body.pos[0] = 0.0; body.pos[1] = 0.0; body.pos[2] = 0.0;
  if (int rc = malio_store::enqueue_register(h, source, &body, ns, reinterpret_cast<float*>(d_s.data()))) return rc;
  CUDA_TRY(cudaMemsetAsync(d_fin, 0, sizeof(unsigned long long), st));
  if (ns) {
    lp_finite_kernel<<<(ns + 255) / 256 < 1024 ? (ns + 255) / 256 : 1024, 256, 0, st>>>(d_s, ns, d_fin);
    ++launches;
    CUDA_TRY(cudaGetLastError());
  }

  cub::DoubleBuffer<uint64_t> kb(d_key.data(), d_key.data() + nt1);
  cub::DoubleBuffer<uint32_t> vb(d_idx.data(), d_idx.data() + nt1);
  auto sort_call = [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, kb, vb, (int)nt, 0, 64, st); };
  auto rle_call = [&](void* t, size_t& b) {
    return cub::DeviceRunLengthEncode::Encode(t, b, kb.Current(), d_uk.data(), d_cnt.data(), d_word.data(), (int)nt, st);
  };
  auto scan_call = [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_cnt.data(), d_off.data(), (int)nt, st); };
  if (nt) {
    if (int rc = cub_temp.reserve(h, st, sort_call, rle_call, scan_call)) return rc;
  }
  bytes += cub_temp.bytes();

  // one evaluation at level l under (q, p): the 29 sums
  uint32_t n_vox = 0;
  Model m{};
  auto evaluate = [&](double sums[NSUM]) -> int {
    Pose ps{};
    malio_se3::q_to_R(q, ps.R);
    for (int i = 0; i < 3; ++i) ps.p[i] = p[i];
    double* in = d_red.data();
    double* out = d_red.data() + blocks0 * NSUM;
    lp_eval_kernel<<<(unsigned)blocks0, LP_THREADS, 0, st>>>(d_s, ns, m, ps, W0, in);
    ++launches;
    CUDA_TRY(cudaGetLastError());
    for (uint64_t M = blocks0; M > 1;) {
      const uint32_t W = (uint32_t)(M < LP_THREADS ? M : LP_THREADS);
      lp_tree_kernel<<<(unsigned)(M / W), LP_THREADS, 0, st>>>(in, W, out);
      ++launches;
      CUDA_TRY(cudaGetLastError());
      std::swap(in, out);
      M /= W;
    }
    CUDA_TRY(cudaMemcpyAsync(sums, in, NSUM * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    d2h += NSUM * sizeof(double);
    return (int)MALIO_OK;
  };
  // the plane model of level l
  auto build_model = [&](uint32_t l, uint64_t* n_plane) -> int {
    const double leaf = (double)a->leaf[l];
    CUDA_TRY(cudaMemsetAsync(d_word, 0, 4 * sizeof(uint32_t), st));
    n_vox = 0;
    if (nt) {
      kb.selector = 0; vb.selector = 0;
      lp_key_kernel<<<(nt + 255) / 256, 256, 0, st>>>(d_t, nt, leaf, kb.Current(), vb.Current(), d_word.data() + 2);
      CUDA_TRY(cudaGetLastError());
      if (int rc = cub_temp.run(h, sort_call)) return rc;
      CUDA_TRY(cudaMemsetAsync(d_cnt, 0, nt * sizeof(uint32_t), st));
      if (int rc = cub_temp.run(h, rle_call)) return rc;
      if (int rc = cub_temp.run(h, scan_call)) return rc;
      lp_fit_kernel<<<(nt + 127) / 128, 128, 0, st>>>(d_t, vb.Current(), d_uk, d_cnt, d_off, d_word, a->min_points, a->planarity, d_vox,
                                                      d_plane, d_word.data() + 1);
      CUDA_TRY(cudaGetLastError());
      launches += 5;
    }
    uint32_t w[4];
    CUDA_TRY(cudaMemcpyAsync(w, d_word, sizeof(w), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    d2h += sizeof(w);
    if (w[2]) {
      h->err = "malio_scan_store_match: a target row's voxel key at leaf " + std::to_string(a->leaf[l]) + " lies outside [-2^20, 2^20)";
      return (int)MALIO_ERR_CAPACITY;
    }
    n_vox = w[0];
    *n_plane = w[1];
    m = Model{d_uk.data(), d_vox.data(), d_plane.data(), n_vox, leaf, leaf * leaf, (double)a->gate[l]};
    return (int)MALIO_OK;
  };

  malio_match_report R{};
  R.target_points = nt;
  double sums[NSUM];
  for (uint32_t l = 0; l < a->n_levels; ++l) {
    if (int rc = build_model(l, &R.target_voxels[l])) return rc;
    bool done = false;
    for (uint32_t it = 0; it < a->max_iter && !done; ++it) {
      if (int rc = evaluate(sums)) return rc;
      double A[36], b[6], delta[6];
      full6(sums, A);
      for (int i = 0; i < 6; ++i) b[i] = -sums[21 + i];
      if (sums[28] < 6.0 || !cholesky_solve6(A, b, delta)) break;
      right_update(q, p, delta);
      R.iterations[l] = it + 1;
      done = true;
      for (int i = 0; i < 6; ++i)
        if (!(std::fabs(delta[i]) < (i < 3 ? a->eps_rot : a->eps_pos))) done = false;
    }
    R.converged = done ? 1 : 0;   // the finest level's: the coarser ones only bring the pose into its basin
  }
  // the report at the final pose, finest level (its model is the current one)
  if (int rc = evaluate(sums)) return rc;
  unsigned long long fin = 0;
  CUDA_TRY(cudaMemcpyAsync(&fin, d_fin, sizeof(fin), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  d2h += sizeof(fin);
  double A[36];
  full6(sums, A);
  const double s2 = a->sigma * a->sigma;
  for (int i = 0; i < 36; ++i) R.info[i] = A[i] / s2;
  R.n_inliers = (uint32_t)sums[28];
  R.n_points = (uint32_t)fin;
  R.rms = sums[28] > 0.0 ? std::sqrt(sums[27] / sums[28]) : 0.0;
  R.fitness = fin ? sums[28] / (double)fin : 0.0;
  R.eig_min = eig_min6(R.info);
  for (int i = 0; i < 4; ++i) R.rot[i] = q[i];
  for (int i = 0; i < 3; ++i) R.pos[i] = p[i];
  const malio_pass_state& sa = malio_store::view(h, anchor).rec->state;
  const double qa_conj[4] = {sa.rot[0], -sa.rot[1], -sa.rot[2], -sa.rot[3]};
  malio_se3::q_mul(qa_conj, q, R.rel_rot);
  const double dp[3] = {p[0] - sa.pos[0], p[1] - sa.pos[1], p[2] - sa.pos[2]};
  malio_se3::q_rot_conj(sa.rot, dp, R.rel_pos);
  R.device_bytes = bytes;
  D->ctr.kernel_launches += launches;
  D->ctr.d2h_bytes += d2h;
  *rep = R;
  return MALIO_OK;
}

}  // namespace malio_loop

// loop closure over the scan store (malio_b200.h, after malio_world_voxel_rebuild)
extern "C" int malio_scan_store_match(malio_handle* h, uint64_t source, uint64_t anchor, const malio_pass_state* guess,
                                      const malio_match_args* a, malio_match_report* rep) {
  if (!h || !a || !rep) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_loop::match(h, source, anchor, guess, a, rep);
}
