// malio_reloc.cu — relocalization in a loaded prior map, sm_90a: the first pose of a drive found without a close guess, by an
// exact branch-and-bound over candidate yaws and a position lattice (malio_relocalize, malio_b200.h).  Cartographer's
// real-time correlative search made level-parallel:
//   rl_register_kernel  every scan point under every candidate rotation through body_to_world (the bits malio_world_register
//                       gives), stored as its base voxel floor((double)w / res), yaw-major; per-yaw finite counts, the voxels'
//                       bounding box and a flag for indices outside +-2^30
//   rl_occupy_kernel    level 0 of the occupancy pyramid: one bit per voxel of the box the lookups can reach, set from the
//                       prior's points
//   rl_dilate_kernel    level l from level l-1: the sliding OR G_l[v] = G_{l-1}[v] | G_{l-1}[v + 2^(l-1)] along each axis still
//                       split at l, so that G_l[v] = OR of G_0 over v + [0, 2^d) per axis (d = that axis' depth at level l)
//   rl_bound_kernel     one warp per node (yaw k, level l, lattice corner u): sum over the points of G_l[base_k(p) + u], which
//                       bounds the score of every leaf under the node; at level 0 it is the leaf's score, folded into one 64-bit
//                       atomicMax of (score << 32) | (0xFFFFFFFF - lexindex)
//   rl_expand_kernel    one block per chunk: prune (bound < max(best, 1)), sort the survivors by bound, write their children
// The host pops fixed-size chunks deepest level first, the highest bounds first, so that the search memory is one list of
// CHUNK * 8 nodes per level whatever the scene.  Compiled with -fmad=false like the rest of the library; the host code that
// builds the candidate rotations is compiled without FP contraction (Makefile).
#include <cuda_runtime.h>

#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>

#include "malio_device.cuh"

using namespace malio_devstate;

namespace {

constexpr int REG_T = 256;
constexpr int BOUND_T = 256;                 // 8 warps: one node each
constexpr int EXP_T = 1024;
constexpr uint32_t CHUNK = 2 * EXP_T;        // nodes per popped chunk (two per thread of the expansion block)
constexpr uint32_t FANOUT = 8;               // children per node at most (x, y and z split)
constexpr int32_t NONFINITE = INT32_MIN;     // base voxel x of a point whose registered coordinates are not all finite
constexpr int32_t VOX_LIM = 1 << 30;         // |voxel index| < 2^30
constexpr int64_t AXIS_LIM = 1ll << 31;      // voxels along one axis of the pyramid's box
constexpr uint32_t FLAG_RANGE = 1u;

struct Node { uint32_t k, ux, uy, uz, pb; };   // yaw, lattice corner (offset + half), the parent's bound

// ---------------------------------------------------------------------------------------------------- kernels
// yaw k = blockIdx.y (+ gridDim.y ...): the handle's PassConst with rot = q_k, in shared memory for body_to_world
__global__ void __launch_bounds__(REG_T) rl_register_kernel(const malio_scan_pt* __restrict__ pts, uint32_t n, const double* __restrict__ qk,
                                                            uint32_t n_yaw, PassConst pc0, double res, int3* __restrict__ base,
                                                            uint32_t* __restrict__ n_fin, int* __restrict__ small) {
  __shared__ PassConst pc;
  const uint32_t i = blockIdx.x * REG_T + threadIdx.x;
  const int lane = threadIdx.x & 31;
  for (uint32_t k = blockIdx.y; k < n_yaw; k += gridDim.y) {
    __syncthreads();
    if (threadIdx.x == 0) {
      pc = pc0;
      for (int c = 0; c < 4; ++c) pc.rot[c] = qk[4 * (size_t)k + c];
    }
    __syncthreads();
    bool fin = false;
    int3 b = make_int3(NONFINITE, 0, 0);
    if (i < n) {
      const malio_scan_pt p = pts[i];
      float w[3];
      body_to_world(pc, p.lidar, p.x, p.y, p.z, w);
      if (isfinite(w[0]) && isfinite(w[1]) && isfinite(w[2])) {
        const double f[3] = {floor((double)w[0] / res), floor((double)w[1] / res), floor((double)w[2] / res)};
        if (fabs(f[0]) < (double)VOX_LIM && fabs(f[1]) < (double)VOX_LIM && fabs(f[2]) < (double)VOX_LIM) {
          b = make_int3((int)f[0], (int)f[1], (int)f[2]);
          fin = true;
        } else {
          atomicOr(small, (int)FLAG_RANGE);
        }
      }
      base[(size_t)k * n + i] = b;
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, fin);
    const int mn[3] = {fin ? b.x : INT_MAX, fin ? b.y : INT_MAX, fin ? b.z : INT_MAX};
    const int mx[3] = {fin ? b.x : INT_MIN, fin ? b.y : INT_MIN, fin ? b.z : INT_MIN};
    int rmn[3], rmx[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) { rmn[a] = __reduce_min_sync(0xffffffffu, mn[a]); rmx[a] = __reduce_max_sync(0xffffffffu, mx[a]); }
    if (lane == 0 && bal) {
      atomicAdd(n_fin + k, (uint32_t)__popc(bal));
#pragma unroll
      for (int a = 0; a < 3; ++a) { atomicMin(small + 1 + a, rmn[a]); atomicMax(small + 4 + a, rmx[a]); }
    }
  }
}

// level 0: the bit of voxel o + v for every prior point in the box [o, o + e)
__global__ void __launch_bounds__(256) rl_occupy_kernel(const float4* __restrict__ pts, uint32_t n, double res, double o0, double o1,
                                                        double o2, uint32_t ex, uint32_t ey, uint32_t ez, uint32_t nxw,
                                                        uint32_t* __restrict__ g) {
  const uint32_t i = blockIdx.x * 256u + threadIdx.x;
  if (i >= n) return;
  const float4 p = pts[i];
  const double v0 = floor((double)p.x / res) - o0, v1 = floor((double)p.y / res) - o1, v2 = floor((double)p.z / res) - o2;
  if (!(v0 >= 0.0 && v0 < (double)ex && v1 >= 0.0 && v1 < (double)ey && v2 >= 0.0 && v2 < (double)ez)) return;
  const uint32_t x = (uint32_t)v0, y = (uint32_t)v1, z = (uint32_t)v2;
  atomicOr(g + ((size_t)z * ey + y) * nxw + (x >> 5), 1u << (x & 31));
}

// bits x + s .. x + s + 31 of a row of nxw words, for the word holding x = 32 xw ..
__device__ __forceinline__ uint32_t row_shift(const uint32_t* __restrict__ row, uint32_t xw, uint32_t s, uint32_t nxw) {
  const uint32_t ws = xw + (s >> 5), b = s & 31u;
  const uint32_t lo = ws < nxw ? row[ws] : 0u;
  if (b == 0) return lo;
  const uint32_t hi = ws + 1 < nxw ? row[ws + 1] : 0u;
  return (lo >> b) | (hi << (32u - b));
}

// dst[v] = OR of src over v + {0, sxy} (x and y, when sxy > 0) x {0, sz} (z, when sz > 0); beyond the box counts as empty, which
// no lookup reaches (the box holds every G_0 cell a node's window covers)
__global__ void __launch_bounds__(256) rl_dilate_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, uint32_t nxw,
                                                        uint32_t ey, uint32_t ez, uint32_t sxy, uint32_t sz) {
  const size_t w = (size_t)blockIdx.x * 256u + threadIdx.x;
  const size_t total = (size_t)nxw * ey * ez;
  if (w >= total) return;
  const uint32_t xw = (uint32_t)(w % nxw);
  const size_t r = w / nxw;
  const uint32_t y = (uint32_t)(r % ey), z = (uint32_t)(r / ey);
  uint32_t acc = 0;
  for (int iz = 0; iz < (sz ? 2 : 1); ++iz) {
    const uint32_t zz = z + (iz ? sz : 0u);
    if (zz >= ez) continue;
    for (int iy = 0; iy < (sxy ? 2 : 1); ++iy) {
      const uint32_t yy = y + (iy ? sxy : 0u);
      if (yy >= ey) continue;
      const uint32_t* row = src + ((size_t)zz * ey + yy) * nxw;
      acc |= row[xw];
      if (sxy) acc |= row_shift(row, xw, sxy, nxw);
    }
  }
  dst[w] = acc;
}

struct BoundArgs {
  const int3* base; uint32_t n;
  int bmin[3];                        // smallest finite base voxel: grid cell of base b + lattice corner u is (b - bmin) + u
  const uint32_t* g; uint32_t nxw, ey;
  uint32_t wxy, wz;
};
// nodes[j] (NULL: the top level, node j = yaw k0 + j at corner 0); a node whose parent's bound is below max(best, 1) is skipped
// (bound 0); leaf: fold the score instead of storing it.  ctr: [0] best (packed), [1] nodes bounded, [2] leaves scored, [3] best
// as the previous kernel left it: every skip of one launch sees the same threshold, so two runs bound the same nodes
__global__ void __launch_bounds__(BOUND_T) rl_bound_kernel(BoundArgs a, const Node* __restrict__ nodes, uint32_t k0, uint32_t m, int leaf,
                                                           uint32_t* __restrict__ bound, unsigned long long* __restrict__ ctr) {
  const uint32_t j = blockIdx.x * (BOUND_T / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= m) return;
  const Node nd = nodes ? nodes[j] : Node{k0 + j, 0, 0, 0, 0xFFFFFFFFu};
  const unsigned long long best = ctr[3];
  const uint32_t thr = (uint32_t)(best >> 32) > 1u ? (uint32_t)(best >> 32) : 1u;
  if (nd.pb < thr) {
    if (lane == 0 && !leaf) bound[j] = 0;
    return;
  }
  const int3* __restrict__ bk = a.base + (size_t)nd.k * a.n;
  uint32_t s = 0;
  for (uint32_t i = lane; i < a.n; i += 32) {
    const int3 b = bk[i];
    if (b.x == NONFINITE) continue;
    const uint32_t vx = (uint32_t)(b.x - a.bmin[0]) + nd.ux, vy = (uint32_t)(b.y - a.bmin[1]) + nd.uy, vz = (uint32_t)(b.z - a.bmin[2]) + nd.uz;
    s += (__ldg(a.g + ((size_t)vz * a.ey + vy) * a.nxw + (vx >> 5)) >> (vx & 31)) & 1u;
  }
  s = __reduce_add_sync(0xffffffffu, s);
  if (lane != 0) return;
  atomicAdd(ctr + 1, 1ull);
  if (!leaf) { bound[j] = s; return; }
  atomicAdd(ctr + 2, 1ull);
  if (s == 0) return;
  const unsigned long long lex = (((unsigned long long)nd.k * a.wz + nd.uz) * a.wxy + nd.uy) * a.wxy + nd.ux;
  atomicMax(ctr, ((unsigned long long)s << 32) | (0xFFFFFFFFull - lex));
}

// the m nodes of a chunk at a level above 0 -> the children of the survivors (bound >= max(best, 1)) at out[0 ..), the survivors
// in ascending (bound, chunk index) order, so that the list's tail holds the children of the highest bounds.  h: the children's
// half-size step on the split axes (sxy / sz = 0 where an axis is not split).  *n_out = children written.
__global__ void __launch_bounds__(EXP_T) rl_expand_kernel(const Node* __restrict__ nodes, uint32_t k0, uint32_t m,
                                                          const uint32_t* __restrict__ bound, const unsigned long long* __restrict__ ctr,
                                                          uint32_t sxy, uint32_t sz, uint32_t wxy, uint32_t wz, Node* __restrict__ out,
                                                          uint32_t* __restrict__ n_out) {
  using Sort = cub::BlockRadixSort<uint32_t, EXP_T, 2, uint32_t>;
  using Scan = cub::BlockScan<uint32_t, EXP_T>;
  __shared__ union { typename Sort::TempStorage sort; typename Scan::TempStorage scan; } tmp;
  const uint32_t best = (uint32_t)(ctr[0] >> 32);
  const uint32_t thr = best > 1u ? best : 1u;
  uint32_t key[2], val[2];
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const uint32_t j = threadIdx.x * 2 + it;
    const uint32_t b = j < m ? bound[j] : 0u;
    key[it] = b >= thr ? b : 0u;   // pruned and padding sort first and expand to nothing
    val[it] = j;
  }
  Sort(tmp.sort).Sort(key, val);
  __syncthreads();
  Node nd[2];
  uint32_t cnt[2], off[2], total;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    cnt[it] = 0;
    if (key[it]) {
      nd[it] = nodes ? nodes[val[it]] : Node{k0 + val[it], 0, 0, 0, 0};
      const uint32_t cx = (sxy && nd[it].ux + sxy < wxy) ? 2u : 1u, cy = (sxy && nd[it].uy + sxy < wxy) ? 2u : 1u;
      const uint32_t cz = (sz && nd[it].uz + sz < wz) ? 2u : 1u;
      cnt[it] = cx * cy * cz;
    }
  }
  Scan(tmp.scan).ExclusiveSum(cnt, off, total);
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    if (!cnt[it]) continue;
    uint32_t o = off[it];
    for (uint32_t dz = 0; dz < 2; ++dz)
      for (uint32_t dy = 0; dy < 2; ++dy)
        for (uint32_t dx = 0; dx < 2; ++dx) {
          const uint32_t ux = nd[it].ux + dx * sxy, uy = nd[it].uy + dy * sxy, uz = nd[it].uz + dz * sz;
          if ((dx && (!sxy || ux >= wxy)) || (dy && (!sxy || uy >= wxy)) || (dz && (!sz || uz >= wz))) continue;
          out[o++] = Node{nd[it].k, ux, uy, uz, key[it]};
        }
  }
  if (threadIdx.x == 0) *n_out = total;
}

// ---------------------------------------------------------------------------------------------------- host
int ceil_log2(uint64_t w) { int d = 0; while ((1ull << d) < w) ++d; return d; }

// every buffer of one call, released (after the drain in relocalize) before it returns
struct Scratch {
  DeviceBuffer<double> d_q;
  DeviceBuffer<int3> d_base;
  DeviceBuffer<uint32_t> d_fin, d_bound, d_nout;
  DeviceBuffer<int> d_small;
  DeviceBuffer<unsigned long long> d_ctr;
  DeviceBuffer<uint32_t> d_grid;
  DeviceBuffer<Node> d_list;
  size_t bytes() const {
    return d_q.bytes() + d_base.bytes() + d_fin.bytes() + d_bound.bytes() + d_nout.bytes() + d_small.bytes() + d_ctr.bytes() +
           d_grid.bytes() + d_list.bytes();
  }
};

int search(malio_handle* h, DeviceState* D, const malio_pass_state* s, const malio_reloc_args* a, const float4* prior, uint32_t n_prior,
           Scratch& S, malio_reloc_report* rep) {
  cudaStream_t st = D->stream;
  const uint32_t n = D->N, n_yaw = a->n_yaw;
  const uint64_t wxy = 2ull * a->half_xy + 1, wz = 2ull * a->half_z + 1;
  // the candidate rotations, q_yaw(theta_k) (x) s.rot (malio_b200.h, step 1)
  std::vector<double> q(4 * (size_t)n_yaw);
  for (uint32_t k = 0; k < n_yaw; ++k) malio_se3::q_yaw_mul(a->yaw_lo + (double)k * a->yaw_step, s->rot, &q[4 * (size_t)k]);
  malio_reloc_report r{};   // written to *rep only on success
  r.n_candidates = (uint64_t)n_yaw * wxy * wxy * wz;
  uint64_t best = 0;
  uint32_t n_fin_best = 0;
  if (int rc = S.d_small.allocate(h, st, 8)) return rc;
  if (int rc = S.d_ctr.allocate(h, st, 4)) return rc;
  if (int rc = S.d_q.allocate(h, st, q.size())) return rc;
  if (int rc = S.d_fin.allocate(h, st, n_yaw)) return rc;
  if (n) {
    if (int rc = S.d_base.allocate(h, st, (size_t)n_yaw * n)) return rc;
  }
  CUDA_TRY(cudaMemcpyAsync(S.d_q, q.data(), q.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  const int init[8] = {0, INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN, 0};
  CUDA_TRY(cudaMemcpyAsync(S.d_small, init, sizeof(init), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemsetAsync(S.d_fin, 0, (size_t)n_yaw * sizeof(uint32_t), st));
  CUDA_TRY(cudaMemsetAsync(S.d_ctr, 0, 4 * sizeof(unsigned long long), st));
  D->ctr.h2d_bytes += q.size() * sizeof(double) + sizeof(init);
  int small[8];
  std::memcpy(small, init, sizeof(small));
  if (n) {
    const PassConst pc = make_pass_const(h, D, s);   // extrinsics from s, the temporal compensation of the last upload
    const dim3 grid((n + REG_T - 1) / REG_T, n_yaw < 65535u ? n_yaw : 65535u);
    rl_register_kernel<<<grid, REG_T, 0, st>>>(D->d_pts, n, S.d_q, n_yaw, pc, a->res, S.d_base, S.d_fin, S.d_small);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 1;
    CUDA_TRY(cudaMemcpyAsync(small, S.d_small, 7 * sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    D->ctr.d2h_bytes += 7 * sizeof(int);
    if (small[0] & FLAG_RANGE) {
      h->err = "malio_relocalize: a registered scan point's voxel index lies outside +-2^30 (res too small for the scene)";
      return MALIO_ERR_CAPACITY;
    }
  }
  const bool any = small[1] <= small[4];   // a finite point under some yaw
  if (any) {
    // the box every lookup reaches: base voxels + lattice corner + the top window, per axis
    const int dxy = ceil_log2(wxy), dz = ceil_log2(wz);
    const int L = dxy > dz ? dxy : dz;
    int64_t e[3];
    for (int ax = 0; ax < 3; ++ax)
      e[ax] = (int64_t)small[4 + ax] - small[1 + ax] + (int64_t)(ax < 2 ? wxy : wz) + (1ll << (ax < 2 ? dxy : dz));
    const uint64_t nxw = (uint64_t)((e[0] + 31) / 32);
    const uint64_t level_words = nxw * (uint64_t)e[1] * (uint64_t)e[2];
    const long double pyr = (long double)level_words * 4.0L * (L + 1);
    if (e[0] >= AXIS_LIM || e[1] >= AXIS_LIM || e[2] >= AXIS_LIM || pyr > (long double)MALIO_RELOC_MAX_PYRAMID_BYTES) {
      h->err = "malio_relocalize: the occupancy pyramid needs " + std::to_string((double)pyr) + " bytes over a box of " +
               std::to_string(e[0]) + " x " + std::to_string(e[1]) + " x " + std::to_string(e[2]) +
               " voxels (limit MALIO_RELOC_MAX_PYRAMID_BYTES, 2^31 voxels per axis): a smaller box, scan or a coarser res";
      return MALIO_ERR_CAPACITY;
    }
    if (int rc = S.d_grid.allocate(h, st, level_words * (L + 1))) return rc;
    if (int rc = S.d_list.allocate(h, st, (size_t)(L > 0 ? L : 1) * CHUNK * FANOUT)) return rc;
    if (int rc = S.d_bound.allocate(h, st, CHUNK)) return rc;
    if (int rc = S.d_nout.allocate(h, st, 1)) return rc;
    auto grid_of = [&](int l) { return S.d_grid.data() + level_words * (size_t)l; };
    CUDA_TRY(cudaMemsetAsync(grid_of(0), 0, level_words * 4, st));
    const double o[3] = {(double)small[1] - (double)a->half_xy, (double)small[2] - (double)a->half_xy, (double)small[3] - (double)a->half_z};
    if (n_prior) {
      rl_occupy_kernel<<<(n_prior + 255) / 256, 256, 0, st>>>(prior, n_prior, a->res, o[0], o[1], o[2], (uint32_t)e[0], (uint32_t)e[1],
                                                               (uint32_t)e[2], (uint32_t)nxw, grid_of(0));
      D->ctr.kernel_launches += 1;
    }
    for (int l = 1; l <= L; ++l) {
      const uint32_t sxy = l <= dxy ? 1u << (l - 1) : 0u, sz = l <= dz ? 1u << (l - 1) : 0u;
      rl_dilate_kernel<<<(unsigned)((level_words + 255) / 256), 256, 0, st>>>(grid_of(l - 1), grid_of(l), (uint32_t)nxw, (uint32_t)e[1],
                                                                             (uint32_t)e[2], sxy, sz);
      D->ctr.kernel_launches += 1;
    }
    CUDA_TRY(cudaGetLastError());
    // the lattice corner u = offset + half: grid cell of a point's base b is (b - bmin) + u, since the box starts at bmin - half
    BoundArgs ba{S.d_base, n, {small[1], small[2], small[3]}, nullptr, (uint32_t)nxw, (uint32_t)e[1], (uint32_t)wxy, (uint32_t)wz};
    std::vector<uint32_t> cnt((size_t)(L > 0 ? L : 1), 0);
    auto list_of = [&](int l) { return S.d_list.data() + (size_t)l * CHUNK * FANOUT; };
    uint32_t k_next = 0;
    for (;;) {
      int l = 0;
      while (l < L && cnt[l] == 0) ++l;
      const Node* nodes;
      uint32_t m, k0 = 0;
      if (l < L) {                       // the deepest non-empty list: its tail, the children of the highest bounds
        m = cnt[l] < CHUNK ? cnt[l] : CHUNK;
        cnt[l] -= m;
        nodes = list_of(l) + cnt[l];
      } else if (k_next < n_yaw) {       // the top level: the next yaws, corner 0
        m = n_yaw - k_next < CHUNK ? n_yaw - k_next : CHUNK;
        k0 = k_next;
        k_next += m;
        nodes = nullptr;
      } else {
        break;
      }
      ba.g = grid_of(l);
      rl_bound_kernel<<<(m + BOUND_T / 32 - 1) / (BOUND_T / 32), BOUND_T, 0, st>>>(ba, nodes, k0, m, l == 0, S.d_bound, S.d_ctr);
      D->ctr.kernel_launches += 1;
      if (l == 0) {   // the next launch's threshold
        CUDA_TRY(cudaMemcpyAsync(S.d_ctr + 3, S.d_ctr.data(), sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
        continue;
      }
      const uint32_t sxy = l <= dxy ? 1u << (l - 1) : 0u, sz = l <= dz ? 1u << (l - 1) : 0u;
      rl_expand_kernel<<<1, EXP_T, 0, st>>>(nodes, k0, m, S.d_bound, S.d_ctr, sxy, sz, (uint32_t)wxy, (uint32_t)wz, list_of(l - 1) + cnt[l - 1],
                                            S.d_nout);
      CUDA_TRY(cudaGetLastError());
      D->ctr.kernel_launches += 1;
      uint32_t pushed = 0;
      CUDA_TRY(cudaMemcpyAsync(&pushed, S.d_nout, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      D->ctr.d2h_bytes += sizeof(uint32_t);
      cnt[l - 1] += pushed;   // the list below was empty: at most CHUNK * FANOUT children
    }
    CUDA_TRY(cudaGetLastError());
    unsigned long long ctr[3];
    CUDA_TRY(cudaMemcpyAsync(ctr, S.d_ctr, sizeof(ctr), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    D->ctr.d2h_bytes += sizeof(ctr);
    best = ctr[0];
    r.nodes_bounded = ctr[1];
    r.leaves_scored = ctr[2];
  }
  // the winner (the first candidate when nothing scores) and its yaw's finite count
  const uint32_t score = (uint32_t)(best >> 32);
  const uint64_t lex = score ? 0xFFFFFFFFull - (best & 0xFFFFFFFFull) : 0;
  const uint64_t ux = lex % wxy, uy = (lex / wxy) % wxy, uz = (lex / wxy / wxy) % wz, k = lex / wxy / wxy / wz;
  if (n) {
    CUDA_TRY(cudaMemcpyAsync(&n_fin_best, S.d_fin + k, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    D->ctr.d2h_bytes += sizeof(uint32_t);
  }
  r.yaw_index = (int32_t)k;
  r.offset[0] = (int32_t)((int64_t)ux - a->half_xy);
  r.offset[1] = (int32_t)((int64_t)uy - a->half_xy);
  r.offset[2] = (int32_t)((int64_t)uz - a->half_z);
  r.score = score;
  r.n_points = n_fin_best;
  std::memcpy(r.rot, &q[4 * (size_t)k], sizeof(r.rot));
  for (int i = 0; i < 3; ++i) r.pos[i] = s->pos[i] + (double)r.offset[i] * a->res;
  r.device_bytes = S.bytes();
  *rep = r;
  return MALIO_OK;
}

}  // namespace

namespace malio_reloc {

int relocalize(malio_handle* h, const malio_pass_state* s, const malio_reloc_args* a, malio_reloc_report* rep) {
  bool finite = std::isfinite(a->yaw_lo) && std::isfinite(a->yaw_step);
  for (int i = 0; i < 4; ++i) finite = finite && std::isfinite(s->rot[i]);
  for (int i = 0; i < 3; ++i) finite = finite && std::isfinite(s->pos[i]);
  if (a->n_yaw == 0 || !(a->res > 0.0) || !std::isfinite(a->res) || !finite) {
    h->err = "malio_relocalize: n_yaw must be > 0, res finite and > 0, yaw_lo / yaw_step / s.pos / s.rot finite";
    return MALIO_ERR_INVALID_ARG;
  }
  DeviceState* D = h->dev.get();
  const float* prior = nullptr;
  uint32_t n_prior = 0;
  if (malio_prior::points(h, &prior, &n_prior) != MALIO_OK) { h->err = "malio_relocalize before malio_prior_map_load"; return MALIO_ERR_STATE; }
  if (!D->scan_ready) { h->err = "malio_relocalize before a scan upload"; return MALIO_ERR_STATE; }
  if (D->comm) { h->err = "malio_relocalize: a communicator is attached (each rank holds only its block of the scan)"; return MALIO_ERR_STATE; }
  const unsigned __int128 w = 2 * (unsigned __int128)a->half_xy + 1;
  const unsigned __int128 n_cand = (unsigned __int128)a->n_yaw * w * w * (2 * (unsigned __int128)a->half_z + 1);
  if (n_cand > ((unsigned __int128)1 << 32)) { h->err = "malio_relocalize: more than 2^32 candidates"; return MALIO_ERR_CAPACITY; }
  if ((unsigned __int128)a->n_yaw * (D->N * sizeof(int3) + 4 * sizeof(double) + sizeof(uint32_t)) > MALIO_RELOC_MAX_INDEX_BYTES) {
    h->err = "malio_relocalize: the per-yaw voxel indices need more than MALIO_RELOC_MAX_INDEX_BYTES (fewer yaws or scan points)";
    return MALIO_ERR_CAPACITY;
  }
  CUDA_TRY(cudaSetDevice(D->device));
  Scratch S;
  const int rc = search(h, D, s, a, reinterpret_cast<const float4*>(prior), n_prior, S, rep);
  CUDA_TRY(cudaStreamSynchronize(D->stream));   // before the scratch goes back (its destructors do not drain)
  return rc;
}

}  // namespace malio_reloc

// relocalization in a loaded prior map (malio_b200.h, after the prior-map block)
extern "C" int malio_relocalize(malio_handle* h, const malio_pass_state* s, const malio_reloc_args* a, malio_reloc_report* rep) {
  if (!h || !s || !a || !rep) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_reloc::relocalize(h, s, a, rep);
}
