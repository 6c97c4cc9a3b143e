// malio_mapops.cu — SURVEY.md §8f N1: the map as a device-resident point set kept in step with the host's ikd-Tree by
// deltas (host side and reasoning: include/malio_mapsync.hpp), sm_90a.
//
// Reference calls mirrored (paths relative to /root/reference/MA_LIO/include/ikd-Tree):
//   KD_TREE::Build                ikd_Tree.cpp:370-424     -> build()
//   KD_TREE::Delete_Point_Boxes   :648-676, Delete_by_range :785-857   -> delete_boxes()   (half-open boxes, :807)
//   KD_TREE::Add_Points(.,false)  :478-584, Add_by_point :982-1042     -> add_points()
//   KD_TREE::Add_Points(.,true)   + KD_TREE::Box_Search per touched voxel (:464-468, Search_by_range :1257-1296) -> sync_voxels()
//
// Storage: slots in DeviceState::d_mpts (x, y, z, link word = MALIO_LINK_POINT_DELETED or 0), d_cov (normal_y), d_ids.
// Deltas append slots and set deleted bits; nothing moves until a commit finds more than half of the slots dead, then a
// stable compaction packs the live ones.  commit() = bounding box of the live points (one reduction, 24 B back to the host
// for the grid geometry) + the same five-kernel cell-list build a snapshot upload runs (malio_knn.cu: grid_build).
// Killing the content of a voxel box uses the CURRENT index (cells overlapping the box, exact half-open test per point),
// so a sync after uncommitted appends commits first; boxes of one call are distinct voxels and cannot see each other's points.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <vector>

#include "malio_device.cuh"

using namespace malio_devstate;

namespace malio_map {

struct MapOps {
  uint32_t n_slots = 0, n_live = 0;
  bool dirty = false;            // slots changed since the index was built
  bool appended = false;         // ... by appends (those are invisible to the index until the next commit)
  bool active = false;           // a build() happened: the handle is in device-resident map mode
  DeviceBuffer<float> d_stage;     // staged host input, 5 rows of size() / 5: xyz (3 rows) | normal_y | ids
  DeviceBuffer<float> d_boxes;
  DeviceBuffer<uint32_t> d_small;   // [0..5] bbox keys, [6] kill counter, [7] live counter
  PinnedBuffer<uint32_t> h_small;   // pinned mirror
  DeviceBuffer<uint32_t> d_blk, d_blkoff;   // compaction: live count / offset per 1024-slot block
  DeviceBuffer<float4> d_mpts2; DeviceBuffer<float> d_cov2; DeviceBuffer<int32_t> d_ids2;   // compaction targets
  // small batches (the per-scan deltas) go through a pinned bounce buffer: one host memcpy, one H2D, and the call returns
  // without waiting for the device — the caller's arrays are consumed, the bounce buffer is protected by ev_bounce
  PinnedBuffer<float> h_bounce[2]; cudaEvent_t ev_bounce[2] = {nullptr, nullptr}; bool bounce_busy[2] = {false, false}; int bounce_next = 0;
  PinnedBuffer<float> h_bounce_box; cudaEvent_t ev_bounce_box = nullptr; bool bounce_box_busy = false;   // same for the voxel boxes

  int init(malio_handle* h, DeviceState* D) {
    if (int rc = d_small.allocate(h, D->stream, 8)) return rc;
    return h_small.allocate(h, 8);
  }
  ~MapOps() {
    for (cudaEvent_t e : ev_bounce) if (e) cudaEventDestroy(e);
    if (ev_bounce_box) cudaEventDestroy(ev_bounce_box);
  }
};

}  // namespace malio_map

namespace {

using malio_map::MapOps;

constexpr uint32_t BOUNCE_POINTS = 65536;      // 5 floats per point: 1.3 MB of pinned memory
constexpr uint32_t BOUNCE_BOXES = 16384;       // 6 floats per box

__device__ __forceinline__ uint32_t fkey(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
inline float fkey_inv(uint32_t k) {
  const uint32_t b = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

// staged host arrays -> slots [at, at + n)
__global__ void append_kernel(const float* __restrict__ xyz, const float* __restrict__ ny, const int32_t* __restrict__ ids, uint32_t n,
                              uint32_t at, int32_t id_base, float4* __restrict__ mpts, float* __restrict__ cov, int32_t* __restrict__ out_ids) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  mpts[at + i] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], __uint_as_float(0u));
  cov[at + i] = ny[i];
  out_ids[at + i] = ids ? ids[i] : id_base + (int32_t)i;
}
// Delete_Point_Boxes: few, large boxes -> every slot tests every box (Delete_by_range's point test, ikd_Tree.cpp:807)
constexpr int MAX_BIG_BOXES = 16;
struct BigBoxes { float b[MAX_BIG_BOXES][6]; int nb; };
__global__ void kill_big_boxes_kernel(float4* __restrict__ mpts, uint32_t n_slots, BigBoxes B, uint32_t* __restrict__ killed) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = false;
  if (i < n_slots) {
    const float4 a = mpts[i];
    if (!(__float_as_uint(a.w) & MALIO_LINK_POINT_DELETED)) {
      for (int k = 0; k < B.nb; ++k)
        hit |= (B.b[k][0] <= a.x && B.b[k][3] > a.x && B.b[k][1] <= a.y && B.b[k][4] > a.y && B.b[k][2] <= a.z && B.b[k][5] > a.z);
      if (hit) mpts[i].w = __uint_as_float(__float_as_uint(a.w) | MALIO_LINK_POINT_DELETED);
    }
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && bal) atomicAdd(killed, (uint32_t)__popc(bal));
}
// sync_voxels: many small boxes -> one WARP per box; the lanes take the x-rows of cells the box overlaps (the index holds every
// live point that existed at the last commit) and kill what lies inside (Search_by_range's test, ikd_Tree.cpp:1270).  A thread
// per box was 95 us for 2000 boxes (16 blocks of dependent cell_start -> point -> slot loads); boxes are disjoint voxels, so a
// slot is written by one lane only.
// COUNT: the same walk counts the live points of each box into out[k] and changes nothing (malio_prior_map_extend's admission);
// otherwise out is the kill counter.
constexpr int KV_T = 128;
template <bool COUNT>
__global__ void __launch_bounds__(KV_T) kill_voxel_boxes_kernel(const float* __restrict__ boxes, uint32_t nb, GridConst G,
                                                                const uint32_t* __restrict__ cell_start, const float4* __restrict__ cell_pts,
                                                                float4* __restrict__ mpts, uint32_t* __restrict__ out) {
  const uint32_t k = (blockIdx.x * KV_T + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (k >= nb) return;                         // warp-uniform
  const float* b = boxes + 6 * (size_t)k;
  const float b0 = b[0], b1 = b[1], b2 = b[2], b3 = b[3], b4 = b[4], b5 = b[5];
  // one cell of slack on both sides covers the float rounding of the cell arithmetic; the exact test below decides
  int c0[3], c1[3];
  const float o[3] = {G.ox, G.oy, G.oz};
  const int nn[3] = {G.nx, G.ny, G.nz};
  const float bl[3] = {b0, b1, b2}, bh[3] = {b3, b4, b5};
  bool outside = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float lo = floorf((bl[a] - o[a]) * G.inv_h) - 1.f, hi = floorf((bh[a] - o[a]) * G.inv_h) + 1.f;
    c0[a] = (int)fminf(fmaxf(lo, 0.f), (float)(nn[a] - 1));
    c1[a] = (int)fminf(fmaxf(hi, 0.f), (float)(nn[a] - 1));
    outside |= hi < 0.f || lo > (float)(nn[a] - 1);   // the box lies outside the grid: nothing indexed there
  }
  const int ny = c1[1] - c0[1] + 1, nz = c1[2] - c0[2] + 1;
  uint32_t n = 0;
  for (int row = (int)lane; !outside && row < ny * nz; row += 32) {
    const int y = c0[1] + row % ny, z = c0[2] + row / ny;
    const uint32_t rs = cell_start[grid_cell_index(G, c0[0], y, z)], re = cell_start[grid_cell_index(G, c1[0], y, z) + 1];
    for (uint32_t j = rs; j < re; ++j) {
      const float4 c = cell_pts[j];
      if (b0 <= c.x && b3 > c.x && b1 <= c.y && b4 > c.y && b2 <= c.z && b5 > c.z) {
        const uint32_t slot = __float_as_uint(c.w);
        const uint32_t w = __float_as_uint(mpts[slot].w);
        if (!(w & MALIO_LINK_POINT_DELETED)) {
          if (!COUNT) mpts[slot].w = __uint_as_float(w | MALIO_LINK_POINT_DELETED);
          ++n;
        }
      }
    }
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o2);
  if (COUNT) { if (lane == 0) out[k] = n; }
  else if (lane == 0 && n) atomicAdd(out, n);
}
// bounding box + count of the live slots: grid-stride, warp shuffle + one shared-memory stage per block, ONE set of atomics
// per block (a few hundred blocks: the atomics on the 8 result words stay uncontended)
constexpr int BB_T = 256;
__global__ void __launch_bounds__(BB_T) bbox_kernel(const float4* __restrict__ mpts, uint32_t n_slots, uint32_t* __restrict__ keys) {
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  uint32_t live = 0;
  for (uint32_t i = blockIdx.x * BB_T + threadIdx.x; i < n_slots; i += gridDim.x * BB_T) {
    const float4 a = mpts[i];
    if (!(__float_as_uint(a.w) & MALIO_LINK_POINT_DELETED)) {
      lo[0] = fminf(lo[0], a.x); hi[0] = fmaxf(hi[0], a.x); lo[1] = fminf(lo[1], a.y); hi[1] = fmaxf(hi[1], a.y);
      lo[2] = fminf(lo[2], a.z); hi[2] = fmaxf(hi[2], a.z);
      live += 1;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
      hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
    }
    live += __shfl_xor_sync(0xffffffffu, live, o);
  }
  __shared__ float s_lo[BB_T / 32][3], s_hi[BB_T / 32][3];
  __shared__ uint32_t s_live[BB_T / 32];
  if ((threadIdx.x & 31) == 0) {
    for (int k = 0; k < 3; ++k) { s_lo[threadIdx.x >> 5][k] = lo[k]; s_hi[threadIdx.x >> 5][k] = hi[k]; }
    s_live[threadIdx.x >> 5] = live;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t tot = 0;
    for (int w = 0; w < BB_T / 32; ++w) {
      tot += s_live[w];
      for (int k = 0; k < 3; ++k) { lo[k] = fminf(lo[k], s_lo[w][k]); hi[k] = fmaxf(hi[k], s_hi[w][k]); }
    }
    if (tot) {
      for (int k = 0; k < 3; ++k) { atomicMin(keys + 2 * k, fkey(lo[k])); atomicMax(keys + 2 * k + 1, fkey(hi[k])); }
      atomicAdd(keys + 7, tot);
    }
  }
}
// stable compaction, three steps: live count per block of 1024 slots, exclusive scan of the block counts (one block),
// scatter with a block-local ballot scan
constexpr int CP_T = 1024;
__global__ void __launch_bounds__(CP_T) cp_count_kernel(const float4* __restrict__ mpts, uint32_t n_slots, uint32_t* __restrict__ blk) {
  const uint32_t i = blockIdx.x * CP_T + threadIdx.x;
  const bool live = i < n_slots && !(__float_as_uint(mpts[i].w) & MALIO_LINK_POINT_DELETED);
  const int c = __syncthreads_count(live);
  if (threadIdx.x == 0) blk[blockIdx.x] = (uint32_t)c;
}
__global__ void __launch_bounds__(1024) cp_scan_kernel(const uint32_t* __restrict__ blk, uint32_t nblk, uint32_t* __restrict__ off) {
  __shared__ uint32_t s_w[32];
  __shared__ uint32_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < nblk; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < nblk ? blk[i] : 0u;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= (unsigned)o) inc += t; }
    if ((threadIdx.x & 31) == 31) s_w[threadIdx.x >> 5] = inc;
    __syncthreads();
    uint32_t wb = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wb += s_w[w];
    const uint32_t carry = s_carry;
    if (i < nblk) off[i] = carry + wb + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + wb + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) off[nblk] = s_carry;
}
__global__ void __launch_bounds__(CP_T) cp_scatter_kernel(const float4* __restrict__ mpts, const float* __restrict__ cov, const int32_t* __restrict__ ids,
                                                          uint32_t n_slots, const uint32_t* __restrict__ off, float4* __restrict__ mpts2,
                                                          float* __restrict__ cov2, int32_t* __restrict__ ids2) {
  __shared__ uint32_t s_w[CP_T / 32];
  const uint32_t i = blockIdx.x * CP_T + threadIdx.x;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  bool live = false;
  if (i < n_slots) { a = mpts[i]; live = !(__float_as_uint(a.w) & MALIO_LINK_POINT_DELETED); }
  const uint32_t bal = __ballot_sync(0xffffffffu, live);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = (uint32_t)__popc(bal);
  __syncthreads();
  uint32_t pos = off[blockIdx.x];
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pos += s_w[w];
  pos += (uint32_t)__popc(bal & ((1u << (threadIdx.x & 31)) - 1u));
  if (live) { mpts2[pos] = a; cov2[pos] = cov[i]; ids2[pos] = ids[i]; }
}
__global__ void gather_live_kernel(const float4* __restrict__ mpts, const float* __restrict__ cov, const int32_t* __restrict__ ids,
                                   uint32_t n_slots, const uint32_t* __restrict__ off, float* __restrict__ o_xyz, float* __restrict__ o_ny,
                                   int32_t* __restrict__ o_ids, uint32_t* __restrict__ o_slots) {
  __shared__ uint32_t s_w[CP_T / 32];
  const uint32_t i = blockIdx.x * CP_T + threadIdx.x;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  bool live = false;
  if (i < n_slots) { a = mpts[i]; live = !(__float_as_uint(a.w) & MALIO_LINK_POINT_DELETED); }
  const uint32_t bal = __ballot_sync(0xffffffffu, live);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = (uint32_t)__popc(bal);
  __syncthreads();
  uint32_t pos = off[blockIdx.x];
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pos += s_w[w];
  pos += (uint32_t)__popc(bal & ((1u << (threadIdx.x & 31)) - 1u));
  if (live) {
    if (o_xyz) { o_xyz[3 * (size_t)pos] = a.x; o_xyz[3 * (size_t)pos + 1] = a.y; o_xyz[3 * (size_t)pos + 2] = a.z; }
    if (o_ny) o_ny[pos] = cov[i];
    if (o_ids) o_ids[pos] = ids[i];
    if (o_slots) o_slots[pos] = i;
  }
}

// host arrays -> staging buffer on the device: xyz | normal_y | ids
int stage(malio_handle* h, DeviceState* D, MapOps* M, const float* xyz, const float* ny, const int32_t* ids, uint32_t n, const float** d_xyz,
          const float** d_ny, const int32_t** d_ids, bool* synced_needed) {
  if (n > M->d_stage.size() / 5) { if (int rc = M->d_stage.allocate(h, D->stream, (size_t)(n + n / 4 + 1024) * 5)) return rc; }
  float* base = M->d_stage;
  const size_t stride = M->d_stage.size() / 5;
  *d_xyz = base; *d_ny = base + 3 * stride;
  *d_ids = ids ? reinterpret_cast<const int32_t*>(base + 4 * stride) : nullptr;
  D->ctr.h2d_bytes += (uint64_t)n * (16 + (ids ? 4 : 0));
  *synced_needed = true;
  if (n <= BOUNCE_POINTS) {
    // two bounce slots used in turn: the sync-voxel points and the plain appends of one scan do not wait for each other
    const int bs = M->bounce_next;
    M->bounce_next ^= 1;
    if (!M->h_bounce[bs]) {
      if (int rc = M->h_bounce[bs].allocate(h, (size_t)BOUNCE_POINTS * 5)) return rc;
      CUDA_TRY(cudaEventCreateWithFlags(&M->ev_bounce[bs], cudaEventDisableTiming));
    }
    if (M->bounce_busy[bs]) { CUDA_TRY(cudaEventSynchronize(M->ev_bounce[bs])); M->bounce_busy[bs] = false; }   // its previous batch has left it
    float* hb = M->h_bounce[bs];
    // packed xyz | normal_y | ids, then three device-side destinations out of one pinned source (no host wait)
    std::memcpy(hb, xyz, (size_t)n * 12);
    std::memcpy(hb + 3 * (size_t)n, ny, (size_t)n * 4);
    if (ids) std::memcpy(hb + 4 * (size_t)n, ids, (size_t)n * 4);
    CUDA_TRY(cudaMemcpyAsync(base, hb, (size_t)n * 12, cudaMemcpyHostToDevice, D->stream));
    CUDA_TRY(cudaMemcpyAsync(base + 3 * stride, hb + 3 * (size_t)n, (size_t)n * 4, cudaMemcpyHostToDevice, D->stream));
    if (ids) CUDA_TRY(cudaMemcpyAsync(base + 4 * stride, hb + 4 * (size_t)n, (size_t)n * 4, cudaMemcpyHostToDevice, D->stream));
    CUDA_TRY(cudaEventRecord(M->ev_bounce[bs], D->stream));
    M->bounce_busy[bs] = true;
    *synced_needed = false;
    return MALIO_OK;
  }
  CUDA_TRY(cudaMemcpyAsync(base, xyz, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, D->stream));
  CUDA_TRY(cudaMemcpyAsync(base + 3 * stride, ny, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, D->stream));
  if (ids) CUDA_TRY(cudaMemcpyAsync(base + 4 * stride, ids, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, D->stream));
  return MALIO_OK;
}
// on_device: xyz / ny / ids are device memory the append kernel reads in place, ordered on the caller's stream `caller`
// (no staging, no host wait); otherwise host arrays, staged as above
int append(malio_handle* h, DeviceState* D, MapOps* M, const float* xyz, const float* ny, const int32_t* ids, uint32_t n,
           bool on_device = false, cudaStream_t caller = nullptr) {
  if (n == 0) return MALIO_OK;
  if ((uint64_t)M->n_slots + n > MALIO_LINK_INDEX_MASK) { h->err = "device-resident map: too many slots"; return MALIO_ERR_CAPACITY; }
  if (int rc = malio_dev::grow_slots(h, M->n_slots + n, M->n_slots)) return rc;   // (drains D->stream before it frees anything)
  if (M->n_slots + n > D->d_mpts.size()) { h->err = "device-resident map: slot storage smaller than its recorded use"; return MALIO_ERR_CAPACITY; }
  const float *d_xyz = xyz, *d_ny = ny;
  const int32_t* d_ids = ids;
  bool need_sync = false;
  if (on_device) {
    if (int rc = caller_enter(h, D, caller)) return rc;
  } else {
    if (int rc = stage(h, D, M, xyz, ny, ids, n, &d_xyz, &d_ny, &d_ids, &need_sync)) return rc;
  }
  append_kernel<<<(n + 255) / 256, 256, 0, D->stream>>>(d_xyz, d_ny, d_ids, n, M->n_slots, (int32_t)M->n_slots, D->d_mpts, D->d_cov, D->d_ids);
  CUDA_TRY(cudaGetLastError());
  if (on_device) { if (int rc = caller_leave(h, D, caller)) return rc; }   // the kernel is the last reader of the caller's arrays
  // large batches are copied straight from the caller's arrays: wait until they are consumed.  (The device staging buffer itself is
  // reused in stream order.)
  if (need_sync) CUDA_TRY(cudaStreamSynchronize(D->stream));
  D->ctr.kernel_launches += 1;
  M->n_slots += n;
  M->dirty = true;
  M->appended = true;
  return MALIO_OK;
}

}  // namespace

namespace malio_map {

void leave(malio_handle* h) {
  ++h->map_epoch;
  MapOps* M = h->mapst.get();
  if (!M) return;
  M->active = false;
  M->n_slots = 0; M->n_live = 0;
  M->dirty = false; M->appended = false;
}

int commit(malio_handle* h) {
  MapOps* M = h->mapst.get();
  if (!M || !M->active) return MALIO_OK;
  DeviceState* D = h->dev.get();
  if (!M->dirty && D->tree_free) return MALIO_OK;
  CUDA_TRY(cudaSetDevice(D->device));
  cudaStream_t st = D->stream;
  const uint32_t n = M->n_slots;
  // ---- bounding box + live count
  const uint32_t init[8] = {0xFFFFFFFFu, 0u, 0xFFFFFFFFu, 0u, 0xFFFFFFFFu, 0u, 0u, 0u};
  CUDA_TRY(cudaMemcpyAsync(M->d_small, init, sizeof(init), cudaMemcpyHostToDevice, st));
  if (n) bbox_kernel<<<(n + BB_T - 1) / BB_T < 592u ? (n + BB_T - 1) / BB_T : 592u, BB_T, 0, st>>>(D->d_mpts, n, M->d_small);
  CUDA_TRY(cudaMemcpyAsync(M->h_small, M->d_small, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  D->ctr.kernel_launches += 1;
  M->n_live = M->h_small[7];
  // ---- compaction when more than half of the slots are dead (stable: slot order = age order is kept)
  if (n > 65536 && M->n_live * 2 < n) {
    const uint32_t nblk = (n + CP_T - 1) / CP_T;
    if (nblk + 1 > M->d_blk.size()) {
      if (int rc = malio_buf::allocate_group(h, st, {{M->d_blk, nblk + 1024}, {M->d_blkoff, nblk + 1025}})) return rc;
    }
    const size_t cap2 = D->d_mpts.size();
    if (cap2 > M->d_mpts2.size()) {
      if (int rc = malio_buf::allocate_group(h, st, {{M->d_mpts2, cap2}, {M->d_cov2, cap2}, {M->d_ids2, cap2}})) return rc;
    }
    cp_count_kernel<<<nblk, CP_T, 0, st>>>(D->d_mpts, n, M->d_blk);
    cp_scan_kernel<<<1, 1024, 0, st>>>(M->d_blk, nblk, M->d_blkoff);
    cp_scatter_kernel<<<nblk, CP_T, 0, st>>>(D->d_mpts, D->d_cov, D->d_ids, n, M->d_blkoff, M->d_mpts2, M->d_cov2, M->d_ids2);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(st));
    std::swap(D->d_mpts, M->d_mpts2); std::swap(D->d_cov, M->d_cov2); std::swap(D->d_ids, M->d_ids2);   // sizes go along
    M->n_slots = M->n_live;
    D->ctr.kernel_launches += 3;
    D->ctr.map_compactions += 1;
  }
  float box[6] = {0, 0, 0, 0, 0, 0};
  if (M->n_live) for (int k = 0; k < 6; ++k) box[k] = fkey_inv(M->h_small[k]);
  // no live point, whether built empty, compacted to nothing or with dead slots left: the index is empty and the search answers
  // like a snapshot of 0 nodes (empty lists, nothing selected), whatever the history
  const int rc = malio_dev::index_from_slots(h, M->n_live ? M->n_slots : 0, box);
  if (rc != MALIO_OK) return rc;
  M->dirty = false;
  M->appended = false;
  D->ctr.map_slots = M->n_slots;
  D->ctr.map_live = M->n_live;
  return MALIO_OK;
}

// build / add_points from host arrays (on_device false) or from device arrays ordered on `caller`
static int build_from(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n, bool on_device,
                      cudaStream_t caller) {
  MapOps* M;
  DeviceState* D;
  if (int rc = acquire(h, h->mapst, M, D)) return rc;
  ++h->map_epoch;
  if (D->refit_pending) { CUDA_TRY(cudaStreamSynchronize(D->stream2)); D->refit_pending = false; }
  M->n_slots = 0; M->n_live = 0;
  M->active = true;
  D->tree_free = true;      // grow_slots copies existing slots only in this mode; none are kept here
  if (int rc = malio_dev::grow_slots(h, n > 0 ? n : 1, 0)) return rc;
  M->dirty = true;
  if (int rc = append(h, D, M, xyz, normal_y, ids, n, on_device, caller)) return rc;
  return commit(h);
}

static int add_points_from(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n, bool on_device,
                           cudaStream_t caller) {
  MapOps* M = h->mapst.get();
  if (!M || !M->active) { h->err = "malio_map_add_points before malio_map_build"; return MALIO_ERR_STATE; }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  return append(h, D, M, xyz, normal_y, ids, n, on_device, caller);
}
int build(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n) {
  return build_from(h, xyz, normal_y, ids, n, false, nullptr);
}
int add_points(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n) {
  return add_points_from(h, xyz, normal_y, ids, n, false, nullptr);
}

// the device-memory variants: every argument the host can check is checked before anything is launched
static int check_device_points(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n) {
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  if (n == 0) return MALIO_OK;
  if (int rc = check_device_ptr(h, D, xyz, "xyz")) return rc;
  if (int rc = check_device_ptr(h, D, normal_y, "normal_y")) return rc;
  return check_device_ptrs(h, D, {{ids, "ids"}});
}
int build_device(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n, cudaStream_t caller) {
  if (int rc = check_device_points(h, xyz, normal_y, ids, n)) return rc;
  return build_from(h, xyz, normal_y, ids, n, true, caller);
}
int add_points_device(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n, cudaStream_t caller) {
  if (int rc = check_device_points(h, xyz, normal_y, ids, n)) return rc;
  return add_points_from(h, xyz, normal_y, ids, n, true, caller);
}

int delete_boxes(malio_handle* h, const float* boxes, uint32_t nb, uint32_t* n_deleted) {
  MapOps* M = h->mapst.get();
  if (!M || !M->active) { h->err = "malio_map_delete_boxes before malio_map_build"; return MALIO_ERR_STATE; }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  uint32_t total = 0;
  for (uint32_t at = 0; at < nb; at += MAX_BIG_BOXES) {
    BigBoxes B{};
    B.nb = (int)((nb - at) < (uint32_t)MAX_BIG_BOXES ? (nb - at) : (uint32_t)MAX_BIG_BOXES);
    for (int k = 0; k < B.nb; ++k) std::memcpy(B.b[k], boxes + 6 * (size_t)(at + k), 6 * sizeof(float));
    CUDA_TRY(cudaMemsetAsync(M->d_small + 6, 0, sizeof(uint32_t), D->stream));
    if (M->n_slots) kill_big_boxes_kernel<<<(M->n_slots + 255) / 256, 256, 0, D->stream>>>(D->d_mpts, M->n_slots, B, M->d_small + 6);
    CUDA_TRY(cudaMemcpyAsync(M->h_small + 6, M->d_small + 6, sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    total += M->h_small[6];
    D->ctr.kernel_launches += 1;
  }
  if (total) M->dirty = true;
  if (n_deleted) *n_deleted = total;
  return MALIO_OK;
}

int sync_voxels(malio_handle* h, const float* boxes, uint32_t nb, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t m,
                uint32_t* n_deleted) {
  MapOps* M = h->mapst.get();
  if (!M || !M->active) { h->err = "malio_map_sync_voxels before malio_map_build"; return MALIO_ERR_STATE; }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  if (M->appended || !D->tree_free) { if (int rc = commit(h)) return rc; }   // the kill below reads the index: it must know every live slot
  uint32_t killed = 0;
  if (nb && D->grid_on) {
    if (nb > M->d_boxes.size() / 6) { if (int rc = M->d_boxes.allocate(h, D->stream, (size_t)(nb + nb / 4 + 1024) * 6)) return rc; }
    const bool via_bounce = !n_deleted && nb <= BOUNCE_BOXES;
    if (via_bounce) {
      if (!M->h_bounce_box) {
        if (int rc = M->h_bounce_box.allocate(h, (size_t)BOUNCE_BOXES * 6)) return rc;
        CUDA_TRY(cudaEventCreateWithFlags(&M->ev_bounce_box, cudaEventDisableTiming));
      }
      if (M->bounce_box_busy) { CUDA_TRY(cudaEventSynchronize(M->ev_bounce_box)); M->bounce_box_busy = false; }
      std::memcpy(M->h_bounce_box, boxes, (size_t)nb * 6 * sizeof(float));
      CUDA_TRY(cudaMemcpyAsync(M->d_boxes, M->h_bounce_box, (size_t)nb * 6 * sizeof(float), cudaMemcpyHostToDevice, D->stream));
      CUDA_TRY(cudaEventRecord(M->ev_bounce_box, D->stream));
      M->bounce_box_busy = true;
    } else {
      CUDA_TRY(cudaMemcpyAsync(M->d_boxes, boxes, (size_t)nb * 6 * sizeof(float), cudaMemcpyHostToDevice, D->stream));
    }
    CUDA_TRY(cudaMemsetAsync(M->d_small + 6, 0, sizeof(uint32_t), D->stream));
    kill_voxel_boxes_kernel<false><<<(nb + KV_T / 32 - 1) / (KV_T / 32), KV_T, 0, D->stream>>>(M->d_boxes, nb, D->grid, D->d_cell_start, D->d_cell_pts, D->d_mpts, M->d_small + 6);
    CUDA_TRY(cudaGetLastError());
    if (n_deleted) {   // the count is only fetched (and waited for) when the caller asks for it
      CUDA_TRY(cudaMemcpyAsync(M->h_small + 6, M->d_small + 6, sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
      CUDA_TRY(cudaStreamSynchronize(D->stream));
      killed = M->h_small[6];
    } else {
      if (!via_bounce) CUDA_TRY(cudaStreamSynchronize(D->stream));   // boxes were copied straight from the caller's array
      killed = 1;      // unknown: treat the index as stale
    }
    D->ctr.kernel_launches += 1;
    D->ctr.h2d_bytes += (uint64_t)nb * 24;
  }
  if (killed) M->dirty = true;
  if (n_deleted) *n_deleted = killed;
  return append(h, D, M, xyz, normal_y, ids, m);
}

int count_boxes(malio_handle* h, const float* d_boxes, uint32_t nb, uint32_t* d_counts) {
  MapOps* M = h->mapst.get();
  if (!M || !M->active) { h->err = "device-resident map: box count before malio_map_build"; return MALIO_ERR_STATE; }
  DeviceState* D = h->dev.get();
  if (M->dirty || !D->tree_free) { h->err = "device-resident map: box count on an uncommitted index"; return MALIO_ERR_STATE; }
  if (nb == 0) return MALIO_OK;
  if (!D->grid_on) {   // no live point (a committed map with live points always has its index)
    CUDA_TRY(cudaMemsetAsync(d_counts, 0, (size_t)nb * sizeof(uint32_t), D->stream));
    return MALIO_OK;
  }
  kill_voxel_boxes_kernel<true><<<(nb + KV_T / 32 - 1) / (KV_T / 32), KV_T, 0, D->stream>>>(d_boxes, nb, D->grid, D->d_cell_start, D->d_cell_pts,
                                                                                            D->d_mpts, d_counts);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

int info(malio_handle* h, uint32_t* n_live, uint32_t* n_slots) {
  MapOps* M = h->mapst.get();
  if (!M || !M->active) { h->err = "malio_map_info before malio_map_build"; return MALIO_ERR_STATE; }
  if (int rc = commit(h)) return rc;
  if (n_live) *n_live = M->n_live;
  if (n_slots) *n_slots = M->n_slots;
  return MALIO_OK;
}

int download(malio_handle* h, float* xyz, float* normal_y, int32_t* ids, uint32_t* slots, uint32_t cap, uint32_t* n_out) {
  MapOps* M = h->mapst.get();
  if (!M || !M->active) { h->err = "malio_map_download before malio_map_build"; return MALIO_ERR_STATE; }
  if (int rc = commit(h)) return rc;
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t n = M->n_slots, live = M->n_live;
  if (n_out) *n_out = live;
  if (live == 0 || (!xyz && !normal_y && !ids && !slots)) return MALIO_OK;
  if (cap < live) { h->err = "malio_map_download: capacity below the number of live points"; return MALIO_ERR_CAPACITY; }
  const uint32_t nblk = (n + CP_T - 1) / CP_T;
  if (nblk + 1 > M->d_blk.size()) {
    if (int rc = malio_buf::allocate_group(h, D->stream, {{M->d_blk, nblk + 1024}, {M->d_blkoff, nblk + 1025}})) return rc;
  }
  DeviceBuffer<float> d_out;   // freed on return, after the wait below
  if (int rc = d_out.allocate(h, D->stream, (size_t)live * 6)) return rc;
  float* o_xyz = d_out; float* o_ny = d_out + 3 * (size_t)live;
  int32_t* o_ids = reinterpret_cast<int32_t*>(d_out + 4 * (size_t)live); uint32_t* o_slots = reinterpret_cast<uint32_t*>(d_out + 5 * (size_t)live);
  cp_count_kernel<<<nblk, CP_T, 0, D->stream>>>(D->d_mpts, n, M->d_blk);
  cp_scan_kernel<<<1, 1024, 0, D->stream>>>(M->d_blk, nblk, M->d_blkoff);
  gather_live_kernel<<<nblk, CP_T, 0, D->stream>>>(D->d_mpts, D->d_cov, D->d_ids, n, M->d_blkoff, o_xyz, o_ny, o_ids, o_slots);
  if (xyz) cudaMemcpyAsync(xyz, o_xyz, (size_t)live * 12, cudaMemcpyDeviceToHost, D->stream);
  if (normal_y) cudaMemcpyAsync(normal_y, o_ny, (size_t)live * 4, cudaMemcpyDeviceToHost, D->stream);
  if (ids) cudaMemcpyAsync(ids, o_ids, (size_t)live * 4, cudaMemcpyDeviceToHost, D->stream);
  if (slots) cudaMemcpyAsync(slots, o_slots, (size_t)live * 4, cudaMemcpyDeviceToHost, D->stream);
  const cudaError_t e = cudaStreamSynchronize(D->stream);
  if (e != cudaSuccess) { h->err = std::string("malio_map_download: ") + cudaGetErrorString(e); return MALIO_ERR_CUDA; }
  D->ctr.kernel_launches += 3;
  return MALIO_OK;
}

}  // namespace malio_map

extern "C" int malio_map_build_device(malio_handle* h, const float* d_xyz, const float* d_normal_y, const int32_t* d_ids, uint32_t n,
                                      void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_map::build_device(h, d_xyz, d_normal_y, d_ids, n, (cudaStream_t)stream);
}
extern "C" int malio_map_add_points_device(malio_handle* h, const float* d_xyz, const float* d_normal_y, const int32_t* d_ids,
                                           uint32_t n, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_map::add_points_device(h, d_xyz, d_normal_y, d_ids, n, (cudaStream_t)stream);
}
