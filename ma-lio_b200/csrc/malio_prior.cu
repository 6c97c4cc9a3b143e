// malio_prior.cu — localization in a saved map, sm_90a: a prior map of any extent kept on the device, sorted by tile, and the
// local-map window over it that lasermap_fov_segment (laserMapping.cpp:171-224) keeps around the sensor.  The window is the
// device-resident map of malio_mapops.cu (slots + cell-list index): every search, pass and map call works on it unchanged.
//
// Why no host tree is needed here: without inserts the map is a fixed point set, and the window's live set is a pure function
// of that set and the cube, prior ∩ cube (min <= p < max per axis).  The device can compute it alone; nothing order-dependent
// (Add_Points(.., true)) has to be replayed from a host ikd-Tree.
//
// Prior store (one load, O(n log n) on the device):
//   pm_key_kernel     absolute tile of every point, floor(x / TILE) per axis in float, packed (z, y, x) into 63 bits; a flag
//                     word for non-finite points and tile indices outside the 21 bits an axis has
//   radix sort        stable CUB sort of (key, input index): tile-key order, input order within a tile
//   pm_gather_kernel  the points as float4 {x, y, z, normal_y} and their ids, in sorted order
//   run-length        the tile directory: sorted unique keys and the offset of each tile's first point
// Window slide (O(points entering), whatever the size of the prior):
//   host              the tile rows (ty, tz) the new cube meets, each cut to the tiles that are not strictly inside the old cube
//                     (a tile strictly inside holds only points inside: floor of a correctly rounded division is monotone)
//   pm_range_kernel   one binary search per row range in the directory -> a contiguous run of points
//   pm_count / pm_scatter_kernel   the exact test in(new) && !in(old) per candidate, compacted stably into a scratch area
//   malio_mapops      delete_boxes (the reference's cub_needrm slabs), add_points_device (the append), commit
// Compiled with -fmad=false like the rest of the library.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

#include "malio_device.cuh"

using namespace malio_devstate;

namespace {

// Tile edge (m).  Small enough that a slide tests few points besides the entering ones (the candidates of a slide are the
// entering slab plus at most one tile layer on each of its faces), large enough that a tile row of a 1000 m cube is a few
// dozen tiles and the directory is 12 B per tile.  DESIGN.md, "Localization in a prior map", has the measurement.
constexpr float TILE = 25.0f;
constexpr int TILE_BITS = 21;                               // per axis; the key is (z, y, x), 63 bits
constexpr int TILE_BIAS = 1 << (TILE_BITS - 1);             // tile index range [-2^20, 2^20)
constexpr uint32_t FLAG_NONFINITE = 1u, FLAG_RANGE = 2u;
constexpr int CP_T = 1024;                                  // candidates per compaction block

}  // namespace

namespace malio_prior {

struct PriorState {
  bool loaded = false;
  uint32_t n = 0, n_tiles = 0;
  int tlo[3] = {0, 0, 0}, thi[3] = {-1, -1, -1};            // tile bounding box of the prior (empty: lo > hi)
  DeviceBuffer<float4> d_pts;                               // {x, y, z, normal_y}, tile-key order
  DeviceBuffer<int32_t> d_ids;
  DeviceBuffer<unsigned long long> d_tkey;                  // directory: sorted unique tile keys ...
  DeviceBuffer<uint32_t> d_toff;                            // ... and n_tiles + 1 point offsets
  // the window: lasermap_fov_segment's LocalMap_Points, valid while the device map is the one this window built (epoch)
  bool win = false;
  uint64_t win_epoch = 0;
  float cube[6] = {0, 0, 0, 0, 0, 0};                       // {min3, max3}
  // window scratch (grow-only): range queries, per-range first point / exclusive candidate offsets, compaction blocks, the
  // entering points (xyz rows | normal_y | ids, 5 floats a point)
  DeviceBuffer<unsigned long long> d_rq;
  DeviceBuffer<uint32_t> d_rbeg, d_roff, d_blk, d_blkoff;
  DeviceBuffer<float> d_out;
  DeviceBuffer<char> d_temp;                                // CUB's temporary storage of the window's scans
  DeviceBuffer<uint32_t> d_small;                           // [0] flags, [1..6] biased tile min/max, [7] tile count
  PinnedBuffer<uint32_t> h_small;

  int init(malio_handle* h, DeviceState* D) {
    if (int rc = d_small.allocate(h, D->stream, 8)) return rc;
    return h_small.allocate(h, 8);
  }
};

}  // namespace malio_prior

namespace {

using malio_prior::PriorState;

__host__ __device__ __forceinline__ unsigned long long tile_key(int tx, int ty, int tz) {
  return ((unsigned long long)(uint32_t)(tz + TILE_BIAS) << (2 * TILE_BITS)) |
         ((unsigned long long)(uint32_t)(ty + TILE_BIAS) << TILE_BITS) | (unsigned long long)(uint32_t)(tx + TILE_BIAS);
}

__global__ void __launch_bounds__(256) pm_key_kernel(const float* __restrict__ xyz, uint32_t n, unsigned long long* __restrict__ key,
                                                     uint32_t* __restrict__ val, uint32_t* __restrict__ small) {
  const uint32_t i = blockIdx.x * 256u + threadIdx.x;
  if (i >= n) return;
  const float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
  val[i] = i;
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) { atomicOr(small, FLAG_NONFINITE); key[i] = ~0ull; return; }
  const float f[3] = {floorf(x / TILE), floorf(y / TILE), floorf(z / TILE)};
  int t[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!(f[a] >= -(float)TILE_BIAS && f[a] < (float)TILE_BIAS)) { atomicOr(small, FLAG_RANGE); key[i] = ~0ull; return; }
    t[a] = (int)f[a];
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    atomicMin(small + 1 + a, (uint32_t)(t[a] + TILE_BIAS));
    atomicMax(small + 4 + a, (uint32_t)(t[a] + TILE_BIAS));
  }
  key[i] = tile_key(t[0], t[1], t[2]);
}

__global__ void __launch_bounds__(256) pm_gather_kernel(const uint32_t* __restrict__ perm, uint32_t n, const float* __restrict__ xyz,
                                                        const float* __restrict__ ny, const int32_t* __restrict__ ids,
                                                        float4* __restrict__ pts, int32_t* __restrict__ out_ids) {
  const uint32_t i = blockIdx.x * 256u + threadIdx.x;
  if (i >= n) return;
  const uint32_t p = perm[i];
  pts[i] = make_float4(xyz[3 * (size_t)p], xyz[3 * (size_t)p + 1], xyz[3 * (size_t)p + 2], ny[p]);
  out_ids[i] = ids ? ids[p] : (int32_t)p;
}

// one row range [rq[2r], rq[2r+1]] of tile keys -> the points of its tiles: first point rbeg[r], count cnt[r]
__global__ void __launch_bounds__(256) pm_range_kernel(const unsigned long long* __restrict__ rq, uint32_t nr,
                                                       const unsigned long long* __restrict__ tkey, uint32_t nt,
                                                       const uint32_t* __restrict__ toff, uint32_t* __restrict__ rbeg,
                                                       uint32_t* __restrict__ cnt) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= nr) return;
  const unsigned long long lo = rq[2 * r], hi = rq[2 * r + 1];
  uint32_t a = 0, b = nt;                       // first tile with key >= lo
  while (a < b) { const uint32_t m = (a + b) >> 1; if (tkey[m] < lo) a = m + 1; else b = m; }
  uint32_t c = a, d = nt;                       // first tile with key > hi
  while (c < d) { const uint32_t m = (c + d) >> 1; if (tkey[m] <= hi) c = m + 1; else d = m; }
  rbeg[r] = toff[a];
  cnt[r] = toff[c] - toff[a];
}

struct Cubes { float nw[6], od[6]; int has_old; };
// lasermap_fov_segment's box test, half-open (Delete_by_range, ikd_Tree.cpp:807)
__device__ __forceinline__ bool in_box(const float b[6], const float4& p) {
  return b[0] <= p.x && p.x < b[3] && b[1] <= p.y && p.y < b[4] && b[2] <= p.z && p.z < b[5];
}
// candidate j -> its point (range found by a binary search over the exclusive offsets roff[0..nr]) and the verdict
__device__ __forceinline__ bool candidate(const Cubes& c, const uint32_t* __restrict__ rbeg, const uint32_t* __restrict__ roff,
                                          uint32_t nr, const float4* __restrict__ pts, uint32_t j, uint32_t& p) {
  uint32_t a = 0, b = nr;                       // last range with roff <= j
  while (b - a > 1) { const uint32_t m = (a + b) >> 1; if (roff[m] <= j) a = m; else b = m; }
  p = rbeg[a] + (j - roff[a]);
  const float4 q = pts[p];
  return in_box(c.nw, q) && !(c.has_old && in_box(c.od, q));
}
__global__ void __launch_bounds__(CP_T) pm_count_kernel(Cubes c, const uint32_t* __restrict__ rbeg, const uint32_t* __restrict__ roff,
                                                        uint32_t nr, uint32_t n_cand, const float4* __restrict__ pts,
                                                        uint32_t* __restrict__ blk) {
  const uint32_t j = blockIdx.x * CP_T + threadIdx.x;
  uint32_t p;
  const bool keep = j < n_cand && candidate(c, rbeg, roff, nr, pts, j, p);
  const int k = __syncthreads_count(keep);
  if (threadIdx.x == 0) blk[blockIdx.x] = (uint32_t)k;
}
// stable scatter of the survivors: block offset + warp ballots, in candidate order
__global__ void __launch_bounds__(CP_T) pm_scatter_kernel(Cubes c, const uint32_t* __restrict__ rbeg, const uint32_t* __restrict__ roff,
                                                          uint32_t nr, uint32_t n_cand, const float4* __restrict__ pts,
                                                          const int32_t* __restrict__ ids, const uint32_t* __restrict__ blkoff,
                                                          float* __restrict__ out, uint32_t cap) {
  __shared__ uint32_t s_w[CP_T / 32];
  const uint32_t j = blockIdx.x * CP_T + threadIdx.x;
  uint32_t p = 0;
  const bool keep = j < n_cand && candidate(c, rbeg, roff, nr, pts, j, p);
  const uint32_t bal = __ballot_sync(0xffffffffu, keep);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = (uint32_t)__popc(bal);
  __syncthreads();
  uint32_t pos = blkoff[blockIdx.x];
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pos += s_w[w];
  pos += (uint32_t)__popc(bal & ((1u << (threadIdx.x & 31)) - 1u));
  if (keep) {
    const float4 q = pts[p];
    out[3 * (size_t)pos] = q.x; out[3 * (size_t)pos + 1] = q.y; out[3 * (size_t)pos + 2] = q.z;
    out[3 * (size_t)cap + pos] = q.w;
    reinterpret_cast<int32_t*>(out + 4 * (size_t)cap)[pos] = ids[p];
  }
}

int grow_temp(malio_handle* h, DeviceBuffer<char>& temp, cudaStream_t st, size_t t) {
  if (t <= temp.size()) return MALIO_OK;
  return temp.allocate(h, st, t + t / 8 + 4096);
}

// the prior from device arrays read on the handle's stream (the caller has ordered them there).  Refusals leave the previous
// prior and the window as they were.
int load_core(malio_handle* h, PriorState* P, DeviceState* D, const float* xyz, const float* ny, const int32_t* ids, uint32_t n) {
  cudaStream_t st = D->stream;
  if (n > 0x7FFFFFFFu) { h->err = "prior map: more than 2^31 - 1 points"; return MALIO_ERR_CAPACITY; }
  // sort area: keys | alternate keys | values | alternate values, released at the end of the load
  DeviceBuffer<unsigned long long> d_key;
  DeviceBuffer<uint32_t> d_val;
  DeviceBuffer<char> d_temp;
  if (int rc = malio_buf::allocate_group(h, st, {{d_key, 2 * (size_t)n}, {d_val, 2 * (size_t)n}})) return rc;
  cub::DoubleBuffer<unsigned long long> k(d_key.data(), d_key.data() + n);
  cub::DoubleBuffer<uint32_t> v(d_val.data(), d_val.data() + n);
  const uint32_t init[8] = {0, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0, 0, 0, 0};
  CUDA_TRY(cudaMemcpyAsync(P->d_small, init, sizeof(init), cudaMemcpyHostToDevice, st));
  pm_key_kernel<<<(n + 255) / 256, 256, 0, st>>>(xyz, n, k.Current(), v.Current(), P->d_small);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(P->h_small, P->d_small, 7 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  D->ctr.kernel_launches += 1;
  if (P->h_small[0] & FLAG_NONFINITE) { h->err = "prior map: a point has a non-finite coordinate; the previous prior is kept"; return MALIO_ERR_INVALID_ARG; }
  if (P->h_small[0] & FLAG_RANGE) {
    h->err = "prior map: a point's tile index lies outside +-2^20 tiles of " + std::to_string(TILE) + " m; the previous prior is kept";
    return MALIO_ERR_CAPACITY;
  }
  int tlo[3], thi[3];
  for (int a = 0; a < 3; ++a) { tlo[a] = (int)P->h_small[1 + a] - TILE_BIAS; thi[a] = (int)P->h_small[4 + a] - TILE_BIAS; }
  size_t t = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t, k, v, (int)n, 0, 3 * TILE_BITS, st));
  size_t t2 = 0;
  unsigned long long* un = nullptr; uint32_t* uu = nullptr;
  CUDA_TRY(cub::DeviceRunLengthEncode::Encode(nullptr, t2, un, un, uu, uu, (int)n, st));
  if (t2 > t) t = t2;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t2, uu, uu, (int)n, st));
  if (t2 > t) t = t2;
  if (int rc = d_temp.allocate(h, st, t)) return rc;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(d_temp, t, k, v, (int)n, 0, 3 * TILE_BITS, st));
  // the new store replaces the old one (the window it fed ends with it)
  CUDA_TRY(cudaStreamSynchronize(st));
  P->d_pts.release(); P->d_ids.release(); P->d_tkey.release(); P->d_toff.release();
  P->loaded = false; P->win = false; P->n = 0; P->n_tiles = 0;
  if (int rc = malio_buf::allocate_group(h, st, {{P->d_pts, n}, {P->d_ids, n}})) return rc;
  pm_gather_kernel<<<(n + 255) / 256, 256, 0, st>>>(v.Current(), n, xyz, ny, ids, P->d_pts, P->d_ids);
  // tile directory: unique keys into the free key half, counts into the free value half, offsets (exclusive sum) into the other
  unsigned long long* uk = k.Alternate();
  uint32_t* cnt = v.Alternate();
  uint32_t* off = v.Current();   // the permutation is dead once gathered (stream order)
  t2 = d_temp.size();
  CUDA_TRY(cub::DeviceRunLengthEncode::Encode(d_temp, t2, k.Current(), uk, cnt, P->d_small + 7, (int)n, st));
  CUDA_TRY(cudaMemcpyAsync(P->h_small + 7, P->d_small + 7, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  const uint32_t nt = P->h_small[7];
  t2 = d_temp.size();
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(d_temp, t2, cnt, off, (int)nt, st));
  if (int rc = malio_buf::allocate_group(h, st, {{P->d_tkey, nt}, {P->d_toff, (size_t)nt + 1}})) return rc;
  CUDA_TRY(cudaMemcpyAsync(P->d_tkey, uk, (size_t)nt * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(P->d_toff, off, (size_t)nt * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
  P->h_small[6] = n;   // (the pinned word is free again: the tile count was read above)
  CUDA_TRY(cudaMemcpyAsync(P->d_toff + nt, P->h_small + 6, sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(st));   // before the sort area goes back
  D->ctr.kernel_launches += 4;           // key, gather, and the sort / run-length / scan passes counted as two
  P->n = n; P->n_tiles = nt;
  for (int a = 0; a < 3; ++a) { P->tlo[a] = tlo[a]; P->thi[a] = thi[a]; }
  P->loaded = true;
  return MALIO_OK;
}

int load_empty(malio_handle* h, PriorState* P, DeviceState* D) {
  CUDA_TRY(cudaStreamSynchronize(D->stream));   // the store may still be read by an enqueued append
  P->d_pts.release(); P->d_ids.release(); P->d_tkey.release(); P->d_toff.release();
  P->n = 0; P->n_tiles = 0;
  for (int a = 0; a < 3; ++a) { P->tlo[a] = 0; P->thi[a] = -1; }
  P->win = false;
  P->loaded = true;
  return MALIO_OK;
}

// floor(v / TILE) in float as the key kernel takes it, clamped to [lo, hi] (lo - 1 / hi + 1 mark "below" / "above")
int tile_of(float v, int lo, int hi) {
  const float f = std::floor(v / TILE);
  if (!(f >= (float)lo)) return lo - 1;
  if (!(f <= (float)hi)) return hi + 1;
  return (int)f;
}

// prior ∩ nw ∖ od (od ignored when has_old == 0) -> d_out rows, in tile-key order and input order within a tile; *m = count
int gather(malio_handle* h, PriorState* P, DeviceState* D, const Cubes& c, uint32_t* m) {
  *m = 0;
  if (P->n == 0) return MALIO_OK;
  cudaStream_t st = D->stream;
  int lo[3], hi[3], ilo[3], ihi[3];
  for (int a = 0; a < 3; ++a) {
    lo[a] = tile_of(c.nw[a], P->tlo[a], P->thi[a]);
    hi[a] = tile_of(c.nw[3 + a], P->tlo[a], P->thi[a]);
    if (lo[a] < P->tlo[a]) lo[a] = P->tlo[a];
    if (hi[a] > P->thi[a]) hi[a] = P->thi[a];
    if (lo[a] > hi[a]) return MALIO_OK;   // the cube misses the prior's tiles
    // tiles strictly between the old cube's min and max tiles hold only points inside it
    ilo[a] = c.has_old ? tile_of(c.od[a], P->tlo[a] - 1, P->thi[a] + 1) + 1 : 1;
    ihi[a] = c.has_old ? tile_of(c.od[3 + a], P->tlo[a] - 1, P->thi[a] + 1) - 1 : 0;
  }
  std::vector<unsigned long long> rq;
  for (int tz = lo[2]; tz <= hi[2]; ++tz)
    for (int ty = lo[1]; ty <= hi[1]; ++ty) {
      const bool inner = ilo[2] <= tz && tz <= ihi[2] && ilo[1] <= ty && ty <= ihi[1] && ilo[0] <= ihi[0];
      auto add = [&](int a, int b) { if (a <= b) { rq.push_back(tile_key(a, ty, tz)); rq.push_back(tile_key(b, ty, tz)); } };
      if (inner) { add(lo[0], std::min(hi[0], ilo[0] - 1)); add(std::max(lo[0], ihi[0] + 1), hi[0]); }
      else add(lo[0], hi[0]);
    }
  const uint32_t nr = (uint32_t)(rq.size() / 2);
  if (nr == 0) return MALIO_OK;
  if (rq.size() > P->d_rq.size()) {
    if (int rc = P->d_rq.allocate(h, st, rq.size() + rq.size() / 4 + 256)) return rc;
  }
  if ((size_t)nr + 1 > P->d_rbeg.size()) {
    const size_t c2 = nr + nr / 4 + 256;
    if (int rc = malio_buf::allocate_group(h, st, {{P->d_rbeg, c2}, {P->d_roff, c2}})) return rc;
  }
  size_t t = 0;
  uint32_t* un = nullptr;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t, un, un, (int)nr + 1, st));
  if (int rc = grow_temp(h, P->d_temp, st, t)) return rc;
  CUDA_TRY(cudaMemcpyAsync(P->d_rq, rq.data(), rq.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
  D->ctr.h2d_bytes += rq.size() * sizeof(unsigned long long);
  // counts go to d_roff[0..nr) with d_roff[nr] = 0 (the "+1" row), then an exclusive sum in place: d_roff[nr] = candidates
  CUDA_TRY(cudaMemsetAsync(P->d_roff + nr, 0, sizeof(uint32_t), st));
  pm_range_kernel<<<(nr + 255) / 256, 256, 0, st>>>(P->d_rq, nr, P->d_tkey, P->n_tiles, P->d_toff, P->d_rbeg, P->d_roff);
  t = P->d_temp.size();
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(P->d_temp, t, P->d_roff.data(), P->d_roff.data(), (int)nr + 1, st));
  CUDA_TRY(cudaMemcpyAsync(P->h_small, P->d_roff + nr, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  D->ctr.kernel_launches += 2;
  const uint32_t n_cand = P->h_small[0];
  if (n_cand == 0) return MALIO_OK;
  const uint32_t nblk = (n_cand + CP_T - 1) / CP_T;
  if ((size_t)nblk + 1 > P->d_blk.size()) {
    const size_t c2 = nblk + nblk / 4 + 256;
    if (int rc = malio_buf::allocate_group(h, st, {{P->d_blk, c2}, {P->d_blkoff, c2}})) return rc;
  }
  if ((size_t)n_cand * 5 > P->d_out.size()) {
    if (int rc = P->d_out.allocate(h, st, ((size_t)n_cand + n_cand / 4 + 1024) * 5)) return rc;
  }
  t = 0;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t, un, un, (int)nblk + 1, st));
  if (int rc = grow_temp(h, P->d_temp, st, t)) return rc;
  const uint32_t cap = (uint32_t)(P->d_out.size() / 5);
  CUDA_TRY(cudaMemsetAsync(P->d_blk + nblk, 0, sizeof(uint32_t), st));
  pm_count_kernel<<<nblk, CP_T, 0, st>>>(c, P->d_rbeg, P->d_roff, nr, n_cand, P->d_pts, P->d_blk);
  t = P->d_temp.size();
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(P->d_temp, t, P->d_blk.data(), P->d_blkoff.data(), (int)nblk + 1, st));
  pm_scatter_kernel<<<nblk, CP_T, 0, st>>>(c, P->d_rbeg, P->d_roff, nr, n_cand, P->d_pts, P->d_ids, P->d_blkoff, P->d_out, cap);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(P->h_small, P->d_blkoff + nblk, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  D->ctr.kernel_launches += 3;
  *m = P->h_small[0];
  return MALIO_OK;
}

// the entering points d_out[0 .. m) -> a new device map (first call) or the slots' tail
int feed(malio_handle* h, PriorState* P, DeviceState* D, uint32_t m, bool build) {
  const size_t cap = P->d_out.size() / 5;
  const float* xyz = m ? P->d_out.data() : nullptr;
  const float* ny = m ? P->d_out + 3 * cap : nullptr;
  const int32_t* ids = m ? reinterpret_cast<const int32_t*>(P->d_out + 4 * cap) : nullptr;
  if (build) return malio_map::build_device(h, xyz, ny, ids, m, D->stream);
  return malio_map::add_points_device(h, xyz, ny, ids, m, D->stream);
}

}  // namespace

namespace malio_prior {

int load(malio_handle* h, const float* xyz, const float* ny, const int32_t* ids, uint32_t n, bool on_device, cudaStream_t caller) {
  PriorState* P;
  DeviceState* D;
  if (int rc = acquire(h, h->prior, P, D)) return rc;
  release(h->place, D->stream);   // the place database describes the prior this load replaces
  if (n == 0) return load_empty(h, P, D);
  if (on_device) {
    if (int rc = check_device_ptr(h, D, xyz, "xyz")) return rc;
    if (int rc = check_device_ptr(h, D, ny, "normal_y")) return rc;
    if (int rc = check_device_ptrs(h, D, {{ids, "ids"}})) return rc;
    if (int rc = caller_enter(h, D, caller)) return rc;
    const int rc = load_core(h, P, D, xyz, ny, ids, n);
    // the caller's arrays were last read by the gather, which the load waited for; caller_leave orders `caller` behind it
    if (int rc2 = caller_leave(h, D, caller)) return rc ? rc : rc2;
    return rc;
  }
  // host arrays: staged in one device buffer, freed once the load has waited for its last kernel
  DeviceBuffer<float> stage;
  if (int rc = stage.allocate(h, D->stream, (size_t)n * (ids ? 5 : 4))) return rc;
  CUDA_TRY(cudaMemcpyAsync(stage, xyz, (size_t)n * 12, cudaMemcpyHostToDevice, D->stream));
  CUDA_TRY(cudaMemcpyAsync(stage + 3 * (size_t)n, ny, (size_t)n * 4, cudaMemcpyHostToDevice, D->stream));
  if (ids) CUDA_TRY(cudaMemcpyAsync(stage + 4 * (size_t)n, ids, (size_t)n * 4, cudaMemcpyHostToDevice, D->stream));
  D->ctr.h2d_bytes += (uint64_t)n * (ids ? 20 : 16);
  const int rc = load_core(h, P, D, stage, stage + 3 * (size_t)n, ids ? reinterpret_cast<const int32_t*>(stage + 4 * (size_t)n) : nullptr, n);
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  return rc;
}

int window(malio_handle* h, const double pos[3], double cube_len, float det_range, malio_window_report* rep) {
  PriorState* P = h->prior.get();
  if (!P || !P->loaded) { h->err = "malio_prior_map_window before malio_prior_map_load"; return MALIO_ERR_STATE; }
  for (int a = 0; a < 3; ++a)
    if (!std::isfinite(pos[a])) { h->err = "malio_prior_map_window: non-finite position"; return MALIO_ERR_INVALID_ARG; }
  if (!(cube_len > 0.0) || !std::isfinite(cube_len) || !(det_range >= 0.f) || !std::isfinite(det_range)) {
    h->err = "malio_prior_map_window: cube_len must be finite and > 0, det_range finite and >= 0";
    return MALIO_ERR_INVALID_ARG;
  }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  std::memset(rep, 0, sizeof(*rep));
  const bool first = !P->win || P->win_epoch != h->map_epoch;
  Cubes c{};
  if (first) {                                                                        // laserMapping.cpp:177-186
    for (int i = 0; i < 3; ++i) {
      c.nw[i] = (float)(pos[i] - cube_len / 2.0);
      c.nw[3 + i] = (float)(pos[i] + cube_len / 2.0);
    }
    c.has_old = 0;
    uint32_t m = 0;
    P->win = false;
    if (int rc = gather(h, P, D, c, &m)) return rc;
    if (int rc = feed(h, P, D, m, true)) return rc;   // malio_map_build: replaces the device map, commits
    std::memcpy(P->cube, c.nw, sizeof(c.nw));
    P->win = true;
    P->win_epoch = h->map_epoch;
    rep->initialized = 1;
    rep->n_entered = m;
  } else {                                                                            // :187-219
    const float thr = 1.5f * det_range;                                              // MOV_THRESHOLD * DET_RANGE
    float dist[3][2];
    bool need_move = false;
    for (int i = 0; i < 3; ++i) {
      dist[i][0] = (float)std::fabs(pos[i] - (double)P->cube[i]);
      dist[i][1] = (float)std::fabs(pos[i] - (double)P->cube[3 + i]);
      if (dist[i][0] <= thr || dist[i][1] <= thr) need_move = true;
    }
    if (need_move) {
      const double a = (cube_len - 2.0 * 1.5f * det_range) * 0.5 * 0.9, b = (double)(det_range * (1.5f - 1));
      const float mov_dist = (float)(a > b ? a : b);                                 // std::max<double>, stored as float
      float boxes[3][6];
      uint32_t nb = 0;
      std::memcpy(c.od, P->cube, sizeof(c.od));
      std::memcpy(c.nw, P->cube, sizeof(c.nw));
      for (int i = 0; i < 3; ++i) {
        float* tb = boxes[nb];
        std::memcpy(tb, P->cube, sizeof(P->cube));
        if (dist[i][0] <= thr) {
          c.nw[3 + i] -= mov_dist; c.nw[i] -= mov_dist;
          tb[i] = P->cube[3 + i] - mov_dist;
          ++nb;
        } else if (dist[i][1] <= thr) {
          c.nw[3 + i] += mov_dist; c.nw[i] += mov_dist;
          tb[3 + i] = P->cube[i] + mov_dist;
          ++nb;
        }
      }
      c.has_old = 1;
      uint32_t killed = 0, m = 0;
      P->win = false;   // until the slide is complete: after a failure the next call builds the window afresh
      if (int rc = malio_map::delete_boxes(h, &boxes[0][0], nb, &killed)) return rc;
      if (int rc = gather(h, P, D, c, &m)) return rc;
      if (int rc = feed(h, P, D, m, false)) return rc;
      std::memcpy(P->cube, c.nw, sizeof(c.nw));
      if (int rc = malio_map::commit(h)) return rc;
      P->win = true;
      rep->moved = 1;
      rep->n_boxes = nb;
      std::memcpy(rep->boxes, boxes, sizeof(float) * 6 * nb);
      rep->n_killed = killed;
      rep->n_entered = m;
    }
  }
  std::memcpy(rep->cube, P->cube, sizeof(P->cube));
  rep->n_live = (uint32_t)D->ctr.map_live;
  return MALIO_OK;
}

int points(const malio_handle* h, const float** xyzw, uint32_t* n) {
  const PriorState* P = h->prior.get();
  if (!P || !P->loaded) return MALIO_ERR_STATE;
  *xyzw = reinterpret_cast<const float*>(P->d_pts.data());
  *n = P->n;
  return MALIO_OK;
}

int info(malio_handle* h, uint64_t* n_points, uint32_t* n_tiles, uint64_t* device_bytes) {
  PriorState* P;
  DeviceState* D;
  if (int rc = acquire(h, h->prior, P, D)) return rc;
  if (n_points) *n_points = P->n;
  if (n_tiles) *n_tiles = P->n_tiles;
  if (device_bytes)
    *device_bytes = P->d_pts.bytes() + P->d_ids.bytes() + P->d_tkey.bytes() + P->d_toff.bytes() + P->d_rq.bytes() + P->d_rbeg.bytes() +
                    P->d_roff.bytes() + P->d_blk.bytes() + P->d_blkoff.bytes() + P->d_out.bytes() + P->d_temp.bytes();
  return MALIO_OK;
}

int clear(malio_handle* h) {
  if (!h->prior) return MALIO_OK;   // (nor a place database: one is built from a loaded prior)
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  release(h->place, D->stream);
  // an enqueued append may still read the scratch
  if (cudaError_t e = release(h->prior, D->stream)) return malio_buf::cuda_fail(h, "cudaStreamSynchronize(D->stream)", e);
  return MALIO_OK;
}

}  // namespace malio_prior

// localization in a prior map (malio_b200.h, after the device-resident map)
extern "C" int malio_prior_map_load(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n) {
  if (!h || (n && (!xyz || !normal_y))) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_prior::load(h, xyz, normal_y, ids, n, false, nullptr);
}
extern "C" int malio_prior_map_load_device(malio_handle* h, const float* d_xyz, const float* d_normal_y, const int32_t* d_ids, uint32_t n,
                                           void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_prior::load(h, d_xyz, d_normal_y, d_ids, n, true, (cudaStream_t)stream);
}
extern "C" int malio_prior_map_window(malio_handle* h, const double pos_lid[3], double cube_len, float det_range, malio_window_report* rep) {
  if (!h || !pos_lid || !rep) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_prior::window(h, pos_lid, cube_len, det_range, rep);
}
extern "C" int malio_prior_map_info(malio_handle* h, uint64_t* n_points, uint32_t* n_tiles, uint64_t* device_bytes) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_prior::info(h, n_points, n_tiles, device_bytes);
}
extern "C" int malio_prior_map_clear(malio_handle* h) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_prior::clear(h);
}
