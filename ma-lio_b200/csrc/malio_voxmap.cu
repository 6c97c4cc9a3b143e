// malio_voxmap.cu — the saved map as a bounded voxel map on the device, sm_90a: every accumulated dense registered scan
// (the cloud malio_world_accumulate appends, laserMapping.cpp:466-488) folded into per-voxel centroids, so that the saved
// map grows with the mapped area instead of with the length of the run.  A deliberate extension beyond the reference, which
// keeps and writes the dense pcl_wait_save.  What it writes is pcl::VoxelGrid (malio_voxel_grid, DESIGN.md §(f) N3) applied
// to the concatenation of those clouds, with absolute voxel indices instead of a grid over one cloud's bounding box:
//   voxel of a point  (int)floorf(x * il) per axis, il = 1.0f / leaf (float); non-finite points are skipped
//   centroid          float sums from 0.f in accumulation order (slot 0..L-1, point order, scan after scan), u32 count,
//                     sum / (float)count: vg_centroid_kernel's arithmetic on the concatenated cloud
//   output order      ascending (k, j, i) = (z, y, x) voxel index as signed ints
// Per scan, O(points in the scan), whatever the size of the map:
//   vm_key_kernel     body_to_world (the bits of world_kernel) and the voxel key of every dense point
//   radix sort        stable, of (key, point index) over the 96-bit key (CUB, k most significant, double-buffered)
//   runs              one run per distinct key; each run looked up in a persistent open-addressing hash (key -> entry)
//   new entries       numbered by an exclusive scan over the runs in key order (deterministic, whatever the hash layout)
//   vm_fold_kernel    one thread per run continues its voxel's sums in point order (the points registered again)
// The map is sorted by key on download / save only.  Compiled with -fmad=false like the rest of the library.
// Carving (malio_world_voxel_accumulate_carve, DESIGN.md "Clearing moving objects"): the same fold, then per scan
//   vc_hit_kernel     one thread per run: hit += 1 on the run's entry (rent, or small[2] + rank for a new one), stamp = scan
//   vc_carve_kernel   one thread per ray (slot origin -> dense point): a double-precision DDA over the voxel indices; every
//                     passed cell that the hash holds gets miss += 1 once per scan (the first thread to raise its stamp)
// and on a kept download / save a flag per voxel in key order, an exclusive scan and a compaction of the order, ahead of
// vm_centroid_kernel's arithmetic (the kept centroids are the unfiltered ones' bits).
// Seeding (malio_world_voxel_seed*, DESIGN.md "Keeping a saved map current"): the same pipeline per chunk of saved points, with
// vs_key_kernel / vs_fold_kernel reading float4 rows, then vs_hits_kernel over the seeded entries [0, n_seeded); the changes
// are vs_change_kernel's two flags per voxel in key order, each scanned and compacted as the kept download is.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <string>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda/std/tuple>

#include "malio_device.cuh"

using namespace malio_devstate;

namespace {

struct VKey { int k, j, i; };   // voxel index along z, y, x
struct VKeyDecomposer {
  __host__ __device__ ::cuda::std::tuple<int&, int&, int&> operator()(VKey& v) const { return {v.k, v.j, v.i}; }
};

constexpr uint32_t EMPTY = 0xFFFFFFFFu;      // hash slot without an entry
// key of the points that are not folded (non-finite, or outside int).  No voxel has it: an index in int is floorf(..) < 2^31
// in float, so at most 2147483520
constexpr int SKIP_K = INT_MAX;
constexpr uint32_t RUN_NONE = 0xFFFFFFFFu;   // the run of the skipped points
constexpr uint32_t RUN_NEW = 0xFFFFFFFEu;    // run whose voxel the map does not hold yet
constexpr uint64_t VOX_MIN_ENTRIES = 1u << 16;

struct VoxState {
  bool leaf_set = false;
  float leaf = 0.f;
  uint64_t n_vox = 0;                        // entries in use (exact on the host after every call)
  DeviceBuffer<VKey> d_ekey; DeviceBuffer<float4> d_esum; DeviceBuffer<uint32_t> d_ecnt;   // entries
  DeviceBuffer<uint32_t> d_hash;                                                           // power of two
  // sort area, rows of 32 B (one allocation): keys | alternate keys (12 B each) | values | alternate values (4 B each), sized
  // for the points of a scan or, on download and save, for the entries.  A save writes the sorted centroids (16 B a row)
  // over the two key halves and then releases the area; a download keeps it until the next save.
  DeviceBuffer<char> d_sort;
  // run scratch, 16 B a row, sized for the points of a scan only
  DeviceBuffer<uint32_t> d_head, d_run, d_rent, d_new;
  DeviceBuffer<char> d_temp;                 // CUB's temporary storage (sort histograms, scan carries)
  DeviceBuffer<uint32_t> d_small;            // [0] fault flag, [1] run count, [2] entries in use, [3] kept / removed count, [5] added
  PinnedBuffer<uint32_t> h_small;            // pinned mirror of d_small
  PinnedBuffer<float4> h_bounce;             // pinned, malio_pcd::CHUNK points
  // carving evidence, 12 B per entry, allocated by the first carve call and grown with the entries.  Entries at or beyond
  // n_vox hold zeros, so that an entry a later fold creates starts at hit = miss = 0.
  DeviceBuffer<uint2> d_hm;                  // (hit, miss)
  DeviceBuffer<uint32_t> d_stamp;            // the last carve scan that hit or passed the entry (0: none)
  uint32_t carve_scan = 0;                   // carve calls since creation or the last clearing save
  // the seeded voxels are the entries [0, n_seeded): entries are numbered in creation order and never renumbered (growth and
  // rehash keep them), and a seed only runs on an empty map.  0 for a map that was never seeded or since a clearing save.
  uint64_t n_seeded = 0;
};
constexpr size_t SORT_ROW = 2 * sizeof(VKey) + 2 * sizeof(uint32_t);
constexpr size_t RUN_ROW = 4 * sizeof(uint32_t);

// the four arrays of the sort area as CUB's double buffers
struct SortBufs {
  cub::DoubleBuffer<VKey> k;
  cub::DoubleBuffer<uint32_t> v;
};
uint64_t sort_rows(const VoxState* V) { return V->d_sort.size() / SORT_ROW; }
SortBufs sort_bufs(const VoxState* V) {
  const uint64_t rows = sort_rows(V);
  VKey* k = reinterpret_cast<VKey*>(V->d_sort.data());
  uint32_t* v = reinterpret_cast<uint32_t*>(V->d_sort + 2 * sizeof(VKey) * rows);
  return SortBufs{cub::DoubleBuffer<VKey>(k, k + rows), cub::DoubleBuffer<uint32_t>(v, v + rows)};
}

// the dense cloud: slot of global point p and its undistorted row
struct VmSlots {
  const float* ud[MALIO_MAX_LIDAR];
  float tag[MALIO_MAX_LIDAR];
  uint32_t first[MALIO_MAX_LIDAR + 1];
  int L;
};

__device__ __forceinline__ float world_point(const VmSlots& c, const PassConst& pc, uint32_t p, float w[3]) {
  int l = 0;
  while (l + 1 < c.L && p >= c.first[l + 1]) ++l;
  const float* r = c.ud[l] + 5 * (size_t)(p - c.first[l]);
  body_to_world(pc, l, r[0], r[1], r[2], w);
  return c.tag[l];
}

__device__ __forceinline__ uint64_t vhash(const VKey& a) {
  uint64_t h = (uint64_t)(uint32_t)a.i * 0x9E3779B97F4A7C15ull ^ (uint64_t)(uint32_t)a.j * 0xC2B2AE3D27D4EB4Full ^
               (uint64_t)(uint32_t)a.k * 0x165667B19E3779F9ull;
  h ^= h >> 31; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 29;
  return h;
}
__device__ __forceinline__ bool same(const VKey& a, const VKey& b) { return a.k == b.k && a.j == b.j && a.i == b.i; }

__global__ void __launch_bounds__(256) vm_key_kernel(VmSlots c, PassConst pc, float il, uint32_t n, VKey* __restrict__ key,
                                                     uint32_t* __restrict__ val, uint32_t* __restrict__ fault) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n) return;
  float w[3];
  world_point(c, pc, p, w);
  const VKey none{SKIP_K, SKIP_K, SKIP_K};
  val[p] = p;
  if (!(isfinite(w[0]) && isfinite(w[1]) && isfinite(w[2]))) { key[p] = none; return; }
  const float fx = floorf(w[0] * il), fy = floorf(w[1] * il), fz = floorf(w[2] * il);
  const bool in_int = fx >= -2147483648.f && fx < 2147483648.f && fy >= -2147483648.f && fy < 2147483648.f &&
                      fz >= -2147483648.f && fz < 2147483648.f;
  if (!in_int) { atomicOr(fault, 1u); key[p] = none; return; }
  key[p] = VKey{(int)fz, (int)fy, (int)fx};
}

__global__ void __launch_bounds__(256) vm_head_kernel(const VKey* __restrict__ key, uint32_t n, uint32_t* __restrict__ head) {
  const uint32_t q = blockIdx.x * 256u + threadIdx.x;
  if (q >= n) return;
  head[q] = (q == 0 || !same(key[q], key[q - 1])) ? 1u : 0u;
}

// run r starts at run[r]; small[1] = number of runs
__global__ void __launch_bounds__(256) vm_run_kernel(const uint32_t* __restrict__ head, const uint32_t* __restrict__ incl, uint32_t n,
                                                     uint32_t* __restrict__ run, uint32_t* __restrict__ small) {
  const uint32_t q = blockIdx.x * 256u + threadIdx.x;
  if (q >= n) return;
  if (head[q]) run[incl[q] - 1] = q;
  if (q == n - 1) small[1] = incl[q];
}

__global__ void __launch_bounds__(256) vm_lookup_kernel(const uint32_t* __restrict__ run, const VKey* __restrict__ key,
                                                        uint32_t n, const uint32_t* __restrict__ small,
                                                        const uint32_t* __restrict__ hash, uint64_t mask, const VKey* __restrict__ ekey,
                                                        uint32_t* __restrict__ rent, uint32_t* __restrict__ is_new) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  const uint32_t nr = small[1];
  if (r >= nr) { is_new[r] = 0; return; }
  const VKey k = key[run[r]];
  if (k.k == SKIP_K) { rent[r] = RUN_NONE; is_new[r] = 0; return; }
  for (uint64_t s = vhash(k) & mask;; s = (s + 1) & mask) {
    const uint32_t e = hash[s];
    if (e == EMPTY) { rent[r] = RUN_NEW; is_new[r] = 1; return; }
    if (same(ekey[e], k)) { rent[r] = e; is_new[r] = 0; return; }
  }
}

// one thread per run: the voxel's entry (a new one numbered in key order and entered into the hash), then its sums continued
// point by point.  Nothing is written when the scan has a point outside int (small[0]): the map stays as it was.
__global__ void __launch_bounds__(128) vm_fold_kernel(VmSlots c, PassConst pc, const uint32_t* __restrict__ run,
                                                      const VKey* __restrict__ key, const uint32_t* __restrict__ val, uint32_t n,
                                                      const uint32_t* __restrict__ small, const uint32_t* __restrict__ rent,
                                                      const uint32_t* __restrict__ rank, uint32_t* __restrict__ hash, uint64_t mask,
                                                      VKey* __restrict__ ekey, float4* __restrict__ esum, uint32_t* __restrict__ ecnt) {
  const uint32_t r = blockIdx.x * 128u + threadIdx.x;
  if (small[0]) return;
  const uint32_t nr = small[1];
  if (r >= nr) return;
  uint32_t e = rent[r];
  if (e == RUN_NONE) return;
  const uint32_t q0 = run[r], q1 = r + 1 < nr ? run[r + 1] : n;
  float4 s;
  uint32_t cnt;
  if (e == RUN_NEW) {
    e = small[2] + rank[r];
    const VKey k = key[q0];
    uint64_t slot = vhash(k) & mask;
    while (atomicCAS(hash + slot, EMPTY, e) != EMPTY) slot = (slot + 1) & mask;
    ekey[e] = k;
    s = make_float4(0.f, 0.f, 0.f, 0.f);
    cnt = 0;
  } else {
    s = esum[e];
    cnt = ecnt[e];
  }
  for (uint32_t q = q0; q < q1; ++q) {
    const uint32_t p = val[q];
    float w[3];
    const float tag = world_point(c, pc, p, w);
    s.x += w[0]; s.y += w[1]; s.z += w[2]; s.w += tag;
    ++cnt;
  }
  esum[e] = s;
  ecnt[e] = cnt;
}

// after the fold: the entry count grows by the new runs unless the scan was refused
__global__ void vm_count_kernel(const uint32_t* __restrict__ rank, const uint32_t* __restrict__ is_new, uint32_t* __restrict__ small) {
  const uint32_t nr = small[1];
  if (small[0] || nr == 0) return;
  small[2] += rank[nr - 1] + is_new[nr - 1];
}

__global__ void __launch_bounds__(256) vm_rehash_kernel(const VKey* __restrict__ ekey, uint32_t n, uint32_t* __restrict__ hash, uint64_t mask) {
  const uint32_t e = blockIdx.x * 256u + threadIdx.x;
  if (e >= n) return;
  uint64_t slot = vhash(ekey[e]) & mask;
  while (atomicCAS(hash + slot, EMPTY, e) != EMPTY) slot = (slot + 1) & mask;
}

__global__ void __launch_bounds__(256) vm_iota_kernel(const VKey* __restrict__ ekey, uint32_t n, VKey* __restrict__ key, uint32_t* __restrict__ val) {
  const uint32_t e = blockIdx.x * 256u + threadIdx.x;
  if (e >= n) return;
  key[e] = ekey[e];
  val[e] = e;
}

// the r-th voxel in key order -> out[r] (r < cap)
__global__ void __launch_bounds__(256) vm_centroid_kernel(const uint32_t* __restrict__ order, uint32_t n, const float4* __restrict__ esum,
                                                          const uint32_t* __restrict__ ecnt, float4* __restrict__ out, uint32_t cap) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n || r >= cap) return;
  const uint32_t e = order[r];
  const float4 s = esum[e];
  const float cf = (float)ecnt[e];
  out[r] = make_float4(s.x / cf, s.y / cf, s.z / cf, s.w / cf);
}

// ------------------------------------------------------------------ carving (malio_world_voxel_accumulate_carve)
__device__ __forceinline__ bool in_int(float f) { return f >= -2147483648.f && f < 2147483648.f; }

// before the fold: the origin of every slot that has points needs a voxel index in int, like the ends (vm_key_kernel), or
// the scan is refused through the same fault flag
__global__ void vc_origin_kernel(VmSlots c, PassConst pc, float il, uint32_t* __restrict__ fault) {
  const int l = threadIdx.x;
  if (l >= c.L || c.first[l + 1] == c.first[l]) return;
  float o[3];
  body_to_world(pc, l, 0.f, 0.f, 0.f, o);
  if (!(in_int(floorf(o[0] * il)) && in_int(floorf(o[1] * il)) && in_int(floorf(o[2] * il)))) atomicOr(fault, 1u);
}

// between the fold and vm_count_kernel (small[2] still counts the entries before this scan): one thread per run
__global__ void __launch_bounds__(256) vc_hit_kernel(const uint32_t* __restrict__ small, const uint32_t* __restrict__ rent,
                                                     const uint32_t* __restrict__ rank, uint32_t n, uint2* __restrict__ hm,
                                                     uint32_t* __restrict__ stamp, uint32_t scan) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (small[0] || r >= n || r >= small[1]) return;
  uint32_t e = rent[r];
  if (e == RUN_NONE) return;
  if (e == RUN_NEW) e = small[2] + rank[r];
  hm[e].x += 1u;
  stamp[e] = scan;
}

// one axis of the DDA: the next face's parameter, (face - u) * inv in double (the header's order)
__device__ __forceinline__ double vc_face(int cell, int step, float u, double inv) {
  return ((double)cell + (step > 0 ? 1.0 : 0.0) - (double)u) * inv;
}

// one thread per ray of the scan (after the fold and vm_count_kernel: the hash holds this scan's new entries).  The walk takes
// exactly |di| + |dj| + |dk| steps from floor(u) to floor(e), each along the eligible axis (steps left) whose next face comes
// first, ties to x, then y, then z; it stops at the first cell that is not passed (the entry parameters never decrease).
__global__ void __launch_bounds__(256) vc_carve_kernel(VmSlots c, PassConst pc, float il, uint32_t n, double max_range,
                                                       double end_margin, const uint32_t* __restrict__ small,
                                                       const uint32_t* __restrict__ hash, uint64_t mask,
                                                       const VKey* __restrict__ ekey, uint2* __restrict__ hm,
                                                       uint32_t* __restrict__ stamp, uint32_t scan) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n || small[0]) return;
  int l = 0;
  while (l + 1 < c.L && p >= c.first[l + 1]) ++l;
  const float* row = c.ud[l] + 5 * (size_t)(p - c.first[l]);
  float w[3], o[3];
  body_to_world(pc, l, row[0], row[1], row[2], w);
  if (!(isfinite(w[0]) && isfinite(w[1]) && isfinite(w[2]))) return;
  body_to_world(pc, l, 0.f, 0.f, 0.f, o);
  const double dx = (double)w[0] - (double)o[0], dy = (double)w[1] - (double)o[1], dz = (double)w[2] - (double)o[2];
  const double len = sqrt(dx * dx + dy * dy + dz * dz);
  const double lim = fmin(max_range, len - end_margin);
  const float ux = o[0] * il, uy = o[1] * il, uz = o[2] * il;
  const float ex = w[0] * il, ey = w[1] * il, ez = w[2] * il;
  int cx = (int)floorf(ux), cy = (int)floorf(uy), cz = (int)floorf(uz);
  const int gx = (int)floorf(ex), gy = (int)floorf(ey), gz = (int)floorf(ez);
  const int sx = gx > cx ? 1 : -1, sy = gy > cy ? 1 : -1, sz = gz > cz ? 1 : -1;
  uint32_t rx = (uint32_t)(gx > cx ? (long long)gx - cx : (long long)cx - gx);
  uint32_t ry = (uint32_t)(gy > cy ? (long long)gy - cy : (long long)cy - gy);
  uint32_t rz = (uint32_t)(gz > cz ? (long long)gz - cz : (long long)cz - gz);
  const double ix = 1.0 / ((double)ex - (double)ux), iy = 1.0 / ((double)ey - (double)uy), iz = 1.0 / ((double)ez - (double)uz);
  double tx = rx ? vc_face(cx, sx, ux, ix) : 0.0, ty = ry ? vc_face(cy, sy, uy, iy) : 0.0, tz = rz ? vc_face(cz, sz, uz, iz) : 0.0;
  double t = 0.0;   // entry parameter of the current cell
  while ((rx | ry | rz) && t * len < lim) {
    const VKey k{cz, cy, cx};
    for (uint64_t s = vhash(k) & mask;; s = (s + 1) & mask) {
      const uint32_t e = hash[s];
      if (e == EMPTY) break;
      if (same(ekey[e], k)) {
        if (*(volatile const uint32_t*)(stamp + e) != scan && atomicMax(stamp + e, scan) < scan) hm[e].y += 1u;
        break;
      }
    }
    int a = rx ? 0 : (ry ? 1 : 2);
    double ta = rx ? tx : (ry ? ty : tz);
    if (ry && ty < ta) { a = 1; ta = ty; }
    if (rz && tz < ta) { a = 2; ta = tz; }
    t = ta;
    if (a == 0) { cx += sx; --rx; tx = vc_face(cx, sx, ux, ix); }
    else if (a == 1) { cy += sy; --ry; ty = vc_face(cy, sy, uy, iy); }
    else { cz += sz; --rz; tz = vc_face(cz, sz, uz, iz); }
  }
}

// (hit, miss) of the r-th voxel in key order -> out[r], r < n (zeros for a map that was never carved)
__global__ void __launch_bounds__(256) vc_evidence_kernel(const uint32_t* __restrict__ order, uint32_t n, const uint2* __restrict__ hm,
                                                          uint2* __restrict__ out) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  out[r] = hm ? hm[order[r]] : make_uint2(0u, 0u);
}

// the keep rule on the r-th voxel in key order: dropped when miss >= min_miss and (double)miss > ratio * (double)hit
__global__ void __launch_bounds__(256) vc_keep_kernel(const uint32_t* __restrict__ order, uint32_t n, const uint2* __restrict__ hm,
                                                      uint32_t min_miss, double ratio, uint32_t* __restrict__ keep) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  const uint2 v = hm ? hm[order[r]] : make_uint2(0u, 0u);
  keep[r] = (v.y >= min_miss && (double)v.y > ratio * (double)v.x) ? 0u : 1u;
}

// the kept entries in key order -> kept[0 .. small[3])
__global__ void __launch_bounds__(256) vc_compact_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ keep,
                                                         const uint32_t* __restrict__ pos, uint32_t n, uint32_t* __restrict__ kept,
                                                         uint32_t* __restrict__ small) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  if (keep[r]) kept[pos[r]] = order[r];
  if (r == n - 1) small[3] = pos[r] + keep[r];
}

// ------------------------------------------------------------------ seeding (malio_world_voxel_seed*) and the changes
// vm_key_kernel's key on seed row p of a chunk: the row's xyz are the world bits as given
__global__ void __launch_bounds__(256) vs_key_kernel(const float4* __restrict__ xyzi, float il, uint32_t n, VKey* __restrict__ key,
                                                     uint32_t* __restrict__ val, uint32_t* __restrict__ fault) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n) return;
  const float4 r = xyzi[p];
  const VKey none{SKIP_K, SKIP_K, SKIP_K};
  val[p] = p;
  if (!(isfinite(r.x) && isfinite(r.y) && isfinite(r.z))) { key[p] = none; return; }
  const float fx = floorf(r.x * il), fy = floorf(r.y * il), fz = floorf(r.z * il);
  if (!(in_int(fx) && in_int(fy) && in_int(fz))) { atomicOr(fault, 1u); key[p] = none; return; }
  key[p] = VKey{(int)fz, (int)fy, (int)fx};
}

// vm_fold_kernel on seed rows: one thread per run continues its voxel's sums row by row, intensity = the row's fourth float.
// Nothing is written once a chunk of this seed had a point outside int (small[0] is not reset between chunks).
__global__ void __launch_bounds__(128) vs_fold_kernel(const float4* __restrict__ xyzi, const uint32_t* __restrict__ run,
                                                      const VKey* __restrict__ key, const uint32_t* __restrict__ val, uint32_t n,
                                                      const uint32_t* __restrict__ small, const uint32_t* __restrict__ rent,
                                                      const uint32_t* __restrict__ rank, uint32_t* __restrict__ hash, uint64_t mask,
                                                      VKey* __restrict__ ekey, float4* __restrict__ esum, uint32_t* __restrict__ ecnt) {
  const uint32_t r = blockIdx.x * 128u + threadIdx.x;
  if (small[0]) return;
  const uint32_t nr = small[1];
  if (r >= nr) return;
  uint32_t e = rent[r];
  if (e == RUN_NONE) return;
  const uint32_t q0 = run[r], q1 = r + 1 < nr ? run[r + 1] : n;
  float4 s;
  uint32_t cnt;
  if (e == RUN_NEW) {
    e = small[2] + rank[r];
    const VKey k = key[q0];
    uint64_t slot = vhash(k) & mask;
    while (atomicCAS(hash + slot, EMPTY, e) != EMPTY) slot = (slot + 1) & mask;
    ekey[e] = k;
    s = make_float4(0.f, 0.f, 0.f, 0.f);
    cnt = 0;
  } else {
    s = esum[e];
    cnt = ecnt[e];
  }
  for (uint32_t q = q0; q < q1; ++q) {
    const float4 p = xyzi[val[q]];
    s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w;
    ++cnt;
  }
  esum[e] = s;
  ecnt[e] = cnt;
}

// after the last chunk: the seeded entries [0, small[2]) start at (seed_hits, 0), stamp 0
__global__ void __launch_bounds__(256) vs_hits_kernel(const uint32_t* __restrict__ small, uint32_t n, uint32_t seed_hits,
                                                      uint2* __restrict__ hm, uint32_t* __restrict__ stamp) {
  const uint32_t e = blockIdx.x * 256u + threadIdx.x;
  if (small[0] || e >= n || e >= small[2]) return;
  hm[e] = make_uint2(seed_hits, 0u);
  stamp[e] = 0u;
}

// the r-th voxel in key order: removed[r] = seeded and dropped by the keep rule (vc_keep_kernel's arithmetic), added[r] = not
// seeded and kept
__global__ void __launch_bounds__(256) vs_change_kernel(const uint32_t* __restrict__ order, uint32_t n, const uint2* __restrict__ hm,
                                                        uint32_t min_miss, double ratio, uint32_t n_seeded,
                                                        uint32_t* __restrict__ removed, uint32_t* __restrict__ added) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  const uint32_t e = order[r];
  const uint2 v = hm ? hm[e] : make_uint2(0u, 0u);
  const bool kept = !(v.y >= min_miss && (double)v.y > ratio * (double)v.x);
  const bool seeded = e < n_seeded;
  removed[r] = (seeded && !kept) ? 1u : 0u;
  added[r] = (!seeded && kept) ? 1u : 0u;
}

int get_state(malio_handle* h, VoxState*& V) {
  V = (VoxState*)h->voxmap;
  if (V) return MALIO_OK;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  V = new VoxState;
  h->voxmap = V;
  if (int rc = V->d_small.allocate(h, D->stream, 6)) return rc;
  CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 6 * sizeof(uint32_t), D->stream));
  return V->h_small.allocate(h, 6);
}

// CUB's temporary storage for at least t bytes, and the sort area for n rows
int grow_temp(malio_handle* h, VoxState* V, DeviceState* D, size_t t) {
  if (t <= V->d_temp.size()) return MALIO_OK;
  return V->d_temp.allocate(h, D->stream, t + t / 8 + 4096);
}
int grow_sort(malio_handle* h, VoxState* V, DeviceState* D, uint64_t n) {
  if (n > sort_rows(V)) {
    if (int rc = V->d_sort.allocate(h, D->stream, (n + n / 8 + 1024) * SORT_ROW)) return rc;
  }
  SortBufs b = sort_bufs(V);
  size_t t = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t, b.k, b.v, (int)n, VKeyDecomposer{}, D->stream));
  return grow_temp(h, V, D, t);
}
// the run scratch for the n points of a scan
int grow_runs(malio_handle* h, VoxState* V, DeviceState* D, uint64_t n) {
  if (n > V->d_head.size()) {
    const uint64_t c = n + n / 8 + 1024;
    if (int rc = malio_buf::allocate_group(h, D->stream, {{V->d_head, c}, {V->d_run, c}, {V->d_rent, c}, {V->d_new, c}})) return rc;
  }
  size_t t_incl = 0, t_excl = 0;
  uint32_t* un = nullptr;
  CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, t_incl, un, un, (int)n, D->stream));
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t_excl, un, un, (int)n, D->stream));
  return grow_temp(h, V, D, t_incl > t_excl ? t_incl : t_excl);
}

// room for `need` entries and a hash at most half full.  Entries move with a device-side copy, the hash is rebuilt from the
// entries' keys; a failed allocation leaves the map as it was.
int grow_table(malio_handle* h, VoxState* V, DeviceState* D, uint64_t need) {
  uint64_t hc = V->d_hash ? V->d_hash.size() : 2 * VOX_MIN_ENTRIES;
  while (hc < 2 * need) hc *= 2;
  if (need <= V->d_ekey.size() && hc == V->d_hash.size()) return MALIO_OK;
  if (need > 0x7FFFFFFFull) { h->err = "world voxel map: more than 2^31 - 1 voxels"; return MALIO_ERR_CAPACITY; }
  cudaStream_t st = D->stream;
  if (need > V->d_ekey.size()) {
    uint64_t c = V->d_ekey.size() * 2;
    if (c < need) c = need;
    if (c < VOX_MIN_ENTRIES) c = VOX_MIN_ENTRIES;
    const uint64_t k = V->n_vox;
    const cudaError_t e = V->d_hm ? malio_buf::grow_keep(st, {{V->d_ekey, c, k}, {V->d_esum, c, k}, {V->d_ecnt, c, k}, {V->d_hm, c, k},
                                                               {V->d_stamp, c, k}})
                                  : malio_buf::grow_keep(st, {{V->d_ekey, c, k}, {V->d_esum, c, k}, {V->d_ecnt, c, k}});
    if (e) {
      h->err = std::string("world voxel map: cannot grow to ") + std::to_string(c) + " voxels: " + cudaGetErrorString(e);
      return MALIO_ERR_CUDA;
    }
    if (V->d_hm) {   // the evidence of the entries to come starts at zero
      CUDA_TRY(cudaMemsetAsync(V->d_hm + k, 0, (c - k) * sizeof(uint2), st));
      CUDA_TRY(cudaMemsetAsync(V->d_stamp + k, 0, (c - k) * sizeof(uint32_t), st));
    }
  }
  if (hc != V->d_hash.size()) {   // a new table, rebuilt from the entries' keys
    if (const cudaError_t e = malio_buf::grow_keep(st, {{V->d_hash, hc}})) {
      h->err = std::string("world voxel map: cannot grow the hash to ") + std::to_string(hc) + " slots: " + cudaGetErrorString(e);
      return MALIO_ERR_CUDA;
    }
    CUDA_TRY(cudaMemsetAsync(V->d_hash, 0xFF, hc * sizeof(uint32_t), st));
    if (V->n_vox) {
      vm_rehash_kernel<<<(uint32_t)((V->n_vox + 255) / 256), 256, 0, st>>>(V->d_ekey, (uint32_t)V->n_vox, V->d_hash, hc - 1);
      D->ctr.kernel_launches += 1;
    }
    CUDA_TRY(cudaGetLastError());
  }
  return MALIO_OK;
}

// enqueue the sort of the entries by key on the handle's stream (sort area already grown): *order = the entries in key order,
// the values half CUB left current (the other values half and the key halves are free once it is sorted)
int enqueue_order(malio_handle* h, VoxState* V, DeviceState* D, SortBufs& b) {
  cudaStream_t st = D->stream;
  const uint32_t n = (uint32_t)V->n_vox;
  vm_iota_kernel<<<(n + 255) / 256, 256, 0, st>>>(V->d_ekey, n, b.k.Current(), b.v.Current());
  size_t t = V->d_temp.size();
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(V->d_temp, t, b.k, b.v, (int)n, VKeyDecomposer{}, st));
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

// enqueue the centroids in key order into out[0 .. min(n_vox, cap)) on the handle's stream (sort area already grown).  out may
// be the sort area itself (its two key halves, 24 B a row): the keys are dead once sorted, the order is read from the values.
int enqueue_sorted(malio_handle* h, VoxState* V, DeviceState* D, float4* out, uint64_t cap) {
  const uint32_t n = (uint32_t)V->n_vox;
  SortBufs b = sort_bufs(V);
  if (int rc = enqueue_order(h, V, D, b)) return rc;
  vm_centroid_kernel<<<(n + 255) / 256, 256, 0, D->stream>>>(b.v.Current(), n, V->d_esum, V->d_ecnt, out, cap < n ? (uint32_t)cap : n);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

// the kept entries in key order (malio_carve_keep), at 20 B into each row of the sort area: behind the centroids a save stages
// over the key halves (16 B a row), beside the flags' exclusive scan (16 B into the row)
uint32_t* kept_order(const VoxState* V) { return reinterpret_cast<uint32_t*>(V->d_sort + 20 * sort_rows(V)); }

// sort, flag, scan and compact the entries the keep rule does not drop into kept_order(V); waits for their count (*n_kept)
int enqueue_kept(malio_handle* h, VoxState* V, DeviceState* D, const malio_carve_keep* keep, uint64_t* n_kept) {
  cudaStream_t st = D->stream;
  const uint32_t n = (uint32_t)V->n_vox;
  SortBufs b = sort_bufs(V);
  size_t t = 0;
  uint32_t* un = nullptr;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t, un, un, (int)n, st));
  if (int rc = grow_temp(h, V, D, t)) return rc;
  if (int rc = enqueue_order(h, V, D, b)) return rc;
  uint32_t* flag = b.v.Alternate();
  uint32_t* pos = reinterpret_cast<uint32_t*>(V->d_sort + 16 * sort_rows(V));
  const uint32_t g = (n + 255) / 256;
  vc_keep_kernel<<<g, 256, 0, st>>>(b.v.Current(), n, V->d_hm, keep->min_miss, (double)keep->max_miss_per_hit, flag);
  t = V->d_temp.size();
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(V->d_temp, t, flag, pos, (int)n, st));
  vc_compact_kernel<<<g, 256, 0, st>>>(b.v.Current(), flag, pos, n, kept_order(V), V->d_small);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 2;
  CUDA_TRY(cudaMemcpyAsync(V->h_small + 3, V->d_small + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // the kept count sizes the caller's output and the file
  *n_kept = V->h_small[3];
  return MALIO_OK;
}

// The changes against the seed in key order, laid out in the sort area (row offsets in bytes per row): the removed order at 20
// (kept_order) and the added order at 16, both behind the centroids a save stages over the key halves; the added flags at 0,
// the removed flags in the values half the sort left free, the two exclusive scans at 4 and 8.  Sorts, flags, scans and
// compacts, then waits for the two counts.
uint32_t* added_order(const VoxState* V) { return reinterpret_cast<uint32_t*>(V->d_sort + 16 * sort_rows(V)); }
int enqueue_changes(malio_handle* h, VoxState* V, DeviceState* D, const malio_carve_keep* keep, uint64_t* n_removed, uint64_t* n_added) {
  cudaStream_t st = D->stream;
  const uint32_t n = (uint32_t)V->n_vox;
  const uint64_t rows = sort_rows(V);
  SortBufs b = sort_bufs(V);
  size_t t = 0;
  uint32_t* un = nullptr;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t, un, un, (int)n, st));
  if (int rc = grow_temp(h, V, D, t)) return rc;
  if (int rc = enqueue_order(h, V, D, b)) return rc;
  uint32_t* flag_r = b.v.Alternate();
  uint32_t* flag_a = reinterpret_cast<uint32_t*>(V->d_sort.data());
  uint32_t* pos_r = reinterpret_cast<uint32_t*>(V->d_sort + 4 * rows);
  uint32_t* pos_a = reinterpret_cast<uint32_t*>(V->d_sort + 8 * rows);
  const uint32_t g = (n + 255) / 256;
  vs_change_kernel<<<g, 256, 0, st>>>(b.v.Current(), n, V->d_hm, keep->min_miss, (double)keep->max_miss_per_hit,
                                      (uint32_t)V->n_seeded, flag_r, flag_a);
  t = V->d_temp.size();
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(V->d_temp, t, flag_r, pos_r, (int)n, st));
  vc_compact_kernel<<<g, 256, 0, st>>>(b.v.Current(), flag_r, pos_r, n, kept_order(V), V->d_small);        // -> small[3]
  t = V->d_temp.size();
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(V->d_temp, t, flag_a, pos_a, (int)n, st));
  vc_compact_kernel<<<g, 256, 0, st>>>(b.v.Current(), flag_a, pos_a, n, added_order(V), V->d_small + 2);   // -> small[5]
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 3;
  CUDA_TRY(cudaMemcpyAsync(V->h_small + 3, V->d_small + 3, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // the counts size the caller's outputs and the files
  *n_removed = V->h_small[3];
  *n_added = V->h_small[5];
  return MALIO_OK;
}

int check_keep(malio_handle* h, const malio_carve_keep* k) {
  if (!std::isfinite(k->max_miss_per_hit) || k->max_miss_per_hit < 0.f) {
    h->err = "world voxel keep rule: max_miss_per_hit must be finite and >= 0";
    return MALIO_ERR_INVALID_ARG;
  }
  return MALIO_OK;
}

// an empty map with its buffers kept (a clearing save); the next accumulate fixes the leaf again
int clear_map(malio_handle* h, VoxState* V, DeviceState* D) {
  CUDA_TRY(cudaMemsetAsync(V->d_hash, 0xFF, V->d_hash.size() * sizeof(uint32_t), D->stream));
  CUDA_TRY(cudaMemsetAsync(V->d_small + 2, 0, sizeof(uint32_t), D->stream));
  if (V->d_hm) {
    CUDA_TRY(cudaMemsetAsync(V->d_hm, 0, V->d_hm.size() * sizeof(uint2), D->stream));
    CUDA_TRY(cudaMemsetAsync(V->d_stamp, 0, V->d_stamp.size() * sizeof(uint32_t), D->stream));
  }
  V->n_vox = 0;
  V->leaf_set = false;
  V->carve_scan = 0;
  V->n_seeded = 0;
  return MALIO_OK;
}

int check_leaf(malio_handle* h, const VoxState* V, float leaf) {
  if (!(leaf > 0.f) || !std::isfinite(leaf)) { h->err = "world voxel map: leaf must be a finite size > 0"; return MALIO_ERR_INVALID_ARG; }
  if (V->leaf_set && leaf != V->leaf) {
    h->err = "world voxel map: leaf " + std::to_string(leaf) + " differs from the map's " + std::to_string(V->leaf) + " (clear the map to change it)";
    return MALIO_ERR_INVALID_ARG;
  }
  return MALIO_OK;
}

}  // namespace

namespace malio_vox {

void destroy(malio_handle* h) {
  delete (VoxState*)h->voxmap;
  h->voxmap = nullptr;
}

// carve == NULL: malio_world_voxel_accumulate; otherwise the same fold, then the scan's hits and passes (checked first)
int accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf, const malio_carve_args* carve,
               uint64_t* n_voxels) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (carve && !(std::isfinite(carve->max_range) && carve->max_range > 0.f && std::isfinite(carve->end_margin) && carve->end_margin >= 0.f)) {
    h->err = "world voxel carve: max_range must be finite and > 0, end_margin finite and >= 0";
    return MALIO_ERR_INVALID_ARG;
  }
  if (int rc = check_leaf(h, V, leaf)) return rc;
  if (carve && (double)carve->max_range * (double)(1.0f / leaf) > MALIO_CARVE_MAX_RANGE_CELLS) {
    h->err = "world voxel carve: max_range / leaf above MALIO_CARVE_MAX_RANGE_CELLS; the map is unchanged";
    return MALIO_ERR_CAPACITY;
  }
  VmSlots c{};
  uint32_t m[MALIO_MAX_LIDAR] = {0, 0, 0};
  if (int rc = malio_pre::world_dense_source(h, c.ud, m)) return rc;
  c.L = h->cfg.params.n_lidar;
  uint64_t n = 0;
  for (int l = 0; l < c.L; ++l) { c.tag[l] = slot_tag[l]; c.first[l] = (uint32_t)n; n += m[l]; }
  c.first[c.L] = (uint32_t)n;
  if (n > 0x7FFFFFFFull) { h->err = "world voxel map: more than 2^31 - 1 points in one scan"; return MALIO_ERR_CAPACITY; }
  const uint32_t scan = V->carve_scan + 1;
  if (n) {
    if (int rc = grow_table(h, V, D, V->n_vox + n)) return rc;
    if (int rc = grow_sort(h, V, D, n)) return rc;
    if (int rc = grow_runs(h, V, D, n)) return rc;
    if (carve && !V->d_hm) {   // the first carve: every entry so far starts at hit = miss = 0
      const size_t cap = V->d_ekey.size();
      if (int rc = malio_buf::allocate_group(h, D->stream, {{V->d_hm, cap}, {V->d_stamp, cap}})) return rc;
      CUDA_TRY(cudaMemsetAsync(V->d_hm, 0, cap * sizeof(uint2), D->stream));
      CUDA_TRY(cudaMemsetAsync(V->d_stamp, 0, cap * sizeof(uint32_t), D->stream));
    }
    cudaStream_t st = D->stream;
    const PassConst pc = make_pass_const(h, D, s);
    const uint32_t nn = (uint32_t)n, g = (nn + 255) / 256;
    const uint64_t mask = V->d_hash.size() - 1;
    CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 2 * sizeof(uint32_t), st));   // fault flag, run count
    SortBufs b = sort_bufs(V);
    vm_key_kernel<<<g, 256, 0, st>>>(c, pc, 1.0f / leaf, nn, b.k.Current(), b.v.Current(), V->d_small);
    if (carve) vc_origin_kernel<<<1, 32, 0, st>>>(c, pc, 1.0f / leaf, V->d_small);
    size_t t = V->d_temp.size();
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(V->d_temp, t, b.k, b.v, (int)nn, VKeyDecomposer{}, st));
    const VKey* key = b.k.Current();
    const uint32_t* val = b.v.Current();
    vm_head_kernel<<<g, 256, 0, st>>>(key, nn, V->d_head);
    t = V->d_temp.size();
    CUDA_TRY(cub::DeviceScan::InclusiveSum(V->d_temp, t, V->d_head.data(), V->d_rent.data(), (int)nn, st));
    vm_run_kernel<<<g, 256, 0, st>>>(V->d_head, V->d_rent, nn, V->d_run, V->d_small);
    vm_lookup_kernel<<<g, 256, 0, st>>>(V->d_run, key, nn, V->d_small, V->d_hash, mask, V->d_ekey, V->d_rent, V->d_new);
    t = V->d_temp.size();
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(V->d_temp, t, V->d_new.data(), V->d_head.data(), (int)nn, st));
    vm_fold_kernel<<<(nn + 127) / 128, 128, 0, st>>>(c, pc, V->d_run, key, val, nn, V->d_small, V->d_rent, V->d_head,
                                                    V->d_hash, mask, V->d_ekey, V->d_esum, V->d_ecnt);
    if (carve) vc_hit_kernel<<<g, 256, 0, st>>>(V->d_small, V->d_rent, V->d_head, nn, V->d_hm, V->d_stamp, scan);
    vm_count_kernel<<<1, 1, 0, st>>>(V->d_head, V->d_new, V->d_small);
    if (carve)
      vc_carve_kernel<<<g, 256, 0, st>>>(c, pc, 1.0f / leaf, nn, (double)carve->max_range, (double)carve->end_margin, V->d_small,
                                         V->d_hash, mask, V->d_ekey, V->d_hm, V->d_stamp, scan);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += carve ? 10 : 7;
    CUDA_TRY(cudaMemcpyAsync(V->h_small, V->d_small, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));   // the call's one wait: the fault flag and the entry count
    if (V->h_small[0]) {
      h->err = carve ? "world voxel carve: leaf size too small for a point's or a ray origin's coordinates (voxel index outside int); the map is unchanged"
                     : "world voxel map: leaf size too small for a point's coordinates (voxel index outside int); the map is unchanged";
      return MALIO_ERR_CAPACITY;
    }
    V->n_vox = V->h_small[2];
  }
  if (carve) V->carve_scan = scan;
  V->leaf = leaf;
  V->leaf_set = true;
  if (n_voxels) *n_voxels = V->n_vox;
  return MALIO_OK;
}

int download_device(malio_handle* h, float* out, uint64_t cap, uint64_t* n_out, cudaStream_t caller) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  const uint64_t n = V->n_vox, k = n < cap ? n : cap;
  if (out && k) {
    if (int rc = check_device_ptr(h, D, out, "malio_world_voxel_download_device out")) return rc;
    if (reinterpret_cast<uintptr_t>(out) & 15u) {
      h->err = "malio_world_voxel_download_device out: not 16-byte aligned (the centroids are stored as float4)";
      return MALIO_ERR_INVALID_ARG;
    }
  }
  *n_out = n;
  if (!out || k == 0) return MALIO_OK;
  if (int rc = grow_sort(h, V, D, n)) return rc;
  if (int rc = caller_enter(h, D, caller)) return rc;
  if (int rc = enqueue_sorted(h, V, D, reinterpret_cast<float4*>(out), k)) return rc;
  return caller_leave(h, D, caller);
}

// the (hit, miss) pairs in the order of download_device, with its size protocol and device-memory contract
int evidence_device(malio_handle* h, uint32_t* out, uint64_t cap, uint64_t* n_out, cudaStream_t caller) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  const uint64_t n = V->n_vox, k = n < cap ? n : cap;
  if (out && k) {
    if (int rc = check_device_ptr(h, D, out, "malio_world_voxel_evidence_device out")) return rc;
    if (reinterpret_cast<uintptr_t>(out) & 7u) {
      h->err = "malio_world_voxel_evidence_device out: not 8-byte aligned (the pairs are stored as uint2)";
      return MALIO_ERR_INVALID_ARG;
    }
  }
  *n_out = n;
  if (!out || k == 0) return MALIO_OK;
  if (int rc = grow_sort(h, V, D, n)) return rc;
  if (int rc = caller_enter(h, D, caller)) return rc;
  SortBufs b = sort_bufs(V);
  if (int rc = enqueue_order(h, V, D, b)) return rc;
  vc_evidence_kernel<<<(uint32_t)((k + 255) / 256), 256, 0, D->stream>>>(b.v.Current(), (uint32_t)k, V->d_hm, reinterpret_cast<uint2*>(out));
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 1;
  return caller_leave(h, D, caller);
}

// the centroids of the kept voxels in the order of download_device; waits for their count before it enqueues the copy-out
int download_kept_device(malio_handle* h, const malio_carve_keep* keep, float* out, uint64_t cap, uint64_t* n_out, cudaStream_t caller) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (int rc = check_keep(h, keep)) return rc;
  if (out && cap && V->n_vox) {
    if (int rc = check_device_ptr(h, D, out, "malio_world_voxel_download_kept_device out")) return rc;
    if (reinterpret_cast<uintptr_t>(out) & 15u) {
      h->err = "malio_world_voxel_download_kept_device out: not 16-byte aligned (the centroids are stored as float4)";
      return MALIO_ERR_INVALID_ARG;
    }
  }
  uint64_t n = 0;
  if (V->n_vox) {
    if (int rc = grow_sort(h, V, D, V->n_vox)) return rc;
    if (int rc = enqueue_kept(h, V, D, keep, &n)) return rc;
  }
  *n_out = n;
  const uint64_t k = n < cap ? n : cap;
  if (!out || k == 0) return MALIO_OK;
  if (int rc = caller_enter(h, D, caller)) return rc;
  vm_centroid_kernel<<<(uint32_t)((k + 255) / 256), 256, 0, D->stream>>>(kept_order(V), (uint32_t)k, V->d_esum, V->d_ecnt,
                                                                          reinterpret_cast<float4*>(out), (uint32_t)k);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 1;
  return caller_leave(h, D, caller);
}

// keep == NULL: every voxel (malio_world_voxel_save_pcd); otherwise the voxels the rule keeps (malio_world_voxel_save_pcd_kept)
int save_pcd(malio_handle* h, const char* path, const malio_carve_keep* keep, int clear) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (keep) { if (int rc = check_keep(h, keep)) return rc; }
  if (V->n_vox == 0) { h->err = "world voxel save: the voxel map is empty (nothing is written)"; return MALIO_ERR_STATE; }
  uint64_t n = V->n_vox;
  if (int rc = grow_sort(h, V, D, n)) return rc;
  if (!V->h_bounce) { if (int rc = V->h_bounce.allocate(h, malio_pcd::CHUNK)) return rc; }
  float4* stage = reinterpret_cast<float4*>(V->d_sort.data());   // the key halves: 24 B a row, the centroids take 16
  if (keep) {
    if (int rc = enqueue_kept(h, V, D, keep, &n)) return rc;
    if (n == 0) {
      V->d_sort.release();   // enqueue_kept has waited for the stream
      V->d_temp.release();
      h->err = "world voxel save: the keep rule drops every voxel (nothing is written)";
      return MALIO_ERR_STATE;
    }
    vm_centroid_kernel<<<(uint32_t)((n + 255) / 256), 256, 0, D->stream>>>(kept_order(V), (uint32_t)n, V->d_esum, V->d_ecnt, stage,
                                                                            (uint32_t)n);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 1;
  } else if (int rc = enqueue_sorted(h, V, D, stage, n)) {
    return rc;
  }
  const int rc = malio_pcd::write_binary(path, n, [&](uint64_t first, uint64_t cnt, const float** xyzi) {
    if (cudaMemcpyAsync(V->h_bounce, stage + first, cnt * sizeof(float4), cudaMemcpyDeviceToHost, D->stream) != cudaSuccess ||
        cudaStreamSynchronize(D->stream) != cudaSuccess)
      return (int)MALIO_ERR_CUDA;
    D->ctr.d2h_bytes += cnt * sizeof(float4);
    *xyzi = (const float*)V->h_bounce.data();
    return (int)MALIO_OK;
  }, h->err);
  // the entry-sized sort area and CUB's storage go back: between saves the map holds its entries, its hash and the scan-sized
  // scratch only (the next accumulate regrows the sort area for its scan)
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  V->d_sort.release();
  V->d_temp.release();
  if (rc == MALIO_OK && clear) {
    if (int c = clear_map(h, V, D)) return c;
  }
  return rc;
}

// malio_world_voxel_seed (on_device false: xyzi in host memory, staged through the pinned bounce buffer into a chunk-sized
// device buffer) and malio_world_voxel_seed_device (xyzi read in place, ordered on `caller`).  The points are folded chunk by
// chunk in input order, each chunk through accumulate's pipeline with vs_key_kernel / vs_fold_kernel for the row source; the
// table is sized for n points before the first chunk, so the chunks are enqueued back to back and the call waits once.
int seed(malio_handle* h, const float* xyzi, uint64_t n, float leaf, uint32_t seed_hits, bool on_device, cudaStream_t caller,
         uint64_t* n_voxels) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (!(leaf > 0.f) || !std::isfinite(leaf)) { h->err = "world voxel seed: leaf must be a finite size > 0"; return MALIO_ERR_INVALID_ARG; }
  if (V->n_vox || V->leaf_set) {
    h->err = "world voxel seed: the voxel map is not empty (seed a new map or one after a clearing save)";
    return MALIO_ERR_STATE;
  }
  if (on_device) {
    if (int rc = check_device_ptr(h, D, xyzi, "malio_world_voxel_seed_device xyzi")) return rc;
    if (reinterpret_cast<uintptr_t>(xyzi) & 15u) {
      h->err = "malio_world_voxel_seed_device xyzi: not 16-byte aligned (the rows are read as float4)";
      return MALIO_ERR_INVALID_ARG;
    }
  }
  const uint64_t chunk = n < MALIO_SEED_CHUNK ? n : MALIO_SEED_CHUNK;
  if (int rc = grow_table(h, V, D, n)) return rc;
  if (int rc = grow_sort(h, V, D, chunk)) return rc;
  if (int rc = grow_runs(h, V, D, chunk)) return rc;
  const bool had_hm = (bool)V->d_hm;
  if (seed_hits && !had_hm) {   // the counters the first carve would allocate, zero beyond the seed
    const size_t cap = V->d_ekey.size();
    if (int rc = malio_buf::allocate_group(h, D->stream, {{V->d_hm, cap}, {V->d_stamp, cap}})) return rc;
    CUDA_TRY(cudaMemsetAsync(V->d_hm, 0, cap * sizeof(uint2), D->stream));
    CUDA_TRY(cudaMemsetAsync(V->d_stamp, 0, cap * sizeof(uint32_t), D->stream));
  }
  DeviceBuffer<float4> stage;
  if (!on_device) {
    if (int rc = stage.allocate(h, D->stream, chunk)) return rc;
    if (!V->h_bounce) { if (int rc = V->h_bounce.allocate(h, malio_pcd::CHUNK)) return rc; }
  } else if (int rc = caller_enter(h, D, caller)) {
    return rc;
  }
  cudaStream_t st = D->stream;
  const uint64_t mask = V->d_hash.size() - 1;
  const float il = 1.0f / leaf;
  CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 2 * sizeof(uint32_t), st));   // fault flag (kept over the chunks), run count
  const float4* rows = reinterpret_cast<const float4*>(xyzi);
  for (uint64_t first = 0; first < n; first += chunk) {
    const uint32_t m = (uint32_t)(n - first < chunk ? n - first : chunk), g = (m + 255) / 256;
    const float4* src = rows + first;
    if (!on_device) {   // the previous chunk's kernels and copies are done before the bounce buffer and the stage are reused
      for (uint32_t p = 0; p < m; p += malio_pcd::CHUNK) {
        const uint32_t c = m - p < malio_pcd::CHUNK ? m - p : malio_pcd::CHUNK;
        CUDA_TRY(cudaStreamSynchronize(st));
        std::memcpy(V->h_bounce.data(), rows + first + p, (size_t)c * sizeof(float4));
        CUDA_TRY(cudaMemcpyAsync(stage + p, V->h_bounce, (size_t)c * sizeof(float4), cudaMemcpyHostToDevice, st));
      }
      D->ctr.h2d_bytes += (uint64_t)m * sizeof(float4);
      src = stage;
    }
    SortBufs b = sort_bufs(V);
    vs_key_kernel<<<g, 256, 0, st>>>(src, il, m, b.k.Current(), b.v.Current(), V->d_small);
    size_t t = V->d_temp.size();
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(V->d_temp, t, b.k, b.v, (int)m, VKeyDecomposer{}, st));
    const VKey* key = b.k.Current();
    const uint32_t* val = b.v.Current();
    vm_head_kernel<<<g, 256, 0, st>>>(key, m, V->d_head);
    t = V->d_temp.size();
    CUDA_TRY(cub::DeviceScan::InclusiveSum(V->d_temp, t, V->d_head.data(), V->d_rent.data(), (int)m, st));
    vm_run_kernel<<<g, 256, 0, st>>>(V->d_head, V->d_rent, m, V->d_run, V->d_small);
    vm_lookup_kernel<<<g, 256, 0, st>>>(V->d_run, key, m, V->d_small, V->d_hash, mask, V->d_ekey, V->d_rent, V->d_new);
    t = V->d_temp.size();
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(V->d_temp, t, V->d_new.data(), V->d_head.data(), (int)m, st));
    vs_fold_kernel<<<(m + 127) / 128, 128, 0, st>>>(src, V->d_run, key, val, m, V->d_small, V->d_rent, V->d_head, V->d_hash, mask,
                                                   V->d_ekey, V->d_esum, V->d_ecnt);
    vm_count_kernel<<<1, 1, 0, st>>>(V->d_head, V->d_new, V->d_small);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 7;
  }
  if (V->d_hm) {
    const uint32_t nn = (uint32_t)n;
    vs_hits_kernel<<<(nn + 255) / 256, 256, 0, st>>>(V->d_small, nn, seed_hits, V->d_hm, V->d_stamp);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 1;
  }
  CUDA_TRY(cudaMemcpyAsync(V->h_small, V->d_small, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  if (on_device) { if (int rc = caller_leave(h, D, caller)) return rc; }
  CUDA_TRY(cudaStreamSynchronize(st));   // the call's one wait on device rows: the fault flag and the entry count
  if (V->h_small[0]) {   // an earlier chunk may have been folded: the map is made empty again, as it was
    if (int rc = clear_map(h, V, D)) return rc;
    if (!had_hm) {
      CUDA_TRY(cudaStreamSynchronize(st));
      V->d_hm.release();
      V->d_stamp.release();
    }
    h->err = "world voxel seed: leaf size too small for a point's coordinates (voxel index outside int); the map is empty";
    return MALIO_ERR_CAPACITY;
  }
  V->n_vox = V->h_small[2];
  V->n_seeded = V->n_vox;
  V->leaf = leaf;
  V->leaf_set = true;
  if (n_voxels) *n_voxels = V->n_vox;
  return MALIO_OK;
}

// removed / added centroids in the order of download_device, with download_kept_device's size protocol and contract
int changes_device(malio_handle* h, const malio_carve_keep* keep, float* d_removed, uint64_t cap_removed, uint64_t* n_removed,
                   float* d_added, uint64_t cap_added, uint64_t* n_added, cudaStream_t caller) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (int rc = check_keep(h, keep)) return rc;
  if (V->n_vox) {
    const struct { const float* out; uint64_t cap; const char* what; } outs[2] = {
        {d_removed, cap_removed, "malio_world_voxel_changes_device removed"}, {d_added, cap_added, "malio_world_voxel_changes_device added"}};
    for (const auto& o : outs) {
      if (!o.out || !o.cap) continue;
      if (int rc = check_device_ptr(h, D, o.out, o.what)) return rc;
      if (reinterpret_cast<uintptr_t>(o.out) & 15u) {
        h->err = std::string(o.what) + ": not 16-byte aligned (the centroids are stored as float4)";
        return MALIO_ERR_INVALID_ARG;
      }
    }
  }
  uint64_t nr = 0, na = 0;
  if (V->n_vox) {
    if (int rc = grow_sort(h, V, D, V->n_vox)) return rc;
    if (int rc = enqueue_changes(h, V, D, keep, &nr, &na)) return rc;
  }
  *n_removed = nr;
  *n_added = na;
  const uint64_t kr = d_removed ? (nr < cap_removed ? nr : cap_removed) : 0, ka = d_added ? (na < cap_added ? na : cap_added) : 0;
  if (kr == 0 && ka == 0) return MALIO_OK;
  if (int rc = caller_enter(h, D, caller)) return rc;
  if (kr)
    vm_centroid_kernel<<<(uint32_t)((kr + 255) / 256), 256, 0, D->stream>>>(kept_order(V), (uint32_t)kr, V->d_esum, V->d_ecnt,
                                                                             reinterpret_cast<float4*>(d_removed), (uint32_t)kr);
  if (ka)
    vm_centroid_kernel<<<(uint32_t)((ka + 255) / 256), 256, 0, D->stream>>>(added_order(V), (uint32_t)ka, V->d_esum, V->d_ecnt,
                                                                             reinterpret_cast<float4*>(d_added), (uint32_t)ka);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += (kr ? 1 : 0) + (ka ? 1 : 0);
  return caller_leave(h, D, caller);
}

// each set through save_pcd's writer (a NULL path or an empty set writes no file); the map is not cleared
int save_changes_pcd(malio_handle* h, const malio_carve_keep* keep, const char* removed_path, const char* added_path, uint64_t* n_removed,
                     uint64_t* n_added) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (int rc = check_keep(h, keep)) return rc;
  if (V->n_vox == 0) { h->err = "world voxel save: the voxel map is empty (nothing is written)"; return MALIO_ERR_STATE; }
  if (int rc = grow_sort(h, V, D, V->n_vox)) return rc;
  if (!V->h_bounce) { if (int rc = V->h_bounce.allocate(h, malio_pcd::CHUNK)) return rc; }
  uint64_t nr = 0, na = 0;
  if (int rc = enqueue_changes(h, V, D, keep, &nr, &na)) return rc;
  if (n_removed) *n_removed = nr;
  if (n_added) *n_added = na;
  float4* stage = reinterpret_cast<float4*>(V->d_sort.data());   // the key halves: both orders lie behind them
  int rc = MALIO_OK;
  const struct { const char* path; const uint32_t* order; uint64_t cnt; } sets[2] = {{removed_path, kept_order(V), nr},
                                                                                    {added_path, added_order(V), na}};
  for (const auto& set : sets) {
    const uint64_t cnt = set.cnt;
    if (rc != MALIO_OK || !set.path || cnt == 0) continue;
    vm_centroid_kernel<<<(uint32_t)((cnt + 255) / 256), 256, 0, D->stream>>>(set.order, (uint32_t)cnt, V->d_esum, V->d_ecnt, stage,
                                                                              (uint32_t)cnt);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 1;
    rc = malio_pcd::write_binary(set.path, cnt, [&](uint64_t first, uint64_t c, const float** xyzi) {
      if (cudaMemcpyAsync(V->h_bounce, stage + first, c * sizeof(float4), cudaMemcpyDeviceToHost, D->stream) != cudaSuccess ||
          cudaStreamSynchronize(D->stream) != cudaSuccess)
        return (int)MALIO_ERR_CUDA;
      D->ctr.d2h_bytes += c * sizeof(float4);
      *xyzi = (const float*)V->h_bounce.data();
      return (int)MALIO_OK;
    }, h->err);
  }
  CUDA_TRY(cudaStreamSynchronize(D->stream));   // as save_pcd: the entry-sized sort area and CUB's storage go back
  V->d_sort.release();
  V->d_temp.release();
  return rc;
}

int info(malio_handle* h, uint64_t* n_voxels, uint64_t* capacity, uint64_t* device_bytes) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  if (n_voxels) *n_voxels = V->n_vox;
  if (capacity) *capacity = V->d_ekey.size();
  if (device_bytes)
    *device_bytes = V->d_ekey.size() * (sizeof(VKey) + sizeof(float4) + sizeof(uint32_t)) + V->d_hash.size() * sizeof(uint32_t) +
                    V->d_sort.size() + V->d_head.size() * RUN_ROW + V->d_temp.size() +
                    V->d_hm.size() * sizeof(uint2) + V->d_stamp.size() * sizeof(uint32_t);
  return MALIO_OK;
}

}  // namespace malio_vox

// the saved map as a voxel map (malio_b200.h, next to malio_world_accumulate)
extern "C" int malio_world_voxel_accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf, uint64_t* n_voxels) {
  if (!h || !s) return MALIO_ERR_INVALID_ARG;
  if (!slot_tag) { h->err = "world voxel accumulate: the dense cloud needs slot_tag"; return MALIO_ERR_INVALID_ARG; }
  MALIO_SETTLE(h);
  return malio_vox::accumulate(h, s, slot_tag, leaf, nullptr, n_voxels);
}
extern "C" int malio_world_voxel_accumulate_carve(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf,
                                                  const malio_carve_args* a, uint64_t* n_voxels) {
  if (!h || !s || !a) return MALIO_ERR_INVALID_ARG;
  if (!slot_tag) { h->err = "world voxel accumulate: the dense cloud needs slot_tag"; return MALIO_ERR_INVALID_ARG; }
  MALIO_SETTLE(h);
  return malio_vox::accumulate(h, s, slot_tag, leaf, a, n_voxels);
}
extern "C" int malio_world_voxel_evidence_device(malio_handle* h, uint32_t* d_hit_miss, uint64_t cap, uint64_t* n_out, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!n_out || (cap && !d_hit_miss)) return MALIO_ERR_INVALID_ARG;
  return malio_vox::evidence_device(h, d_hit_miss, cap, n_out, (cudaStream_t)stream);
}
extern "C" int malio_world_voxel_download_kept_device(malio_handle* h, const malio_carve_keep* k, float* d_out, uint64_t cap,
                                                      uint64_t* n_out, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!k || !n_out || (cap && !d_out)) return MALIO_ERR_INVALID_ARG;
  return malio_vox::download_kept_device(h, k, d_out, cap, n_out, (cudaStream_t)stream);
}
extern "C" int malio_world_voxel_save_pcd_kept(malio_handle* h, const char* path, const malio_carve_keep* k, int clear) {
  if (!h || !path || !k) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::save_pcd(h, path, k, clear);
}
extern "C" int malio_world_voxel_seed(malio_handle* h, const float* xyzi, uint64_t n, float leaf, uint32_t seed_hits, uint64_t* n_voxels) {
  if (!h || !xyzi || n == 0) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::seed(h, xyzi, n, leaf, seed_hits, false, nullptr, n_voxels);
}
extern "C" int malio_world_voxel_seed_device(malio_handle* h, const float* d_xyzi, uint64_t n, float leaf, uint32_t seed_hits,
                                             uint64_t* n_voxels, void* stream) {
  if (!h || !d_xyzi || n == 0) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::seed(h, d_xyzi, n, leaf, seed_hits, true, (cudaStream_t)stream, n_voxels);
}
extern "C" int malio_world_voxel_changes_device(malio_handle* h, const malio_carve_keep* k, float* d_removed, uint64_t cap_removed,
                                                uint64_t* n_removed, float* d_added, uint64_t cap_added, uint64_t* n_added, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!k || !n_removed || !n_added || (cap_removed && !d_removed) || (cap_added && !d_added)) return MALIO_ERR_INVALID_ARG;
  return malio_vox::changes_device(h, k, d_removed, cap_removed, n_removed, d_added, cap_added, n_added, (cudaStream_t)stream);
}
extern "C" int malio_world_voxel_save_changes_pcd(malio_handle* h, const malio_carve_keep* k, const char* removed_path,
                                                  const char* added_path, uint64_t* n_removed, uint64_t* n_added) {
  if (!h || !k) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::save_changes_pcd(h, k, removed_path, added_path, n_removed, n_added);
}
extern "C" int malio_world_voxel_download_device(malio_handle* h, float* d_out, uint64_t cap, uint64_t* n_out, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!n_out || (cap && !d_out)) return MALIO_ERR_INVALID_ARG;
  return malio_vox::download_device(h, d_out, cap, n_out, (cudaStream_t)stream);
}
extern "C" int malio_world_voxel_save_pcd(malio_handle* h, const char* path, int clear) {
  if (!h || !path) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::save_pcd(h, path, nullptr, clear);
}
extern "C" int malio_world_voxel_info(malio_handle* h, uint64_t* n_voxels, uint64_t* capacity, uint64_t* device_bytes) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::info(h, n_voxels, capacity, device_bytes);
}
