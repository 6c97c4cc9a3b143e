// malio_voxmap.cu — the saved map as a bounded voxel map on the device, sm_90a: every accumulated dense registered scan
// (the cloud malio_world_accumulate appends, laserMapping.cpp:466-488) folded into per-voxel centroids, so that the saved
// map grows with the mapped area instead of with the length of the run.  A deliberate extension beyond the reference, which
// keeps and writes the dense pcl_wait_save.  What it writes is pcl::VoxelGrid (malio_voxel_grid, DESIGN.md §(f) N3) applied
// to the concatenation of those clouds, with absolute voxel indices instead of a grid over one cloud's bounding box:
//   voxel of a point  (int)floorf(x * il) per axis, il = 1.0f / leaf (float); non-finite points are skipped
//   centroid          float sums from 0.f in accumulation order (slot 0..L-1, point order, scan after scan), u32 count,
//                     sum / (float)count: vg_centroid_kernel's arithmetic on the concatenated cloud
//   output order      ascending (k, j, i) = (z, y, x) voxel index as signed ints
// The fold (enqueue_fold), per scan or per chunk of saved points, O(rows folded), whatever the size of the map.  The rows are
// a source type: ScanRows (the dense points, registered with body_to_world: the bits of world_kernel) or SeedRows (float4 rows):
//   vm_key_kernel     the voxel key of every row
//   radix sort        stable, of (key, row index) over the 96-bit key (CUB, k most significant, double-buffered)
//   runs              one run per distinct key; each run looked up in a persistent open-addressing hash (key -> entry)
//   new entries       numbered by an exclusive scan over the runs in key order (deterministic, whatever the hash layout)
//   vm_fold_kernel    one thread per run continues its voxel's sums in row order (the rows read again)
// The map is sorted by key on download / save only.  Compiled with -fmad=false like the rest of the library.
// Carving (malio_world_voxel_accumulate_carve, DESIGN.md "Clearing moving objects"): vc_origin_kernel, the same fold, then
//   vc_hit_kernel     one thread per run: hit += 1 on the run's entry (rent, or small[2] + rank for a new one), stamp = scan
//   vc_carve_kernel   one thread per ray (slot origin -> dense point): a double-precision DDA over the voxel indices; every
//                     passed cell that the hash holds gets miss += 1 once per scan (the first thread to raise its stamp)
// and on a kept download / save a flag per voxel in key order, an exclusive scan and a compaction of the order, ahead of
// vm_centroid_kernel's arithmetic (the kept centroids are the unfiltered ones' bits).
// Seeding (malio_world_voxel_seed*, DESIGN.md "Keeping a saved map current"): the same fold per chunk of saved points, then
// vs_hits_kernel over the seeded entries [0, n_seeded); the changes are vs_change_kernel's two flags per voxel in key order,
// each scanned and compacted as the kept download is.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda/std/tuple>

#include "malio_device.cuh"
#include "malio_voxrule.cuh"

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

}  // namespace

namespace malio_vox {

struct VoxState {
  bool leaf_set = false;
  float leaf = 0.f;
  uint64_t n_vox = 0;                        // entries in use (exact on the host after every call)
  DeviceBuffer<VKey> d_ekey; DeviceBuffer<float4> d_esum; DeviceBuffer<uint32_t> d_ecnt;   // entries
  DeviceBuffer<uint32_t> d_hash;                                                           // power of two
  // sort area, rows of 32 B in one allocation (the columns below), sized for the rows of a fold or, on download and save,
  // for the entries.  A download keeps it until the next save; a save releases it.
  DeviceBuffer<char> d_sort;
  // run scratch, 16 B a row, sized for the rows of a fold only
  DeviceBuffer<uint32_t> d_head, d_run, d_rent, d_new;
  CubTemp d_temp;                            // CUB's temporary storage (sort histograms, scan carries)
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

  int init(malio_handle* h, DeviceState* D) {
    if (int rc = d_small.allocate(h, D->stream, 6)) return rc;
    CUDA_TRY(cudaMemsetAsync(d_small, 0, 6 * sizeof(uint32_t), D->stream));
    return h_small.allocate(h, 6);
  }
};

}  // namespace malio_vox

namespace {

using malio_vox::VoxState;

// The sort area holds sort_rows(V) rows as eight columns of 4 B a row; column c starts at byte 4 * c * rows.  While points or
// entries are sorted, the columns are CUB's double buffers: keys in 0-2, alternate keys in 3-5 (12 B a row), values in 6,
// alternate values in 7.
constexpr uint32_t COL_KEYS = 0;
constexpr uint32_t COL_VALUES = 6;
constexpr size_t SORT_ROW = 8 * sizeof(uint32_t);
static_assert(SORT_ROW == 2 * sizeof(VKey) + 2 * sizeof(uint32_t), "a sort row holds two keys and two values");
// Once the entries are sorted (enqueue_order), their order is in the values column CUB left current and the key columns are
// free.  A selection (enqueue_select) writes there: a flag column beside the one in the values column the sort left free, an
// exclusive scan, and the selected entries in key order.  A save then stages the selected centroids, float4, over bytes 0-16
// of the rows (columns 0-3), so the orders it still reads must lie at byte 16 and above, and below the values.
constexpr uint32_t COL_FLAGS = 0;            // the added flags (enqueue_changes)
constexpr uint32_t COL_SCAN = 1;             // exclusive scan of a flag column
constexpr uint32_t COL_ADDED = 4;            // the added entries in key order
constexpr uint32_t COL_KEPT = 5;             // the kept, or the removed, entries in key order
static_assert(4 * COL_ADDED >= sizeof(float4) && 4 * COL_KEPT >= sizeof(float4), "a save's staged centroids cover the orders");
static_assert(COL_ADDED < COL_VALUES && COL_KEPT < COL_VALUES && COL_ADDED != COL_KEPT, "the orders overlap the values");
constexpr size_t RUN_ROW = 4 * sizeof(uint32_t);

// the four arrays of the sort area as CUB's double buffers
struct SortBufs {
  cub::DoubleBuffer<VKey> k;
  cub::DoubleBuffer<uint32_t> v;
};
uint64_t sort_rows(const VoxState* V) { return V->d_sort.size() / SORT_ROW; }
uint32_t* sort_col(const VoxState* V, uint32_t c) { return reinterpret_cast<uint32_t*>(V->d_sort + 4 * c * sort_rows(V)); }
float4* sort_stage(const VoxState* V) { return reinterpret_cast<float4*>(V->d_sort.data()); }   // a save's centroids
SortBufs sort_bufs(const VoxState* V) {
  const uint64_t rows = sort_rows(V);
  VKey* k = reinterpret_cast<VKey*>(sort_col(V, COL_KEYS));
  uint32_t* v = sort_col(V, COL_VALUES);
  return SortBufs{cub::DoubleBuffer<VKey>(k, k + rows), cub::DoubleBuffer<uint32_t>(v, v + rows)};
}

// the dense cloud: slot of global point p and its undistorted row
struct VmSlots {
  const float* ud[MALIO_MAX_LIDAR];
  float tag[MALIO_MAX_LIDAR];
  uint32_t first[MALIO_MAX_LIDAR + 1];
  int L;
};

__device__ __forceinline__ int slot_row(const VmSlots& c, uint32_t p, const float** row) {
  int l = 0;
  while (l + 1 < c.L && p >= c.first[l + 1]) ++l;
  *row = c.ud[l] + 5 * (size_t)(p - c.first[l]);
  return l;
}

// The rows a fold reads.  point(p) is row p as {x, y, z, tag} in the world frame.
// A scan's dense cloud, registered with the pass state; tag = the slot's
struct ScanRows {
  VmSlots c;
  PassConst pc;
  __device__ __forceinline__ float4 point(uint32_t p) const {
    const float* r;
    const int l = slot_row(c, p, &r);
    float w[3];
    body_to_world(pc, l, r[0], r[1], r[2], w);
    return make_float4(w[0], w[1], w[2], c.tag[l]);
  }
};
// Saved points {x, y, z, intensity} in device memory, as given.  They do not change during the fold, so they are read through
// the read-only path.
struct SeedRows {
  const float4* xyzi;
  __device__ __forceinline__ float4 point(uint32_t p) const { return __ldg(xyzi + p); }
};
// Stored scans (malio_world_voxel_rebuild): a chunk of whole scans of one store block, rows in (scan, slot, point) order as
// {x, y, z} in the LiDAR frame.  Row p belongs to the last scan whose first row is <= p (a binary search; an empty scan shares
// its first row with the next one and is never the last such scan) and is registered with that scan's PassConst through
// body_to_world: the bits of ScanRows for the same scan.  The scan table is in device memory.
struct StoreScan {
  PassConst pc;                          // the scan's state and its stored temporal compensation
  uint32_t first[MALIO_MAX_LIDAR + 1];   // its slots' first rows in the chunk; first[L] = the next scan's first row
  float tag[MALIO_MAX_LIDAR];
};
struct StoreRows {
  const float* xyz;                      // the chunk's first row
  const StoreScan* scan;                 // the chunk's scans in index order
  uint32_t n_scans;
  int L;
  __device__ __forceinline__ float4 point(uint32_t p) const {
    uint32_t lo = 0, hi = n_scans;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (scan[mid].first[0] <= p) lo = mid; else hi = mid;
    }
    const StoreScan& s = scan[lo];
    int l = 0;
    while (l + 1 < L && p >= s.first[l + 1]) ++l;
    const float* r = xyz + 3 * (size_t)p;
    float w[3];
    body_to_world(s.pc, l, r[0], r[1], r[2], w);
    return make_float4(w[0], w[1], w[2], s.tag[l]);
  }
};

__device__ __forceinline__ uint64_t vhash(const VKey& a) {
  uint64_t h = (uint64_t)(uint32_t)a.i * 0x9E3779B97F4A7C15ull ^ (uint64_t)(uint32_t)a.j * 0xC2B2AE3D27D4EB4Full ^
               (uint64_t)(uint32_t)a.k * 0x165667B19E3779F9ull;
  h ^= h >> 31; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 29;
  return h;
}
__device__ __forceinline__ bool same(const VKey& a, const VKey& b) { return a.k == b.k && a.j == b.j && a.i == b.i; }
// the entry of voxel k, or EMPTY when the hash does not hold it
__device__ __forceinline__ uint32_t hash_find(const uint32_t* hash, uint64_t mask, const VKey* ekey, const VKey& k) {
  for (uint64_t s = vhash(k) & mask;; s = (s + 1) & mask) {
    const uint32_t e = hash[s];
    if (e == EMPTY || same(ekey[e], k)) return e;
  }
}
// entry e (voxel k) into the first free slot of k's probe sequence
__device__ __forceinline__ void hash_insert(uint32_t* hash, uint64_t mask, const VKey& k, uint32_t e) {
  uint64_t slot = vhash(k) & mask;
  while (atomicCAS(hash + slot, EMPTY, e) != EMPTY) slot = (slot + 1) & mask;
}
__device__ __forceinline__ bool in_int(float f) { return f >= -2147483648.f && f < 2147483648.f; }

template <class Rows>
__global__ void __launch_bounds__(256) vm_key_kernel(Rows src, float il, uint32_t n, VKey* __restrict__ key,
                                                     uint32_t* __restrict__ val, uint32_t* __restrict__ fault) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n) return;
  const float4 w = src.point(p);
  const VKey none{SKIP_K, SKIP_K, SKIP_K};
  val[p] = p;
  if (!(isfinite(w.x) && isfinite(w.y) && isfinite(w.z))) { key[p] = none; return; }
  const float fx = floorf(w.x * il), fy = floorf(w.y * il), fz = floorf(w.z * il);
  if (!(in_int(fx) && in_int(fy) && in_int(fz))) { atomicOr(fault, 1u); key[p] = none; return; }
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
  const uint32_t e = hash_find(hash, mask, ekey, k);
  rent[r] = e == EMPTY ? RUN_NEW : e;
  is_new[r] = e == EMPTY ? 1u : 0u;
}

// one thread per run: the voxel's entry (a new one numbered in key order and entered into the hash), then its sums continued
// row by row.  Nothing is written once a row of the call was outside int (small[0], which a seed keeps over its chunks): the
// map stays as it was.
template <class Rows>
__global__ void __launch_bounds__(128) vm_fold_kernel(Rows src, const uint32_t* __restrict__ run,
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
    hash_insert(hash, mask, k, e);
    ekey[e] = k;
    s = make_float4(0.f, 0.f, 0.f, 0.f);
    cnt = 0;
  } else {
    s = esum[e];
    cnt = ecnt[e];
  }
  for (uint32_t q = q0; q < q1; ++q) {
    const float4 w = src.point(val[q]);
    s.x += w.x; s.y += w.y; s.z += w.z; s.w += w.w;
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
  hash_insert(hash, mask, ekey[e], e);
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
  out[r] = malio_voxrule::centroid(esum[e], ecnt[e]);
}

// ------------------------------------------------------------------ carving (malio_world_voxel_accumulate_carve)
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
  const float* row;
  const int l = slot_row(c, p, &row);
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
    const uint32_t e = hash_find(hash, mask, ekey, VKey{cz, cy, cx});
    if (e != EMPTY && *(volatile const uint32_t*)(stamp + e) != scan && atomicMax(stamp + e, scan) < scan) hm[e].y += 1u;
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

// the (hit, miss) of an entry and the keep rule, shared with malio_grid.cu
using malio_voxrule::dropped;
using malio_voxrule::evidence;

// (hit, miss) of the r-th voxel in key order -> out[r], r < n
__global__ void __launch_bounds__(256) vc_evidence_kernel(const uint32_t* __restrict__ order, uint32_t n, const uint2* __restrict__ hm,
                                                          uint2* __restrict__ out) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  out[r] = evidence(hm, order[r]);
}

// the keep rule on the r-th voxel in key order
__global__ void __launch_bounds__(256) vc_keep_kernel(const uint32_t* __restrict__ order, uint32_t n, const uint2* __restrict__ hm,
                                                      uint32_t min_miss, double ratio, uint32_t* __restrict__ keep) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  keep[r] = dropped(evidence(hm, order[r]), min_miss, ratio) ? 0u : 1u;
}

// the flagged entries in key order -> out[0 .. *count)
__global__ void __launch_bounds__(256) vc_compact_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ flag,
                                                         const uint32_t* __restrict__ pos, uint32_t n, uint32_t* __restrict__ out,
                                                         uint32_t* __restrict__ count) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  if (flag[r]) out[pos[r]] = order[r];
  if (r == n - 1) *count = pos[r] + flag[r];
}

// ------------------------------------------------------------------ seeding (malio_world_voxel_seed*) and the changes
// after the last chunk: the seeded entries [0, small[2]) start at (seed_hits, 0), stamp 0
__global__ void __launch_bounds__(256) vs_hits_kernel(const uint32_t* __restrict__ small, uint32_t n, uint32_t seed_hits,
                                                      uint2* __restrict__ hm, uint32_t* __restrict__ stamp) {
  const uint32_t e = blockIdx.x * 256u + threadIdx.x;
  if (small[0] || e >= n || e >= small[2]) return;
  hm[e] = make_uint2(seed_hits, 0u);
  stamp[e] = 0u;
}

// the r-th voxel in key order: removed[r] = seeded and dropped by the keep rule, added[r] = not seeded and kept
__global__ void __launch_bounds__(256) vs_change_kernel(const uint32_t* __restrict__ order, uint32_t n, const uint2* __restrict__ hm,
                                                        uint32_t min_miss, double ratio, uint32_t n_seeded,
                                                        uint32_t* __restrict__ removed, uint32_t* __restrict__ added) {
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  if (r >= n) return;
  const uint32_t e = order[r];
  const bool kept = !dropped(evidence(hm, e), min_miss, ratio);
  const bool seeded = e < n_seeded;
  removed[r] = (seeded && !kept) ? 1u : 0u;
  added[r] = (!seeded && kept) ? 1u : 0u;
}

// ------------------------------------------------------------------ rebuilding from the stored scans (malio_world_voxel_rebuild)
// a carved rebuild's scan: its 12-byte stored rows -> the 20-byte rows of an undistorted cloud (x, y, z; the other two words
// are not read), which ScanRows and the carve kernels take as they take a live scan's
__global__ void __launch_bounds__(256) vr_unpack_kernel(const float* __restrict__ xyz, uint32_t n, float* __restrict__ ud) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n) return;
  const float* r = xyz + 3 * (size_t)p;
  float* o = ud + 5 * (size_t)p;
  o[0] = r[0]; o[1] = r[1]; o[2] = r[2];
}

// CUB's calls on d_temp, reserved by grow_sort, grow_runs and enqueue_select_order.  The stable sort of n rows of b by key:
auto sort_call(SortBufs& b, uint64_t n, cudaStream_t st) {
  return [&b, n, st](void* t, size_t& c) { return cub::DeviceRadixSort::SortPairs(t, c, b.k, b.v, (int)n, VKeyDecomposer{}, st); };
}
// the fold's scans of n rows: the head flags into the run numbers (d_rent), the new flags into the new runs' ranks (d_head)
auto runs_call(VoxState* V, uint64_t n, cudaStream_t st) {
  return [=](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, V->d_head.data(), V->d_rent.data(), (int)n, st); };
}
auto new_call(VoxState* V, uint64_t n, cudaStream_t st) {
  return [=](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, V->d_new.data(), V->d_head.data(), (int)n, st); };
}
// a selection's exclusive scan of the flag column over the entries into COL_SCAN (its storage does not depend on the column)
auto select_call(VoxState* V, const uint32_t* flag, cudaStream_t st) {
  return [=](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, flag, sort_col(V, COL_SCAN), (int)V->n_vox, st); };
}

// the sort area for n rows and CUB's storage for their sort
int grow_sort(malio_handle* h, VoxState* V, DeviceState* D, uint64_t n) {
  if (n > sort_rows(V)) {
    if (int rc = V->d_sort.allocate(h, D->stream, (n + n / 8 + 1024) * SORT_ROW)) return rc;
  }
  SortBufs b = sort_bufs(V);
  return V->d_temp.reserve(h, D->stream, sort_call(b, n, D->stream));
}
// the run scratch for n rows
int grow_runs(malio_handle* h, VoxState* V, DeviceState* D, uint64_t n) {
  if (n > V->d_head.size()) {
    const uint64_t c = n + n / 8 + 1024;
    if (int rc = malio_buf::allocate_group(h, D->stream, {{V->d_head, c}, {V->d_run, c}, {V->d_rent, c}, {V->d_new, c}})) return rc;
  }
  return V->d_temp.reserve(h, D->stream, runs_call(V, n, D->stream), new_call(V, n, D->stream));
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

// the carving evidence of every entry the table holds room for, zero: allocated by the first carve, or by a seed with hits
int ensure_evidence(malio_handle* h, VoxState* V, DeviceState* D) {
  if (V->d_hm) return MALIO_OK;
  const size_t cap = V->d_ekey.size();
  if (int rc = malio_buf::allocate_group(h, D->stream, {{V->d_hm, cap}, {V->d_stamp, cap}})) return rc;
  CUDA_TRY(cudaMemsetAsync(V->d_hm, 0, cap * sizeof(uint2), D->stream));
  CUDA_TRY(cudaMemsetAsync(V->d_stamp, 0, cap * sizeof(uint32_t), D->stream));
  return MALIO_OK;
}

// enqueue the fold of rows [0, n) of src on the handle's stream, from vm_key_kernel to vm_fold_kernel (table, sort area and
// run scratch grown for them; small[0] is the call's fault flag, cleared by the caller).  Then d_rent holds each run's entry
// and d_head the new runs' ranks; the caller enqueues vm_count_kernel, which raises small[2] by the new entries.
template <class Rows>
int enqueue_fold(malio_handle* h, VoxState* V, DeviceState* D, const Rows& src, float il, uint32_t n) {
  cudaStream_t st = D->stream;
  const uint32_t g = (n + 255) / 256;
  const uint64_t mask = V->d_hash.size() - 1;
  SortBufs b = sort_bufs(V);
  vm_key_kernel<<<g, 256, 0, st>>>(src, il, n, b.k.Current(), b.v.Current(), V->d_small);
  if (int rc = V->d_temp.run(h, sort_call(b, n, st))) return rc;
  const VKey* key = b.k.Current();
  const uint32_t* val = b.v.Current();
  vm_head_kernel<<<g, 256, 0, st>>>(key, n, V->d_head);
  if (int rc = V->d_temp.run(h, runs_call(V, n, st))) return rc;
  vm_run_kernel<<<g, 256, 0, st>>>(V->d_head, V->d_rent, n, V->d_run, V->d_small);
  vm_lookup_kernel<<<g, 256, 0, st>>>(V->d_run, key, n, V->d_small, V->d_hash, mask, V->d_ekey, V->d_rent, V->d_new);
  if (int rc = V->d_temp.run(h, new_call(V, n, st))) return rc;
  vm_fold_kernel<<<(n + 127) / 128, 128, 0, st>>>(src, V->d_run, key, val, n, V->d_small, V->d_rent, V->d_head, V->d_hash, mask,
                                                 V->d_ekey, V->d_esum, V->d_ecnt);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 6;   // the radix sort counted as one
  return MALIO_OK;
}

// enqueue the sort of the entries by key on the handle's stream (sort area already grown): *order = the entries in key order,
// the values half CUB left current (the other values half and the key halves are free once it is sorted)
int enqueue_order(malio_handle* h, VoxState* V, DeviceState* D, SortBufs& b) {
  cudaStream_t st = D->stream;
  const uint32_t n = (uint32_t)V->n_vox;
  vm_iota_kernel<<<(n + 255) / 256, 256, 0, st>>>(V->d_ekey, n, b.k.Current(), b.v.Current());
  if (int rc = V->d_temp.run(h, sort_call(b, n, st))) return rc;
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

// enqueue the centroids of the entries order[0 .. min(n, cap)) into out on the handle's stream, one thread per order row
int enqueue_centroids(malio_handle* h, VoxState* V, DeviceState* D, const uint32_t* order, uint32_t n, float4* out, uint32_t cap) {
  vm_centroid_kernel<<<(n + 255) / 256, 256, 0, D->stream>>>(order, n, V->d_esum, V->d_ecnt, out, cap);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

// enqueue the centroids in key order into out[0 .. min(n_vox, cap)) on the handle's stream (sort area already grown).  out may
// be the sort area itself (sort_stage): the keys are dead once sorted, the order is read from the values.
int enqueue_sorted(malio_handle* h, VoxState* V, DeviceState* D, float4* out, uint64_t cap) {
  const uint32_t n = (uint32_t)V->n_vox;
  SortBufs b = sort_bufs(V);
  if (int rc = enqueue_order(h, V, D, b)) return rc;
  return enqueue_centroids(h, V, D, b.v.Current(), n, out, cap < n ? (uint32_t)cap : n);
}

// A selection of the entries in key order (sort area grown for the entries): enqueue_select_order, one kernel that flags
// every entry, then enqueue_select per flag column.
int enqueue_select_order(malio_handle* h, VoxState* V, DeviceState* D, SortBufs& b) {
  if (int rc = V->d_temp.reserve(h, D->stream, select_call(V, sort_col(V, COL_FLAGS), D->stream))) return rc;
  b = sort_bufs(V);
  return enqueue_order(h, V, D, b);
}
// the exclusive scan of flag into COL_SCAN, then the flagged entries of order compacted into column `col`, their count into
// small[word]
int enqueue_select(malio_handle* h, VoxState* V, DeviceState* D, const uint32_t* order, const uint32_t* flag, uint32_t col, int word) {
  const uint32_t n = (uint32_t)V->n_vox;
  if (int rc = V->d_temp.run(h, select_call(V, flag, D->stream))) return rc;
  vc_compact_kernel<<<(n + 255) / 256, 256, 0, D->stream>>>(order, flag, sort_col(V, COL_SCAN), n, sort_col(V, col), V->d_small + word);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

// the entries the keep rule does not drop into COL_KEPT; waits for their count (*n_kept)
int enqueue_kept(malio_handle* h, VoxState* V, DeviceState* D, const malio_carve_keep* keep, uint64_t* n_kept) {
  cudaStream_t st = D->stream;
  const uint32_t n = (uint32_t)V->n_vox;
  SortBufs b;
  if (int rc = enqueue_select_order(h, V, D, b)) return rc;
  vc_keep_kernel<<<(n + 255) / 256, 256, 0, st>>>(b.v.Current(), n, V->d_hm, keep->min_miss, (double)keep->max_miss_per_hit,
                                                  b.v.Alternate());
  D->ctr.kernel_launches += 1;
  if (int rc = enqueue_select(h, V, D, b.v.Current(), b.v.Alternate(), COL_KEPT, 3)) return rc;
  CUDA_TRY(cudaMemcpyAsync(V->h_small + 3, V->d_small + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // the kept count sizes the caller's output and the file
  *n_kept = V->h_small[3];
  return MALIO_OK;
}

// the changes against the seed: the removed entries into COL_KEPT, the added ones into COL_ADDED; waits for the two counts
int enqueue_changes(malio_handle* h, VoxState* V, DeviceState* D, const malio_carve_keep* keep, uint64_t* n_removed, uint64_t* n_added) {
  cudaStream_t st = D->stream;
  const uint32_t n = (uint32_t)V->n_vox;
  SortBufs b;
  if (int rc = enqueue_select_order(h, V, D, b)) return rc;
  uint32_t* flag_a = sort_col(V, COL_FLAGS);
  vs_change_kernel<<<(n + 255) / 256, 256, 0, st>>>(b.v.Current(), n, V->d_hm, keep->min_miss, (double)keep->max_miss_per_hit,
                                                    (uint32_t)V->n_seeded, b.v.Alternate(), flag_a);
  D->ctr.kernel_launches += 1;
  if (int rc = enqueue_select(h, V, D, b.v.Current(), b.v.Alternate(), COL_KEPT, 3)) return rc;
  if (int rc = enqueue_select(h, V, D, b.v.Current(), flag_a, COL_ADDED, 5)) return rc;
  CUDA_TRY(cudaMemcpyAsync(V->h_small + 3, V->d_small + 3, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // the counts size the caller's outputs and the files
  *n_removed = V->h_small[3];
  *n_added = V->h_small[5];
  return MALIO_OK;
}

// after a save: the entry-sized sort area and CUB's storage go back once the stream is drained.  Between saves the map holds
// its entries, its hash and the scan-sized scratch only (the next accumulate regrows the sort area for its scan).
int release_scratch(malio_handle* h, VoxState* V, DeviceState* D) {
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  V->d_sort.release();
  V->d_temp.release();
  return MALIO_OK;
}

constexpr const char* CENTROID_ROWS = "the centroids are stored as float4";   // check_device_ptr's reason for 16-byte rows

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

// the argument refusals of an accumulate (carve NULL) or a carved accumulate, in their order: carve arguments, leaf, range cap
int check_fold_args(malio_handle* h, const VoxState* V, float leaf, const malio_carve_args* carve) {
  if (carve && !(std::isfinite(carve->max_range) && carve->max_range > 0.f && std::isfinite(carve->end_margin) && carve->end_margin >= 0.f)) {
    h->err = "world voxel carve: max_range must be finite and > 0, end_margin finite and >= 0";
    return MALIO_ERR_INVALID_ARG;
  }
  if (int rc = check_leaf(h, V, leaf)) return rc;
  if (carve && (double)carve->max_range * (double)(1.0f / leaf) > MALIO_CARVE_MAX_RANGE_CELLS) {
    h->err = "world voxel carve: max_range / leaf above MALIO_CARVE_MAX_RANGE_CELLS; the map is unchanged";
    return MALIO_ERR_CAPACITY;
  }
  return MALIO_OK;
}

// enqueue the fold of one scan's nn > 0 dense rows on the handle's stream (table, sort area, run scratch and, with carve, the
// evidence already grown; small[0] is the fault flag the caller cleared): with carve, the origins' check first and the
// scan's hits and passes (carve scan number `scan`) after the fold
int enqueue_scan(malio_handle* h, VoxState* V, DeviceState* D, const ScanRows& src, float il, uint32_t nn, const malio_carve_args* carve,
                 uint32_t scan) {
  cudaStream_t st = D->stream;
  const uint32_t g = (nn + 255) / 256;
  if (carve) vc_origin_kernel<<<1, 32, 0, st>>>(src.c, src.pc, il, V->d_small);
  if (int rc = enqueue_fold(h, V, D, src, il, nn)) return rc;
  if (carve) vc_hit_kernel<<<g, 256, 0, st>>>(V->d_small, V->d_rent, V->d_head, nn, V->d_hm, V->d_stamp, scan);
  vm_count_kernel<<<1, 1, 0, st>>>(V->d_head, V->d_new, V->d_small);
  if (carve)
    vc_carve_kernel<<<g, 256, 0, st>>>(src.c, src.pc, il, nn, (double)carve->max_range, (double)carve->end_margin, V->d_small,
                                       V->d_hash, V->d_hash.size() - 1, V->d_ekey, V->d_hm, V->d_stamp, scan);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += carve ? 4 : 1;
  return MALIO_OK;
}

// the table holds room for `need` entries with the hash at most half full (grow_table would change nothing)
bool table_fits(const VoxState* V, uint64_t need) {
  return V->d_hash && need <= V->d_ekey.size() && 2 * need <= V->d_hash.size();
}

}  // namespace

namespace malio_vox {

// carve == NULL: malio_world_voxel_accumulate; otherwise the same fold, then the scan's hits and passes (checked first)
int accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf, const malio_carve_args* carve,
               uint64_t* n_voxels) {
  VoxState* V;
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  if (int rc = check_fold_args(h, V, leaf, carve)) return rc;
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
    if (carve) { if (int rc = ensure_evidence(h, V, D)) return rc; }   // the first carve: every entry so far at hit = miss = 0
    cudaStream_t st = D->stream;
    const ScanRows src{c, make_pass_const(h, D, s)};
    CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 2 * sizeof(uint32_t), st));   // fault flag, run count
    if (int rc = enqueue_scan(h, V, D, src, 1.0f / leaf, (uint32_t)n, carve, scan)) return rc;
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
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  const uint64_t n = V->n_vox, k = n < cap ? n : cap;
  if (out && k) {
    if (int rc = check_device_ptr(h, D, out, "malio_world_voxel_download_device out", 16, CENTROID_ROWS)) return rc;
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
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  const uint64_t n = V->n_vox, k = n < cap ? n : cap;
  if (out && k) {
    if (int rc = check_device_ptr(h, D, out, "malio_world_voxel_evidence_device out", 8, "the pairs are stored as uint2")) return rc;
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
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  if (int rc = check_keep(h, keep)) return rc;
  if (out && cap && V->n_vox) {
    if (int rc = check_device_ptr(h, D, out, "malio_world_voxel_download_kept_device out", 16, CENTROID_ROWS)) return rc;
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
  if (int rc = enqueue_centroids(h, V, D, sort_col(V, COL_KEPT), (uint32_t)k, reinterpret_cast<float4*>(out), (uint32_t)k)) return rc;
  return caller_leave(h, D, caller);
}

// keep == NULL: every voxel (malio_world_voxel_save_pcd); otherwise the voxels the rule keeps (malio_world_voxel_save_pcd_kept)
int save_pcd(malio_handle* h, const char* path, const malio_carve_keep* keep, int clear) {
  VoxState* V;
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  if (keep) { if (int rc = check_keep(h, keep)) return rc; }
  if (V->n_vox == 0) { h->err = "world voxel save: the voxel map is empty (nothing is written)"; return MALIO_ERR_STATE; }
  uint64_t n = V->n_vox;
  if (int rc = grow_sort(h, V, D, n)) return rc;
  float4* stage = sort_stage(V);
  if (keep) {
    if (int rc = enqueue_kept(h, V, D, keep, &n)) return rc;
    if (n == 0) {
      if (int rc = release_scratch(h, V, D)) return rc;
      h->err = "world voxel save: the keep rule drops every voxel (nothing is written)";
      return MALIO_ERR_STATE;
    }
    if (int rc = enqueue_centroids(h, V, D, sort_col(V, COL_KEPT), (uint32_t)n, stage, (uint32_t)n)) return rc;
  } else if (int rc = enqueue_sorted(h, V, D, stage, n)) {
    return rc;
  }
  const int rc = write_pcd_from_device(h, D, path, stage, n, V->h_bounce);
  if (int e = release_scratch(h, V, D)) return e;
  if (rc == MALIO_OK && clear) {
    if (int c = clear_map(h, V, D)) return c;
  }
  return rc;
}

// malio_world_voxel_seed (on_device false: xyzi in host memory, staged through the pinned bounce buffer into a chunk-sized
// device buffer) and malio_world_voxel_seed_device (xyzi read in place, ordered on `caller`).  The points are folded chunk by
// chunk in input order, each chunk through enqueue_fold with SeedRows; the table is sized for n points before the first chunk,
// so the chunks are enqueued back to back and the call waits once.
int seed(malio_handle* h, const float* xyzi, uint64_t n, float leaf, uint32_t seed_hits, bool on_device, cudaStream_t caller,
         uint64_t* n_voxels) {
  VoxState* V;
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  if (!(leaf > 0.f) || !std::isfinite(leaf)) { h->err = "world voxel seed: leaf must be a finite size > 0"; return MALIO_ERR_INVALID_ARG; }
  if (V->n_vox || V->leaf_set) {
    h->err = "world voxel seed: the voxel map is not empty (seed a new map or one after a clearing save)";
    return MALIO_ERR_STATE;
  }
  if (on_device) {
    if (int rc = check_device_ptr(h, D, xyzi, "malio_world_voxel_seed_device xyzi", 16, "the rows are read as float4")) return rc;
  }
  const uint64_t chunk = n < MALIO_SEED_CHUNK ? n : MALIO_SEED_CHUNK;
  if (int rc = grow_table(h, V, D, n)) return rc;
  if (int rc = grow_sort(h, V, D, chunk)) return rc;
  if (int rc = grow_runs(h, V, D, chunk)) return rc;
  const bool had_hm = (bool)V->d_hm;
  if (seed_hits) { if (int rc = ensure_evidence(h, V, D)) return rc; }   // zero beyond the seed, as the first carve leaves them
  DeviceBuffer<float4> stage;
  if (!on_device) {
    if (int rc = stage.allocate(h, D->stream, chunk)) return rc;
    if (!V->h_bounce) { if (int rc = V->h_bounce.allocate(h, malio_pcd::CHUNK)) return rc; }
  } else if (int rc = caller_enter(h, D, caller)) {
    return rc;
  }
  cudaStream_t st = D->stream;
  CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 2 * sizeof(uint32_t), st));   // fault flag (kept over the chunks), run count
  const float4* rows = reinterpret_cast<const float4*>(xyzi);
  for (uint64_t first = 0; first < n; first += chunk) {
    const uint32_t m = (uint32_t)(n - first < chunk ? n - first : chunk);
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
    if (int rc = enqueue_fold(h, V, D, SeedRows{src}, 1.0f / leaf, m)) return rc;
    vm_count_kernel<<<1, 1, 0, st>>>(V->d_head, V->d_new, V->d_small);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 1;
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

// malio_world_voxel_rebuild (malio_b200.h): the stored scans [first, first + count) through the accumulate pipeline.
//   1. a StoreScan per scan (its PassConst from the given or stored state and its stored compensation), grouped into chunks:
//      plain, consecutive scans of one block up to MALIO_SEED_CHUNK rows (a larger scan alone); carved, one scan per chunk
//   2. the check: vm_key_kernel over every chunk (and vc_origin_kernel per carved scan) raises small[0] for a row or an origin
//      outside int; every kernel after it then writes nothing, so a refused rebuild leaves the map as it was
//   3. per chunk, enqueued back to back: plain, one enqueue_fold with StoreRows and vm_count_kernel; carved, the scan's rows
//      unpacked to 20-byte rows and accumulate's own sequence (enqueue_scan) with carve scan number carve_scan + 1 + i
//   The table grows per chunk for an upper bound of the entries (the rows enqueued so far); only when that bound does not fit
//   does the call wait for the exact count first.  One wait at the end for the verdict and the count.
int rebuild(malio_handle* h, uint64_t first, uint64_t count, const malio_pass_state* states, float leaf, const malio_carve_args* carve,
            uint64_t* n_voxels) {
  VoxState* V;
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  const uint64_t stored = malio_store::count(h);
  if (first > stored || count > stored - first) {
    h->err = "world voxel rebuild: scans [" + std::to_string(first) + ", " + std::to_string(first + count) + ") beyond the store (" +
             std::to_string(stored) + " scans)";
    return MALIO_ERR_INVALID_ARG;
  }
  if (count == 0) {
    if (n_voxels) *n_voxels = V->n_vox;
    return MALIO_OK;
  }
  if (int rc = check_fold_args(h, V, leaf, carve)) return rc;
  const int L = h->cfg.params.n_lidar;
  struct Chunk { uint64_t s0, s1; const float* xyz; uint32_t block; uint64_t rows; };
  std::vector<StoreScan> scans(count);
  std::vector<Chunk> chunks;
  uint64_t max_rows = 0;
  for (uint64_t i = 0; i < count; ++i) {
    const malio_store::View v = malio_store::view(h, first + i);
    malio_rigid tc[MALIO_MAX_LIDAR];
    tc[0] = D->tcomp[0];   // (not read: slot 0 has no compensation)
    for (int l = 1; l < MALIO_MAX_LIDAR; ++l) tc[l] = v.rec->temporal_comp[l - 1];
    StoreScan& sc = scans[i];
    sc.pc = make_pass_const(h, D, states ? states + i : &v.rec->state, tc);
    Chunk* c = chunks.empty() ? nullptr : &chunks.back();
    const bool joins = c && !carve &&
                       (v.rows == 0 || c->rows == 0 ||
                        (v.block == c->block && v.xyz == c->xyz + 3 * c->rows && c->rows + v.rows <= MALIO_SEED_CHUNK));
    if (!joins) { chunks.push_back(Chunk{i, i, v.xyz, v.block, 0}); c = &chunks.back(); }
    if (c->rows == 0 && v.rows) { c->xyz = v.xyz; c->block = v.block; }
    uint64_t at = c->rows;
    for (int l = 0; l < L; ++l) { sc.first[l] = (uint32_t)at; sc.tag[l] = v.rec->slot_tag[l]; at += v.rec->n_points[l]; }
    for (int l = L; l <= MALIO_MAX_LIDAR; ++l) sc.first[l] = (uint32_t)at;
    for (int l = L; l < MALIO_MAX_LIDAR; ++l) sc.tag[l] = 0.f;
    c->s1 = i + 1;
    c->rows = at;
    if (at > max_rows) max_rows = at;
  }
  cudaStream_t st = D->stream;
  const float il = 1.0f / leaf;
  DeviceBuffer<StoreScan> d_scans;   // the chunks' scan tables; freed after the call's wait
  DeviceBuffer<float> d_ud;          // a carved scan's unpacked rows
  if (int rc = d_scans.allocate(h, st, count)) return rc;
  if (carve && max_rows) { if (int rc = d_ud.allocate(h, st, 5 * max_rows)) return rc; }
  if (max_rows) {
    if (int rc = grow_sort(h, V, D, max_rows)) return rc;
    if (int rc = grow_runs(h, V, D, max_rows)) return rc;
  }
  CUDA_TRY(cudaMemcpyAsync(d_scans, scans.data(), count * sizeof(StoreScan), cudaMemcpyHostToDevice, st));
  D->ctr.h2d_bytes += count * sizeof(StoreScan);
  CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 2 * sizeof(uint32_t), st));   // fault flag (kept over the whole call), run count
  auto rows_of = [&](const Chunk& c) { return StoreRows{c.xyz, d_scans + c.s0, (uint32_t)(c.s1 - c.s0), L}; };
  for (const Chunk& c : chunks) {   // the check: nothing is folded once a row or an origin is outside int
    if (c.rows) {
      SortBufs b = sort_bufs(V);
      const uint32_t m = (uint32_t)c.rows;
      vm_key_kernel<<<(m + 255) / 256, 256, 0, st>>>(rows_of(c), il, m, b.k.Current(), b.v.Current(), V->d_small);
      D->ctr.kernel_launches += 1;
    }
    if (carve && c.rows) {
      VmSlots o{};
      o.L = L;
      for (int l = 0; l <= L; ++l) o.first[l] = scans[c.s0].first[l];
      vc_origin_kernel<<<1, 32, 0, st>>>(o, scans[c.s0].pc, il, V->d_small);
      D->ctr.kernel_launches += 1;
    }
  }
  CUDA_TRY(cudaGetLastError());
  uint64_t bound = V->n_vox;   // at least the entries after the chunks enqueued so far
  for (const Chunk& c : chunks) {
    if (c.rows == 0) continue;
    const uint32_t m = (uint32_t)c.rows;
    if (!table_fits(V, bound + m)) {   // the exact count first, then the table for it
      CUDA_TRY(cudaMemcpyAsync(V->h_small, V->d_small, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      if (V->h_small[0]) break;   // refused: the verdict below
      V->n_vox = bound = V->h_small[2];
      if (int rc = grow_table(h, V, D, bound + m)) return rc;
    }
    if (carve) {
      if (int rc = ensure_evidence(h, V, D)) return rc;   // the first carve: every entry so far at hit = miss = 0
      vr_unpack_kernel<<<(m + 255) / 256, 256, 0, st>>>(c.xyz, m, d_ud);
      D->ctr.kernel_launches += 1;
      const StoreScan& sc = scans[c.s0];
      VmSlots u{};
      u.L = L;
      for (int l = 0; l < L; ++l) { u.ud[l] = d_ud + 5 * (size_t)sc.first[l]; u.tag[l] = sc.tag[l]; u.first[l] = sc.first[l]; }
      u.first[L] = sc.first[L];
      if (int rc = enqueue_scan(h, V, D, ScanRows{u, sc.pc}, il, m, carve, V->carve_scan + 1 + (uint32_t)c.s0)) return rc;
    } else {
      if (int rc = enqueue_fold(h, V, D, rows_of(c), il, m)) return rc;
      vm_count_kernel<<<1, 1, 0, st>>>(V->d_head, V->d_new, V->d_small);
      CUDA_TRY(cudaGetLastError());
      D->ctr.kernel_launches += 1;
    }
    bound += m;
  }
  CUDA_TRY(cudaMemcpyAsync(V->h_small, V->d_small, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // the call's one wait: the fault flag and the entry count
  if (V->h_small[0]) {
    h->err = carve ? "world voxel rebuild: leaf size too small for a stored point's or a ray origin's coordinates under its scan's state (voxel index outside int); the map is unchanged"
                   : "world voxel rebuild: leaf size too small for a stored point's coordinates under its scan's state (voxel index outside int); the map is unchanged";
    return MALIO_ERR_CAPACITY;
  }
  V->n_vox = V->h_small[2];
  if (carve) V->carve_scan += (uint32_t)count;
  V->leaf = leaf;
  V->leaf_set = true;
  if (n_voxels) *n_voxels = V->n_vox;
  return MALIO_OK;
}

// removed / added centroids in the order of download_device, with download_kept_device's size protocol and contract
int changes_device(malio_handle* h, const malio_carve_keep* keep, float* d_removed, uint64_t cap_removed, uint64_t* n_removed,
                   float* d_added, uint64_t cap_added, uint64_t* n_added, cudaStream_t caller) {
  VoxState* V;
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  if (int rc = check_keep(h, keep)) return rc;
  if (V->n_vox) {
    if (d_removed && cap_removed) {
      if (int rc = check_device_ptr(h, D, d_removed, "malio_world_voxel_changes_device removed", 16, CENTROID_ROWS)) return rc;
    }
    if (d_added && cap_added) {
      if (int rc = check_device_ptr(h, D, d_added, "malio_world_voxel_changes_device added", 16, CENTROID_ROWS)) return rc;
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
  if (kr) {
    if (int rc = enqueue_centroids(h, V, D, sort_col(V, COL_KEPT), (uint32_t)kr, reinterpret_cast<float4*>(d_removed), (uint32_t)kr)) return rc;
  }
  if (ka) {
    if (int rc = enqueue_centroids(h, V, D, sort_col(V, COL_ADDED), (uint32_t)ka, reinterpret_cast<float4*>(d_added), (uint32_t)ka)) return rc;
  }
  return caller_leave(h, D, caller);
}

// each set through save_pcd's writer (a NULL path or an empty set writes no file); the map is not cleared
int save_changes_pcd(malio_handle* h, const malio_carve_keep* keep, const char* removed_path, const char* added_path, uint64_t* n_removed,
                     uint64_t* n_added) {
  VoxState* V;
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  if (int rc = check_keep(h, keep)) return rc;
  if (V->n_vox == 0) { h->err = "world voxel save: the voxel map is empty (nothing is written)"; return MALIO_ERR_STATE; }
  if (int rc = grow_sort(h, V, D, V->n_vox)) return rc;
  uint64_t nr = 0, na = 0;
  if (int rc = enqueue_changes(h, V, D, keep, &nr, &na)) return rc;
  if (n_removed) *n_removed = nr;
  if (n_added) *n_added = na;
  float4* stage = sort_stage(V);
  int rc = MALIO_OK;
  const struct { const char* path; uint32_t col; uint64_t cnt; } sets[2] = {{removed_path, COL_KEPT, nr}, {added_path, COL_ADDED, na}};
  for (const auto& set : sets) {
    if (rc != MALIO_OK || !set.path || set.cnt == 0) continue;
    if (int e = enqueue_centroids(h, V, D, sort_col(V, set.col), (uint32_t)set.cnt, stage, (uint32_t)set.cnt)) return e;
    rc = write_pcd_from_device(h, D, set.path, stage, set.cnt, V->h_bounce);
  }
  if (int e = release_scratch(h, V, D)) return e;
  return rc;
}

int entries(const malio_handle* h, Entries* e) {
  const VoxState* V = h->voxmap.get();
  if (!V || V->n_vox == 0) return MALIO_ERR_STATE;
  *e = Entries{reinterpret_cast<const float*>(V->d_esum.data()), V->d_ecnt.data(), reinterpret_cast<const uint32_t*>(V->d_hm.data()), V->n_vox};
  return MALIO_OK;
}

int info(malio_handle* h, uint64_t* n_voxels, uint64_t* capacity, uint64_t* device_bytes) {
  VoxState* V;
  DeviceState* D;
  if (int rc = acquire(h, h->voxmap, V, D)) return rc;
  if (n_voxels) *n_voxels = V->n_vox;
  if (capacity) *capacity = V->d_ekey.size();
  if (device_bytes)
    *device_bytes = V->d_ekey.size() * (sizeof(VKey) + sizeof(float4) + sizeof(uint32_t)) + V->d_hash.size() * sizeof(uint32_t) +
                    V->d_sort.size() + V->d_head.size() * RUN_ROW + V->d_temp.bytes() +
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
extern "C" int malio_world_voxel_rebuild(malio_handle* h, uint64_t first, uint64_t count, const malio_pass_state* states, float leaf,
                                         const malio_carve_args* carve, uint64_t* n_voxels) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::rebuild(h, first, count, states, leaf, carve, n_voxels);
}
