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
  VKey* d_ekey = nullptr; float4* d_esum = nullptr; uint32_t* d_ecnt = nullptr; uint64_t cap_e = 0;   // entries
  uint32_t* d_hash = nullptr; uint64_t cap_h = 0;                                                    // power of two
  // sort area, cap_s rows of 32 B (one allocation): keys | alternate keys (12 B each) | values | alternate values (4 B each),
  // sized for the points of a scan or, on download and save, for the entries.  A save writes the sorted centroids (16 B a row)
  // over the two key halves and then releases the area; a download keeps it until the next save.
  char* d_sort = nullptr; uint64_t cap_s = 0;
  // run scratch, cap_p rows of 16 B, sized for the points of a scan only
  uint32_t *d_head = nullptr, *d_run = nullptr, *d_rent = nullptr, *d_new = nullptr;
  uint64_t cap_p = 0;
  char* d_temp = nullptr; size_t cap_temp = 0;   // CUB's temporary storage (sort histograms, scan carries)
  uint32_t* d_small = nullptr;               // [0] fault flag, [1] run count, [2] entries in use
  uint32_t* h_small = nullptr;               // pinned mirror of d_small
  float4* h_bounce = nullptr;                // pinned, malio_pcd::CHUNK points
};
constexpr size_t SORT_ROW = 2 * sizeof(VKey) + 2 * sizeof(uint32_t);
constexpr size_t RUN_ROW = 4 * sizeof(uint32_t);

// the four arrays of the sort area as CUB's double buffers
struct SortBufs {
  cub::DoubleBuffer<VKey> k;
  cub::DoubleBuffer<uint32_t> v;
};
SortBufs sort_bufs(const VoxState* V) {
  VKey* k = reinterpret_cast<VKey*>(V->d_sort);
  uint32_t* v = reinterpret_cast<uint32_t*>(V->d_sort + 2 * sizeof(VKey) * V->cap_s);
  return SortBufs{cub::DoubleBuffer<VKey>(k, k + V->cap_s), cub::DoubleBuffer<uint32_t>(v, v + V->cap_s)};
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

int get_state(malio_handle* h, VoxState*& V) {
  V = (VoxState*)h->voxmap;
  if (V) return MALIO_OK;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  V = new VoxState;
  h->voxmap = V;
  CUDA_TRY(cudaMalloc((void**)&V->d_small, 4 * sizeof(uint32_t)));
  CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 4 * sizeof(uint32_t), D->stream));
  CUDA_TRY(cudaHostAlloc((void**)&V->h_small, 4 * sizeof(uint32_t), cudaHostAllocDefault));
  return MALIO_OK;
}

// CUB's temporary storage for at least t bytes, and the sort area for n rows
int grow_temp(malio_handle* h, VoxState* V, DeviceState* D, size_t t) {
  if (t <= V->cap_temp) return MALIO_OK;
  t += t / 8 + 4096;
  V->cap_temp = 0;
  if (int rc = ensure(h, V->d_temp, t)) return rc;
  V->cap_temp = t;
  return MALIO_OK;
}
int grow_sort(malio_handle* h, VoxState* V, DeviceState* D, uint64_t n) {
  if (n > V->cap_s) {
    const uint64_t c = n + n / 8 + 1024;
    V->cap_s = 0;
    if (int rc = ensure(h, V->d_sort, c * SORT_ROW)) return rc;
    V->cap_s = c;
  }
  SortBufs b = sort_bufs(V);
  size_t t = 0;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t, b.k, b.v, (int)n, VKeyDecomposer{}, D->stream));
  return grow_temp(h, V, D, t);
}
// the run scratch for the n points of a scan
int grow_runs(malio_handle* h, VoxState* V, DeviceState* D, uint64_t n) {
  if (n > V->cap_p) {
    const uint64_t c = n + n / 8 + 1024;
    V->cap_p = 0;
    uint32_t** u[] = {&V->d_head, &V->d_run, &V->d_rent, &V->d_new};
    for (uint32_t** p : u) if (int rc = ensure(h, *p, c)) return rc;
    V->cap_p = c;
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
  uint64_t hc = V->cap_h ? V->cap_h : 2 * VOX_MIN_ENTRIES;
  while (hc < 2 * need) hc *= 2;
  if (need <= V->cap_e && hc == V->cap_h) return MALIO_OK;
  if (need > 0x7FFFFFFFull) { h->err = "world voxel map: more than 2^31 - 1 voxels"; return MALIO_ERR_CAPACITY; }
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  cudaStream_t st = D->stream;
  if (need > V->cap_e) {
    uint64_t c = V->cap_e * 2;
    if (c < need) c = need;
    if (c < VOX_MIN_ENTRIES) c = VOX_MIN_ENTRIES;
    VKey* k = nullptr; float4* s = nullptr; uint32_t* n = nullptr;
    cudaError_t e = cudaMalloc((void**)&k, c * sizeof(VKey));
    if (e == cudaSuccess) e = cudaMalloc((void**)&s, c * sizeof(float4));
    if (e == cudaSuccess) e = cudaMalloc((void**)&n, c * sizeof(uint32_t));
    if (e == cudaSuccess && V->n_vox) {
      e = cudaMemcpyAsync(k, V->d_ekey, V->n_vox * sizeof(VKey), cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(s, V->d_esum, V->n_vox * sizeof(float4), cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(n, V->d_ecnt, V->n_vox * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e != cudaSuccess) {
      cudaGetLastError();
      if (k) cudaFree(k);
      if (s) cudaFree(s);
      if (n) cudaFree(n);
      h->err = std::string("world voxel map: cannot grow to ") + std::to_string(c) + " voxels: " + cudaGetErrorString(e);
      return MALIO_ERR_CUDA;
    }
    if (V->d_ekey) cudaFree(V->d_ekey);
    if (V->d_esum) cudaFree(V->d_esum);
    if (V->d_ecnt) cudaFree(V->d_ecnt);
    V->d_ekey = k; V->d_esum = s; V->d_ecnt = n; V->cap_e = c;
  }
  if (hc != V->cap_h) {
    uint32_t* hp = nullptr;
    const cudaError_t e = cudaMalloc((void**)&hp, hc * sizeof(uint32_t));
    if (e != cudaSuccess) {
      cudaGetLastError();
      h->err = std::string("world voxel map: cannot grow the hash to ") + std::to_string(hc) + " slots: " + cudaGetErrorString(e);
      return MALIO_ERR_CUDA;
    }
    if (V->d_hash) cudaFree(V->d_hash);
    V->d_hash = hp;
    V->cap_h = hc;
    CUDA_TRY(cudaMemsetAsync(V->d_hash, 0xFF, hc * sizeof(uint32_t), st));
    if (V->n_vox) {
      vm_rehash_kernel<<<(uint32_t)((V->n_vox + 255) / 256), 256, 0, st>>>(V->d_ekey, (uint32_t)V->n_vox, V->d_hash, hc - 1);
      D->ctr.kernel_launches += 1;
    }
    CUDA_TRY(cudaGetLastError());
  }
  return MALIO_OK;
}

// enqueue the centroids in key order into out[0 .. min(n_vox, cap)) on the handle's stream (sort area already grown).  out may
// be the sort area itself (its two key halves, 24 B a row): the keys are dead once sorted, the order is read from the values.
int enqueue_sorted(malio_handle* h, VoxState* V, DeviceState* D, float4* out, uint64_t cap) {
  cudaStream_t st = D->stream;
  const uint32_t n = (uint32_t)V->n_vox;
  SortBufs b = sort_bufs(V);
  vm_iota_kernel<<<(n + 255) / 256, 256, 0, st>>>(V->d_ekey, n, b.k.Current(), b.v.Current());
  size_t t = V->cap_temp;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(V->d_temp, t, b.k, b.v, (int)n, VKeyDecomposer{}, st));
  vm_centroid_kernel<<<(n + 255) / 256, 256, 0, st>>>(b.v.Current(), n, V->d_esum, V->d_ecnt, out, cap < n ? (uint32_t)cap : n);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 2;
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
  VoxState* V = (VoxState*)h->voxmap;
  if (!V) return;
  void* p[] = {V->d_ekey, V->d_esum, V->d_ecnt, V->d_hash, V->d_sort, V->d_head, V->d_run, V->d_rent, V->d_new, V->d_temp,
               V->d_small};
  for (void* q : p) if (q) cudaFree(q);
  if (V->h_small) cudaFreeHost(V->h_small);
  if (V->h_bounce) cudaFreeHost(V->h_bounce);
  delete V;
  h->voxmap = nullptr;
}

int accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf, uint64_t* n_voxels) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (int rc = check_leaf(h, V, leaf)) return rc;
  VmSlots c{};
  uint32_t m[MALIO_MAX_LIDAR] = {0, 0, 0};
  if (int rc = malio_pre::world_dense_source(h, c.ud, m)) return rc;
  c.L = h->cfg.params.n_lidar;
  uint64_t n = 0;
  for (int l = 0; l < c.L; ++l) { c.tag[l] = slot_tag[l]; c.first[l] = (uint32_t)n; n += m[l]; }
  c.first[c.L] = (uint32_t)n;
  if (n > 0x7FFFFFFFull) { h->err = "world voxel map: more than 2^31 - 1 points in one scan"; return MALIO_ERR_CAPACITY; }
  if (n) {
    if (int rc = grow_table(h, V, D, V->n_vox + n)) return rc;
    if (int rc = grow_sort(h, V, D, n)) return rc;
    if (int rc = grow_runs(h, V, D, n)) return rc;
    cudaStream_t st = D->stream;
    const PassConst pc = make_pass_const(h, D, s);
    const uint32_t nn = (uint32_t)n, g = (nn + 255) / 256;
    const uint64_t mask = V->cap_h - 1;
    CUDA_TRY(cudaMemsetAsync(V->d_small, 0, 2 * sizeof(uint32_t), st));   // fault flag, run count
    SortBufs b = sort_bufs(V);
    vm_key_kernel<<<g, 256, 0, st>>>(c, pc, 1.0f / leaf, nn, b.k.Current(), b.v.Current(), V->d_small);
    size_t t = V->cap_temp;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(V->d_temp, t, b.k, b.v, (int)nn, VKeyDecomposer{}, st));
    const VKey* key = b.k.Current();
    const uint32_t* val = b.v.Current();
    vm_head_kernel<<<g, 256, 0, st>>>(key, nn, V->d_head);
    t = V->cap_temp;
    CUDA_TRY(cub::DeviceScan::InclusiveSum(V->d_temp, t, V->d_head, V->d_rent, (int)nn, st));
    vm_run_kernel<<<g, 256, 0, st>>>(V->d_head, V->d_rent, nn, V->d_run, V->d_small);
    vm_lookup_kernel<<<g, 256, 0, st>>>(V->d_run, key, nn, V->d_small, V->d_hash, mask, V->d_ekey, V->d_rent, V->d_new);
    t = V->cap_temp;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(V->d_temp, t, V->d_new, V->d_head, (int)nn, st));
    vm_fold_kernel<<<(nn + 127) / 128, 128, 0, st>>>(c, pc, V->d_run, key, val, nn, V->d_small, V->d_rent, V->d_head,
                                                    V->d_hash, mask, V->d_ekey, V->d_esum, V->d_ecnt);
    vm_count_kernel<<<1, 1, 0, st>>>(V->d_head, V->d_new, V->d_small);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 7;
    CUDA_TRY(cudaMemcpyAsync(V->h_small, V->d_small, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));   // the call's one wait: the fault flag and the entry count
    if (V->h_small[0]) {
      h->err = "world voxel map: leaf size too small for a point's coordinates (voxel index outside int); the map is unchanged";
      return MALIO_ERR_CAPACITY;
    }
    V->n_vox = V->h_small[2];
  }
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

int save_pcd(malio_handle* h, const char* path, int clear) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (V->n_vox == 0) { h->err = "world voxel save: the voxel map is empty (nothing is written)"; return MALIO_ERR_STATE; }
  const uint64_t n = V->n_vox;
  if (int rc = grow_sort(h, V, D, n)) return rc;
  if (!V->h_bounce) CUDA_TRY(cudaHostAlloc((void**)&V->h_bounce, (size_t)malio_pcd::CHUNK * sizeof(float4), cudaHostAllocDefault));
  float4* stage = reinterpret_cast<float4*>(V->d_sort);   // the key halves: 24 B a row, the centroids take 16
  if (int rc = enqueue_sorted(h, V, D, stage, n)) return rc;
  const int rc = malio_pcd::write_binary(path, n, [&](uint64_t first, uint64_t cnt, const float** xyzi) {
    if (cudaMemcpyAsync(V->h_bounce, stage + first, cnt * sizeof(float4), cudaMemcpyDeviceToHost, D->stream) != cudaSuccess ||
        cudaStreamSynchronize(D->stream) != cudaSuccess)
      return (int)MALIO_ERR_CUDA;
    D->ctr.d2h_bytes += cnt * sizeof(float4);
    *xyzi = (const float*)V->h_bounce;
    return (int)MALIO_OK;
  }, h->err);
  // the entry-sized sort area and CUB's storage go back: between saves the map holds its entries, its hash and the scan-sized
  // scratch only (the next accumulate regrows the sort area for its scan)
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  cudaFree(V->d_sort); V->d_sort = nullptr; V->cap_s = 0;
  cudaFree(V->d_temp); V->d_temp = nullptr; V->cap_temp = 0;
  if (rc == MALIO_OK && clear) {   // an empty map with its buffers kept; the next accumulate fixes the leaf again
    CUDA_TRY(cudaMemsetAsync(V->d_hash, 0xFF, V->cap_h * sizeof(uint32_t), D->stream));
    CUDA_TRY(cudaMemsetAsync(V->d_small + 2, 0, sizeof(uint32_t), D->stream));
    V->n_vox = 0;
    V->leaf_set = false;
  }
  return rc;
}

int info(malio_handle* h, uint64_t* n_voxels, uint64_t* capacity, uint64_t* device_bytes) {
  VoxState* V;
  if (int rc = get_state(h, V)) return rc;
  if (n_voxels) *n_voxels = V->n_vox;
  if (capacity) *capacity = V->cap_e;
  if (device_bytes)
    *device_bytes = V->cap_e * (sizeof(VKey) + sizeof(float4) + sizeof(uint32_t)) + V->cap_h * sizeof(uint32_t) +
                    V->cap_s * SORT_ROW + V->cap_p * RUN_ROW + V->cap_temp;
  return MALIO_OK;
}

}  // namespace malio_vox

// the saved map as a voxel map (malio_b200.h, next to malio_world_accumulate)
extern "C" int malio_world_voxel_accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf, uint64_t* n_voxels) {
  if (!h || !s) return MALIO_ERR_INVALID_ARG;
  if (!slot_tag) { h->err = "world voxel accumulate: the dense cloud needs slot_tag"; return MALIO_ERR_INVALID_ARG; }
  MALIO_SETTLE(h);
  return malio_vox::accumulate(h, s, slot_tag, leaf, n_voxels);
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
  return malio_vox::save_pcd(h, path, clear);
}
extern "C" int malio_world_voxel_info(malio_handle* h, uint64_t* n_voxels, uint64_t* capacity, uint64_t* device_bytes) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_vox::info(h, n_voxels, capacity, device_bytes);
}
