// malio_grid.cu — a 2-D occupancy grid of a point set for navigation, sm_90a (include/malio_b200.h, "a 2-D occupancy grid"):
// per cell the ground (the lowest point around it), the points in an obstacle band above that ground and the points below it.
// Every step is an integer min, a count or a flag per cell, so the raster does not depend on thread order.
//   grid_zmin_kernel   pass 1 over the rows: atomicMin of the z key into a dense u32 raster over the padded region
//   grid_minx_kernel   the ground filter along x (half-width w) into a raster of the region's columns over the padded rows
//   grid_miny_kernel   then along y, into the region's ground keys (over the pass-1 raster, which is dead by then)
//   grid_band_kernel   pass 2 over the rows: band count and floor bit of each region cell in one u32
//   grid_class_kernel  the class and the ground of each region cell, and the report's class counts
//   grid_extent_kernel the column bounds of a source's finite points (malio_grid_extent_device)
// The row kernels are templated on a row source, as malio_voxmap.cu's fold is: caller points (device memory, or host memory
// staged chunk by chunk), the voxel map's entries in place (malio_voxrule.cuh's centroid and keep rule), or the prior followed
// by its session layer.  All scratch is local to the call and goes back before it returns.  Compiled with -fmad=false like the
// rest of the library (x * ir is one rounding either way; the band's d = z - ground is a subtraction).
#include <cuda_runtime.h>

#include <climits>
#include <cmath>
#include <cstring>
#include <string>

#include "malio_device.cuh"
#include "malio_voxrule.cuh"

using namespace malio_devstate;

namespace {

constexpr int GRID_THREADS = 256;
constexpr uint32_t ZKEY_EMPTY = 0xFFFFFFFFu;   // no point: the key of a finite z is never this (it would be a NaN's)
constexpr uint32_t FLOOR_BIT = 0x80000000u;    // a region cell's word: floor bit | band count (fewer than 2^31 rows a call)
constexpr uint32_t GROUND_NAN = 0x7FC00000u;   // the ground of a cell without a point in its window
constexpr double MAX_BOUND = (double)MALIO_GRID_MAX_BOUND;
// the report's counters on the device, 8 x u64 (64 bytes of the scratch)
enum Counter { C_USED, C_NONFINITE, C_OUTSIDE, C_OCCUPIED, C_FREE, C_UNKNOWN, C_WORDS = 8 };

// order-preserving map float <-> u32 (-0.0 < +0.0), so that the minima are integer atomics
__device__ __forceinline__ uint32_t zkey(float z) {
  const uint32_t b = __float_as_uint(z);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float zkey_inv(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

// The rows of a source.  row(p, &w) gives row p as {x, y, z, w}; false for a row that is not part of the point set.
// Caller points, float4 rows read through the read-only path
struct PointRows {
  const float4* xyzi;
  __device__ __forceinline__ bool row(uint64_t p, float4* w) const { *w = __ldg(xyzi + p); return true; }
};
// The voxel map's entries: the centroid of entry e, the voxels the keep rule drops left out (keep false: every voxel)
struct VoxelRows {
  const float4* sum;
  const uint32_t* cnt;
  const uint2* hm;
  uint32_t min_miss;
  double ratio;
  bool keep;
  __device__ __forceinline__ bool row(uint64_t e, float4* w) const {
    if (keep && malio_voxrule::dropped(malio_voxrule::evidence(hm, (uint32_t)e), min_miss, ratio)) return false;
    *w = malio_voxrule::centroid(sum[e], cnt[e]);
    return true;
  }
};
// The prior's points followed by the session's
struct PriorRows {
  const float4* prior;
  uint64_t n_prior;
  const float4* sess;
  __device__ __forceinline__ bool row(uint64_t p, float4* w) const { *w = p < n_prior ? prior[p] : sess[p - n_prior]; return true; }
};

// the region and the padded region in cells, the bounds also as (exact) floats
struct GridGeom {
  float ir;
  float pi_lo, pi_hi, pj_lo, pj_hi;   // padded region [lo, hi)
  float ri_lo, ri_hi, rj_lo, rj_hi;   // region
  int i_lo, j_lo, i0, j0;             // first padded column / row, first region column / row
  uint32_t px, py, nx, ny, w;         // padded and region extents, ground half-width
  float h_lo, h_hi;
  uint32_t min_pts;
};

// the warp's sum of v into *dst (all lanes of the warp call it)
__device__ __forceinline__ void warp_add(unsigned long long* dst, uint32_t v) {
  const uint32_t s = __reduce_add_sync(0xFFFFFFFFu, v);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(dst, (unsigned long long)s);
}

template <class Rows>
__global__ void __launch_bounds__(GRID_THREADS) grid_zmin_kernel(Rows src, uint64_t n, GridGeom g, uint32_t* __restrict__ zmin,
                                                                unsigned long long* __restrict__ ctr) {
  uint32_t used = 0, nonfinite = 0, outside = 0;
  for (uint64_t p = (uint64_t)blockIdx.x * GRID_THREADS + threadIdx.x; p < n; p += (uint64_t)gridDim.x * GRID_THREADS) {
    float4 w;
    if (!src.row(p, &w)) continue;
    if (!(isfinite(w.x) && isfinite(w.y) && isfinite(w.z))) { ++nonfinite; continue; }
    const float fi = floorf(w.x * g.ir), fj = floorf(w.y * g.ir);
    if (!(fi >= g.pi_lo && fi < g.pi_hi && fj >= g.pj_lo && fj < g.pj_hi)) { ++outside; continue; }
    ++used;
    atomicMin(zmin + (uint64_t)((int)fj - g.j_lo) * g.px + (uint32_t)((int)fi - g.i_lo), zkey(w.z));
  }
  warp_add(ctr + C_USED, used);
  warp_add(ctr + C_NONFINITE, nonfinite);
  warp_add(ctr + C_OUTSIDE, outside);
}

// out[b][i] = min over a in [i, i + 2w] of zmin[b][a]: region column i, padded row b
__global__ void __launch_bounds__(GRID_THREADS) grid_minx_kernel(GridGeom g, const uint32_t* __restrict__ zmin, uint32_t* __restrict__ out) {
  const uint64_t t = (uint64_t)blockIdx.x * GRID_THREADS + threadIdx.x;
  if (t >= (uint64_t)g.nx * g.py) return;
  const uint32_t b = (uint32_t)(t / g.nx), i = (uint32_t)(t % g.nx);
  const uint32_t* r = zmin + (uint64_t)b * g.px + i;
  uint32_t m = ZKEY_EMPTY;
  for (uint32_t a = 0; a <= 2 * g.w; ++a) m = min(m, r[a]);
  out[t] = m;
}

// gk[r][i] = min over b in [r, r + 2w] of half[b][i]: region cell (i, r)
__global__ void __launch_bounds__(GRID_THREADS) grid_miny_kernel(GridGeom g, const uint32_t* __restrict__ half, uint32_t* __restrict__ gk) {
  const uint64_t t = (uint64_t)blockIdx.x * GRID_THREADS + threadIdx.x;
  if (t >= (uint64_t)g.nx * g.ny) return;
  const uint32_t* c = half + t;   // row r of the region is padded row r + w, the window's first row is r
  uint32_t m = ZKEY_EMPTY;
  for (uint32_t b = 0; b <= 2 * g.w; ++b) m = min(m, c[(uint64_t)b * g.nx]);
  gk[t] = m;
}

template <class Rows>
__global__ void __launch_bounds__(GRID_THREADS) grid_band_kernel(Rows src, uint64_t n, GridGeom g, const uint32_t* __restrict__ gk,
                                                                uint32_t* __restrict__ band) {
  for (uint64_t p = (uint64_t)blockIdx.x * GRID_THREADS + threadIdx.x; p < n; p += (uint64_t)gridDim.x * GRID_THREADS) {
    float4 w;
    if (!src.row(p, &w)) continue;
    if (!(isfinite(w.x) && isfinite(w.y) && isfinite(w.z))) continue;
    const float fi = floorf(w.x * g.ir), fj = floorf(w.y * g.ir);
    if (!(fi >= g.ri_lo && fi < g.ri_hi && fj >= g.rj_lo && fj < g.rj_hi)) continue;
    const uint64_t c = (uint64_t)((int)fj - g.j0) * g.nx + (uint32_t)((int)fi - g.i0);
    const float d = w.z - zkey_inv(gk[c]);   // the cell holds this point: its ground is a point's z
    if (d >= g.h_lo && d <= g.h_hi) atomicAdd(band + c, 1u);
    else if (d < g.h_lo && !(*(volatile const uint32_t*)(band + c) & FLOOR_BIT)) atomicOr(band + c, FLOOR_BIT);
  }
}

__global__ void __launch_bounds__(GRID_THREADS) grid_class_kernel(GridGeom g, const uint32_t* __restrict__ gk, const uint32_t* __restrict__ band,
                                                                 uint8_t* __restrict__ cls, float* __restrict__ ground,
                                                                 unsigned long long* __restrict__ ctr) {
  const uint64_t t = (uint64_t)blockIdx.x * GRID_THREADS + threadIdx.x;
  uint32_t v = 0xFFu;
  if (t < (uint64_t)g.nx * g.ny) {
    const uint32_t b = band[t];
    v = (b & ~FLOOR_BIT) >= g.min_pts ? MALIO_GRID_OCCUPIED : ((b & FLOOR_BIT) ? MALIO_GRID_FREE : MALIO_GRID_UNKNOWN);
    cls[t] = (uint8_t)v;
    if (ground) {
      const uint32_t k = gk[t];
      ground[t] = k == ZKEY_EMPTY ? __uint_as_float(GROUND_NAN) : zkey_inv(k);
    }
  }
  const bool in = t < (uint64_t)g.nx * g.ny;
  warp_add(ctr + C_OCCUPIED, in && v == MALIO_GRID_OCCUPIED);
  warp_add(ctr + C_FREE, in && v == MALIO_GRID_FREE);
  warp_add(ctr + C_UNKNOWN, in && v == MALIO_GRID_UNKNOWN);
}

// ext = {imin, jmin, imax, jmax} over the finite rows; fault = a column index beyond +-2^24
template <class Rows>
__global__ void __launch_bounds__(GRID_THREADS) grid_extent_kernel(Rows src, uint64_t n, float ir, int* __restrict__ ext) {
  int lo_i = INT_MAX, lo_j = INT_MAX, hi_i = INT_MIN, hi_j = INT_MIN, fault = 0;
  for (uint64_t p = (uint64_t)blockIdx.x * GRID_THREADS + threadIdx.x; p < n; p += (uint64_t)gridDim.x * GRID_THREADS) {
    float4 w;
    if (!src.row(p, &w)) continue;
    if (!(isfinite(w.x) && isfinite(w.y) && isfinite(w.z))) continue;
    const float fi = floorf(w.x * ir), fj = floorf(w.y * ir);
    if (!(fabsf(fi) <= (float)MALIO_GRID_MAX_BOUND && fabsf(fj) <= (float)MALIO_GRID_MAX_BOUND)) { fault = 1; continue; }
    lo_i = min(lo_i, (int)fi); hi_i = max(hi_i, (int)fi);
    lo_j = min(lo_j, (int)fj); hi_j = max(hi_j, (int)fj);
  }
  lo_i = __reduce_min_sync(0xFFFFFFFFu, lo_i); lo_j = __reduce_min_sync(0xFFFFFFFFu, lo_j);
  hi_i = __reduce_max_sync(0xFFFFFFFFu, hi_i); hi_j = __reduce_max_sync(0xFFFFFFFFu, hi_j);
  fault = __reduce_or_sync(0xFFFFFFFFu, fault);
  if ((threadIdx.x & 31) == 0) {
    if (lo_i <= hi_i) { atomicMin(ext + 0, lo_i); atomicMin(ext + 1, lo_j); atomicMax(ext + 2, hi_i); atomicMax(ext + 3, hi_j); }
    if (fault) atomicOr(ext + 4, 1);
  }
}

// blocks of a grid-stride pass over n rows: enough to fill the device, few enough that the counters see few atomics
uint32_t row_blocks(const DeviceState* D, uint64_t n) {
  const uint64_t b = (n + GRID_THREADS - 1) / GRID_THREADS, cap = 8ull * (uint64_t)D->sm_count;
  return (uint32_t)(b < cap ? (b ? b : 1) : cap);
}
uint32_t cell_blocks(uint64_t cells) { return (uint32_t)((cells + GRID_THREADS - 1) / GRID_THREADS); }

// The rows of a source for one call.  each(k) runs k(rows, m) on each chunk of rows in order, enqueueing the chunk's kernel:
// the device sources are one chunk; caller rows in host memory are staged (HostFeed).
template <class Rows>
struct DeviceFeed {
  Rows rows;
  uint64_t n;
  template <class K>
  int each(K&& k) { return n ? k(rows, n) : MALIO_OK; }
};
// Host rows staged through the pinned bounce buffer into a device buffer of at most MALIO_GRID_CHUNK rows, chunk by chunk
// (as malio_world_voxel_seed stages them); each pass reads the host array again
struct HostFeed {
  malio_handle* h;
  DeviceState* D;
  const float4* xyzi;
  uint64_t n;
  DeviceBuffer<float4>* stage;
  PinnedBuffer<float4>* bounce;
  template <class K>
  int each(K&& k) {
    cudaStream_t st = D->stream;
    for (uint64_t first = 0; first < n; first += MALIO_GRID_CHUNK) {
      const uint64_t m = n - first < MALIO_GRID_CHUNK ? n - first : MALIO_GRID_CHUNK;
      for (uint64_t p = 0; p < m; p += malio_pcd::CHUNK) {   // the previous copy from the bounce buffer is done before it is reused
        const uint64_t c = m - p < malio_pcd::CHUNK ? m - p : malio_pcd::CHUNK;
        CUDA_TRY(cudaStreamSynchronize(st));
        std::memcpy(bounce->data(), xyzi + first + p, (size_t)c * sizeof(float4));
        CUDA_TRY(cudaMemcpyAsync(stage->data() + p, bounce->data(), (size_t)c * sizeof(float4), cudaMemcpyHostToDevice, st));
      }
      D->ctr.h2d_bytes += m * sizeof(float4);
      if (int rc = k(PointRows{stage->data()}, m)) return rc;
    }
    return MALIO_OK;
  }
};

// drains the handle's stream when the call's scratch goes out of scope (declared after the buffers: destroyed before them)
struct Drain {
  cudaStream_t st;
  ~Drain() { cudaStreamSynchronize(st); }
};

int check_args(malio_handle* h, const malio_grid_args* a, GridGeom* g) {
  if (!(a->res > 0.f) || !std::isfinite(a->res)) { h->err = "malio_grid: res must be finite and > 0"; return MALIO_ERR_INVALID_ARG; }
  if (a->nx == 0 || a->ny == 0) { h->err = "malio_grid: nx and ny must be > 0"; return MALIO_ERR_INVALID_ARG; }
  if (!(std::isfinite(a->h_lo) && std::isfinite(a->h_hi) && 0.f < a->h_lo && a->h_lo <= a->h_hi)) {
    h->err = "malio_grid: the band needs finite 0 < h_lo <= h_hi";
    return MALIO_ERR_INVALID_ARG;
  }
  if (a->min_obstacle_points == 0) { h->err = "malio_grid: min_obstacle_points must be > 0"; return MALIO_ERR_INVALID_ARG; }
  const double w = a->ground_halfwidth;
  const double b[4] = {(double)a->i0 - w, (double)a->i0 + a->nx + w, (double)a->j0 - w, (double)a->j0 + a->ny + w};
  for (double v : b)
    if (std::fabs(v) > MAX_BOUND) {
      h->err = "malio_grid: a bound of the padded region lies beyond 2^24 cells (not exact as a float)";
      return MALIO_ERR_INVALID_ARG;
    }
  g->ir = 1.0f / a->res;
  g->pi_lo = (float)b[0]; g->pi_hi = (float)b[1]; g->pj_lo = (float)b[2]; g->pj_hi = (float)b[3];
  g->ri_lo = (float)a->i0; g->ri_hi = (float)((double)a->i0 + a->nx);
  g->rj_lo = (float)a->j0; g->rj_hi = (float)((double)a->j0 + a->ny);
  g->i_lo = (int)b[0]; g->j_lo = (int)b[2]; g->i0 = a->i0; g->j0 = a->j0;
  g->nx = a->nx; g->ny = a->ny; g->w = a->ground_halfwidth;
  g->px = a->nx + 2 * a->ground_halfwidth; g->py = a->ny + 2 * a->ground_halfwidth;
  g->h_lo = a->h_lo; g->h_hi = a->h_hi; g->min_pts = a->min_obstacle_points;
  return MALIO_OK;
}

// the scratch of the header's figure: column minima, the half-way raster, the band words, the counters
uint64_t scratch_bytes(const GridGeom& g) {
  return 4 * ((uint64_t)g.px * g.py + (uint64_t)g.nx * g.py + (uint64_t)g.nx * g.ny) + C_WORDS * sizeof(unsigned long long);
}

// Runs body(feed) on the rows of `source` after checking them: MALIO_GRID_POINTS' pointer (16-byte rows), the voxel map's
// and the prior's state, the keep rule, and fewer than 2^31 rows.
template <class Body>
int with_source(malio_handle* h, DeviceState* D, int source, const float* d_xyzi, uint64_t n, const malio_carve_keep* k,
                const char* what, Body&& body) {
  auto capacity = [&](uint64_t rows) -> int {
    if (rows < 0x80000000ull) return MALIO_OK;
    h->err = std::string(what) + ": 2^31 or more rows";
    return MALIO_ERR_CAPACITY;
  };
  if (source == MALIO_GRID_POINTS) {
    if (n) {
      if (int rc = check_device_ptr(h, D, d_xyzi, what, 16, "the rows are read as float4")) return rc;
    }
    if (int rc = capacity(n)) return rc;
    DeviceFeed<PointRows> f{PointRows{reinterpret_cast<const float4*>(d_xyzi)}, n};
    return body(f);
  }
  if (source == MALIO_GRID_VOXEL_MAP) {
    if (k && !(std::isfinite(k->max_miss_per_hit) && k->max_miss_per_hit >= 0.f)) {
      h->err = "world voxel keep rule: max_miss_per_hit must be finite and >= 0";
      return MALIO_ERR_INVALID_ARG;
    }
    malio_vox::Entries e{};
    if (malio_vox::entries(h, &e)) { h->err = std::string(what) + ": the voxel map is empty"; return MALIO_ERR_STATE; }
    if (int rc = capacity(e.n)) return rc;
    const VoxelRows r{reinterpret_cast<const float4*>(e.sum), e.cnt, reinterpret_cast<const uint2*>(e.hit_miss), k ? k->min_miss : 0u,
                      k ? (double)k->max_miss_per_hit : 0.0, k != nullptr};
    DeviceFeed<VoxelRows> f{r, e.n};
    return body(f);
  }
  if (source == MALIO_GRID_PRIOR) {
    const float *p = nullptr, *s = nullptr;
    uint32_t np = 0, ns = 0;
    if (malio_prior::points(h, &p, &np) || malio_prior::session(h, &s, &ns)) {
      h->err = std::string(what) + ": no prior map loaded";
      return MALIO_ERR_STATE;
    }
    if (int rc = capacity((uint64_t)np + ns)) return rc;
    DeviceFeed<PriorRows> f{PriorRows{reinterpret_cast<const float4*>(p), np, reinterpret_cast<const float4*>(s)}, (uint64_t)np + ns};
    return body(f);
  }
  h->err = std::string(what) + ": unknown source";
  return MALIO_ERR_INVALID_ARG;
}

// The grid of feed's rows into cls / ground (device memory; ground may be NULL), on the handle's stream.  extra: bytes the
// caller holds for the call besides this scratch (the host entry's stage and output copies), for the limit and the report.
// caller: the stream to order the call on (host entry: none).  Waits once, at the end.
template <class Feed>
int build(malio_handle* h, DeviceState* D, const GridGeom& g, Feed& feed, uint64_t extra, uint8_t* cls, float* ground,
          bool ordered, cudaStream_t caller, malio_grid_report* rep) {
  const uint64_t bytes = scratch_bytes(g) + extra;
  if (bytes > MALIO_GRID_MAX_BYTES) {
    h->err = "malio_grid: the call needs " + std::to_string(bytes) + " bytes of scratch, above MALIO_GRID_MAX_BYTES";
    return MALIO_ERR_CAPACITY;
  }
  const uint64_t padded = (uint64_t)g.px * g.py, half = (uint64_t)g.nx * g.py, cells = (uint64_t)g.nx * g.ny;
  DeviceBuffer<uint32_t> d_z, d_half, d_band;
  DeviceBuffer<unsigned long long> d_ctr;
  cudaStream_t st = D->stream;
  if (int rc = malio_buf::allocate_group(h, st, {{d_z, padded}, {d_half, half}, {d_band, cells}, {d_ctr, (size_t)C_WORDS}})) return rc;
  Drain drain{st};
  if (ordered) { if (int rc = caller_enter(h, D, caller)) return rc; }
  CUDA_TRY(cudaMemsetAsync(d_z, 0xFF, padded * sizeof(uint32_t), st));
  CUDA_TRY(cudaMemsetAsync(d_band, 0, cells * sizeof(uint32_t), st));
  CUDA_TRY(cudaMemsetAsync(d_ctr, 0, C_WORDS * sizeof(unsigned long long), st));
  uint32_t launches = 0;
  if (int rc = feed.each([&](const auto& rows, uint64_t m) -> int {
        grid_zmin_kernel<<<row_blocks(D, m), GRID_THREADS, 0, st>>>(rows, m, g, d_z.data(), d_ctr.data());
        ++launches;
        CUDA_TRY(cudaGetLastError());
        return (int)MALIO_OK;
      }))
    return rc;
  grid_minx_kernel<<<cell_blocks(half), GRID_THREADS, 0, st>>>(g, d_z, d_half);
  grid_miny_kernel<<<cell_blocks(cells), GRID_THREADS, 0, st>>>(g, d_half, d_z);   // the ground keys over the pass-1 raster
  CUDA_TRY(cudaGetLastError());
  if (int rc = feed.each([&](const auto& rows, uint64_t m) -> int {
        grid_band_kernel<<<row_blocks(D, m), GRID_THREADS, 0, st>>>(rows, m, g, d_z.data(), d_band.data());
        ++launches;
        CUDA_TRY(cudaGetLastError());
        return (int)MALIO_OK;
      }))
    return rc;
  grid_class_kernel<<<cell_blocks(cells), GRID_THREADS, 0, st>>>(g, d_z, d_band, cls, ground, d_ctr);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += launches + 3;
  if (ordered) { if (int rc = caller_leave(h, D, caller)) return rc; }
  unsigned long long c[C_WORDS];
  CUDA_TRY(cudaMemcpyAsync(c, d_ctr, sizeof(c), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // the call's one wait: the counters, and the scratch may go back
  D->ctr.d2h_bytes += sizeof(c);
  if (rep) {
    rep->n_used = c[C_USED]; rep->n_nonfinite = c[C_NONFINITE]; rep->n_outside = c[C_OUTSIDE];
    rep->n_occupied = c[C_OCCUPIED]; rep->n_free = c[C_FREE]; rep->n_unknown = c[C_UNKNOWN];
    rep->device_bytes = bytes;
  }
  return MALIO_OK;
}

}  // namespace

namespace malio_grid {

int build_device(malio_handle* h, int source, const float* d_xyzi, uint64_t n, const malio_carve_keep* k, const malio_grid_args* a,
                 uint8_t* d_cls, float* d_ground, cudaStream_t caller, malio_grid_report* rep) {
  GridGeom g{};
  if (int rc = check_args(h, a, &g)) return rc;
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  if (int rc = check_device_ptrs(h, D, {{d_cls, "malio_grid_build_device cls"}, {d_ground, "malio_grid_build_device ground"}})) return rc;
  return with_source(h, D, source, d_xyzi, n, k, "malio_grid_build_device", [&](auto& feed) -> int {
    return build(h, D, g, feed, 0, d_cls, d_ground, true, caller, rep);
  });
}

int build_host(malio_handle* h, const float* xyzi, uint64_t n, const malio_grid_args* a, uint8_t* cls, float* ground,
               malio_grid_report* rep) {
  GridGeom g{};
  if (int rc = check_args(h, a, &g)) return rc;
  if (n >= 0x80000000ull) { h->err = "malio_grid_build: 2^31 or more rows"; return MALIO_ERR_CAPACITY; }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  const uint64_t cells = (uint64_t)g.nx * g.ny, chunk = n < MALIO_GRID_CHUNK ? n : MALIO_GRID_CHUNK;
  const uint64_t extra = chunk * sizeof(float4) + cells * (ground ? 5 : 1);
  if (scratch_bytes(g) + extra > MALIO_GRID_MAX_BYTES) {
    h->err = "malio_grid_build: the call needs " + std::to_string(scratch_bytes(g) + extra) + " bytes of scratch, above MALIO_GRID_MAX_BYTES";
    return MALIO_ERR_CAPACITY;
  }
  DeviceBuffer<float4> stage;
  DeviceBuffer<uint8_t> d_cls;
  DeviceBuffer<float> d_ground;
  PinnedBuffer<float4> bounce;
  if (int rc = malio_buf::allocate_group(h, D->stream, {{d_cls, cells}})) return rc;
  if (ground) { if (int rc = d_ground.allocate(h, D->stream, cells)) return rc; }
  if (chunk) {
    if (int rc = stage.allocate(h, D->stream, chunk)) return rc;
    if (int rc = bounce.allocate(h, malio_pcd::CHUNK)) return rc;
  }
  HostFeed feed{h, D, reinterpret_cast<const float4*>(xyzi), n, &stage, &bounce};
  if (int rc = build(h, D, g, feed, extra, d_cls, ground ? d_ground.data() : nullptr, false, nullptr, rep)) return rc;
  CUDA_TRY(cudaMemcpyAsync(cls, d_cls, cells, cudaMemcpyDeviceToHost, D->stream));
  if (ground) CUDA_TRY(cudaMemcpyAsync(ground, d_ground, cells * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  D->ctr.d2h_bytes += cells * (ground ? 5 : 1);
  return MALIO_OK;
}

int extent_device(malio_handle* h, int source, const float* d_xyzi, uint64_t n, const malio_carve_keep* k, float res, int32_t* ext,
                  cudaStream_t caller) {
  if (!(res > 0.f) || !std::isfinite(res)) { h->err = "malio_grid_extent_device: res must be finite and > 0"; return MALIO_ERR_INVALID_ARG; }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  return with_source(h, D, source, d_xyzi, n, k, "malio_grid_extent_device", [&](auto& feed) -> int {
    cudaStream_t st = D->stream;
    DeviceBuffer<int> d_ext;
    if (int rc = d_ext.allocate(h, st, 5)) return rc;
    Drain drain{st};
    int e[5] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN, 0};
    CUDA_TRY(cudaMemcpyAsync(d_ext, e, sizeof(e), cudaMemcpyHostToDevice, st));
    if (int rc = caller_enter(h, D, caller)) return rc;
    const float ir = 1.0f / res;
    if (int rc = feed.each([&](const auto& rows, uint64_t m) -> int {
          grid_extent_kernel<<<row_blocks(D, m), GRID_THREADS, 0, st>>>(rows, m, ir, d_ext.data());
          D->ctr.kernel_launches += 1;
          CUDA_TRY(cudaGetLastError());
          return (int)MALIO_OK;
        }))
      return rc;
    if (int rc = caller_leave(h, D, caller)) return rc;
    CUDA_TRY(cudaMemcpyAsync(e, d_ext, sizeof(e), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (e[4]) { h->err = "malio_grid_extent_device: a point's column index lies beyond 2^24"; return (int)MALIO_ERR_CAPACITY; }
    const bool none = e[0] > e[2];
    ext[0] = none ? 0 : e[0]; ext[1] = none ? 0 : e[1]; ext[2] = none ? -1 : e[2]; ext[3] = none ? -1 : e[3];
    return (int)MALIO_OK;
  });
}

}  // namespace malio_grid

// the 2-D occupancy grid (malio_b200.h, after relocalization)
extern "C" int malio_grid_build_device(malio_handle* h, int source, const float* d_xyzi, uint64_t n, const malio_carve_keep* k,
                                       const malio_grid_args* args, uint8_t* d_cls, float* d_ground, void* stream, malio_grid_report* rep) {
  if (!h || !args || !d_cls) return MALIO_ERR_INVALID_ARG;
  if (source == MALIO_GRID_POINTS && n && !d_xyzi) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_grid::build_device(h, source, d_xyzi, n, k, args, d_cls, d_ground, (cudaStream_t)stream, rep);
}
extern "C" int malio_grid_build(malio_handle* h, const float* xyzi, uint64_t n, const malio_grid_args* args, uint8_t* cls, float* ground,
                                malio_grid_report* rep) {
  if (!h || !args || !cls || (n && !xyzi)) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_grid::build_host(h, xyzi, n, args, cls, ground, rep);
}
extern "C" int malio_grid_extent_device(malio_handle* h, int source, const float* d_xyzi, uint64_t n, const malio_carve_keep* k, float res,
                                        int32_t* ext, void* stream) {
  if (!h || !ext) return MALIO_ERR_INVALID_ARG;
  if (source == MALIO_GRID_POINTS && n && !d_xyzi) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_grid::extent_device(h, source, d_xyzi, n, k, res, ext, (cudaStream_t)stream);
}
