// malio_place.cu — relocalization without a position guess, sm_90a: place descriptors of the loaded prior on a lattice of
// positions, ranked against the resident scan, the best few checked by malio_relocalize (malio_place_db_build /
// malio_relocalize_global, malio_b200.h).  A Scan Context style descriptor made exact: heights binned into 4-bit levels over
// (ring, sector) bins by one host-built table that the database and the query share, so every stage after the heights is
// integer arithmetic.
//   pl_bbox_kernel     the prior's column bounding box (floor((double)x / cell) per axis) and a flag for indices beyond 2^30
//   pl_fold_kernel     the column grids: largest and smallest z per column, folded with order-independent atomics
//   pl_flag_kernel     the lattice columns (indices multiples of step / cell) that hold a point; a CUB scan numbers them
//   pl_scatter_kernel  the positions, (j, i) order: column and virtual sensor height z_s
//   pl_db_desc_kernel  one block per position: the stencil's columns -> per-bin maximum level in shared memory -> nibbles, ring keys
//   pl_query_cols_kernel / pl_query_desc_kernel   the scan's column heights around the slot-0 origin and its descriptor
//   pl_stage1_kernel   ring-key L1 distance of every position, packed (d1, p) and sorted by CUB's radix sort
//   pl_stage2_kernel   one block per stage-1 survivor: bin-wise L1 distance under every sector shift, the minimum
// Stage 3 is malio_relocalize, unchanged, once per stage-2 survivor.  Compiled with -fmad=false like the rest of the library;
// the host code that builds the table and the verification guesses is compiled without FP contraction (Makefile).
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "malio_device.cuh"

using namespace malio_devstate;

namespace {

constexpr int DESC_T = 256;
constexpr int ST2_T = 256;
constexpr int32_t COL_LIM = 1 << 30;       // |column index| < 2^30
constexpr uint32_t FLAG_RANGE = 1u;

struct StEntry { int16_t ox, oy; uint16_t bin; uint8_t cap, pad; };   // one stencil offset: its bin and its ring's level cap

// the binning of one database, shared by the query (malio_b200.h, steps 1-2)
struct Binning {
  const StEntry* st; uint32_t n_st;
  uint32_t n_ring, n_sector, n_bins;
  double z_lo, dz;
  uint32_t block;
};

struct Stage2Out { uint32_t p, d1, d2, shift; int32_t i, j; double z_s; };

// order-preserving float <-> uint32 for the column grids' atomics; 0 is below every finite float's key (the empty column)
__device__ __forceinline__ uint32_t fkey(float v) {
  const uint32_t b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

__device__ __forceinline__ uint32_t level_of(double z_rel, double z_lo, double dz) {
  if (!(z_rel >= z_lo)) return 0;
  double t = floor((z_rel - z_lo) / dz);
  t = t < 0.0 ? 0.0 : (t > 14.0 ? 14.0 : t);
  return 1u + (uint32_t)t;
}

// ---------------------------------------------------------------------------------------------------- database kernels
// small: [0] flags, [1] min i, [2] min j, [3] max i, [4] max j
__global__ void __launch_bounds__(256) pl_bbox_kernel(const float4* __restrict__ pts, uint32_t n, double cell, int* __restrict__ small) {
  const uint32_t t = blockIdx.x * 256u + threadIdx.x;
  bool ok = false;
  int ci = 0, cj = 0;
  if (t < n) {
    const float4 p = pts[t];
    const double fi = floor((double)p.x / cell), fj = floor((double)p.y / cell);
    if (fabs(fi) < (double)COL_LIM && fabs(fj) < (double)COL_LIM) { ci = (int)fi; cj = (int)fj; ok = true; }
    else atomicOr(small, (int)FLAG_RANGE);
  }
  const int mn0 = __reduce_min_sync(0xffffffffu, ok ? ci : INT_MAX), mn1 = __reduce_min_sync(0xffffffffu, ok ? cj : INT_MAX);
  const int mx0 = __reduce_max_sync(0xffffffffu, ok ? ci : INT_MIN), mx1 = __reduce_max_sync(0xffffffffu, ok ? cj : INT_MIN);
  if ((threadIdx.x & 31) == 0 && mn0 <= mx0) {
    atomicMin(small + 1, mn0); atomicMin(small + 2, mn1); atomicMax(small + 3, mx0); atomicMax(small + 4, mx1);
  }
}

__global__ void __launch_bounds__(256) pl_fold_kernel(const float4* __restrict__ pts, uint32_t n, double cell, int ilo, int jlo, uint32_t nx,
                                                      uint32_t* __restrict__ gmax, uint32_t* __restrict__ gmin) {
  const uint32_t t = blockIdx.x * 256u + threadIdx.x;
  if (t >= n) return;
  const float4 p = pts[t];
  const size_t c = (size_t)((int)floor((double)p.y / cell) - jlo) * nx + (size_t)((int)floor((double)p.x / cell) - ilo);
  const uint32_t k = fkey(p.z);
  atomicMax(gmax + c, k);
  atomicMin(gmin + c, k);
}

// lattice cell t = b * lx + a: grid column (gi0 + a m, gj0 + b m); flag[nl] = 0 closes the scan
__global__ void __launch_bounds__(256) pl_flag_kernel(const uint32_t* __restrict__ gmax, uint32_t nx, uint32_t gi0, uint32_t gj0, uint32_t m,
                                                      uint32_t lx, uint32_t nl, uint32_t* __restrict__ flag) {
  const uint32_t t = blockIdx.x * 256u + threadIdx.x;
  if (t > nl) return;
  if (t == nl) { flag[t] = 0; return; }
  const uint32_t a = t % lx, b = t / lx;
  flag[t] = gmax[(size_t)(gj0 + b * m) * nx + gi0 + a * m] != 0u;
}

__global__ void __launch_bounds__(256) pl_scatter_kernel(const uint32_t* __restrict__ gmin, const uint32_t* __restrict__ off, uint32_t nx,
                                                         int ilo, int jlo, uint32_t gi0, uint32_t gj0, uint32_t m, uint32_t lx, uint32_t nl,
                                                         double sensor_height, int2* __restrict__ cols, double* __restrict__ zs) {
  const uint32_t t = blockIdx.x * 256u + threadIdx.x;
  if (t >= nl || off[t + 1] == off[t]) return;
  const uint32_t gi = gi0 + (t % lx) * m, gj = gj0 + (t / lx) * m;
  const uint32_t p = off[t];
  cols[p] = make_int2(ilo + (int)gi, jlo + (int)gj);
  zs[p] = (double)fkey_inv(gmin[(size_t)gj * nx + gi]) + sensor_height;
}

// the per-bin maximum level of a stencil walk, in shared memory lv[n_bins] (zeroed by the caller); height(ox, oy, &z) -> a
// column's height above the sensor, false for an empty or out-of-range column
template <class Height>
__device__ __forceinline__ void walk(const Binning& b, uint32_t* lv, Height height) {
  for (uint32_t t = threadIdx.x; t < b.n_st; t += blockDim.x) {
    const StEntry e = b.st[t];
    double z;
    if (!height(e.ox, e.oy, z)) continue;
    uint32_t l = level_of(z, b.z_lo, b.dz);
    if (!l) continue;
    l = l < e.cap ? l : e.cap;
    atomicMax(lv + e.bin, l);
  }
}

// occlusion (after the walk's barrier): in every sector, the rings beyond the first bin of level >= block are emptied
__device__ __forceinline__ void occlude(const Binning& b, uint32_t* lv) {
  if (!b.block) return;
  for (uint32_t c = threadIdx.x; c < b.n_sector; c += blockDim.x) {
    bool hidden = false;
    for (uint32_t r = 0; r < b.n_ring; ++r) {
      uint32_t& v = lv[r * b.n_sector + c];
      if (hidden) v = 0;
      else if (v >= b.block) hidden = true;
    }
  }
}

__global__ void __launch_bounds__(DESC_T) pl_db_desc_kernel(Binning b, const uint32_t* __restrict__ gmax, int ilo, int jlo, uint32_t nx,
                                                            uint32_t ny, const int2* __restrict__ cols, const double* __restrict__ zs,
                                                            uint32_t bpp, uint8_t* __restrict__ nib, uint16_t* __restrict__ rk) {
  __shared__ uint32_t lv[MALIO_PLACE_MAX_BINS];
  const size_t p = blockIdx.x;
  for (uint32_t k = threadIdx.x; k < b.n_bins; k += DESC_T) lv[k] = 0;
  __syncthreads();
  const int2 c = cols[p];
  const double z_s = zs[p];
  const int gi0 = c.x - ilo, gj0 = c.y - jlo;
  walk(b, lv, [&](int ox, int oy, double& z) {
    const int gi = gi0 + ox, gj = gj0 + oy;
    if (gi < 0 || gj < 0 || gi >= (int)nx || gj >= (int)ny) return false;
    const uint32_t k = __ldg(gmax + (size_t)gj * nx + gi);
    if (!k) return false;
    z = (double)fkey_inv(k) - z_s;
    return true;
  });
  __syncthreads();
  occlude(b, lv);
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < bpp; k += DESC_T) {
    const uint32_t lo = lv[2 * k], hi = 2 * k + 1 < b.n_bins ? lv[2 * k + 1] : 0u;
    nib[p * bpp + k] = (uint8_t)(lo | (hi << 4));
  }
  for (uint32_t r = threadIdx.x; r < b.n_ring; r += DESC_T) {
    uint32_t s = 0;
    for (uint32_t c2 = 0; c2 < b.n_sector; ++c2) s += lv[r * b.n_sector + c2];
    rk[p * b.n_ring + r] = (uint16_t)s;
  }
}

// ---------------------------------------------------------------------------------------------------- query kernels
// qg[(cy + R) * (2R + 1) + cx + R] = the largest dkey(rel z) of the column (0: empty)
__global__ void __launch_bounds__(256) pl_query_cols_kernel(const malio_scan_pt* __restrict__ pts, uint32_t n, PassConst pc, double cell,
                                                            int R, unsigned long long* __restrict__ qg) {
  const uint32_t t = blockIdx.x * 256u + threadIdx.x;
  if (t >= n) return;
  float o[3], w[3];
  body_to_world(pc, 0, 0.f, 0.f, 0.f, o);
  const malio_scan_pt p = pts[t];
  body_to_world(pc, p.lidar, p.x, p.y, p.z, w);
  if (!(isfinite(w[0]) && isfinite(w[1]) && isfinite(w[2]))) return;
  const double cx = floor(((double)w[0] - (double)o[0]) / cell + 0.5), cy = floor(((double)w[1] - (double)o[1]) / cell + 0.5);
  if (!(fabs(cx) <= (double)R && fabs(cy) <= (double)R)) return;
  const int W = 2 * R + 1;
  atomicMax(qg + (size_t)((int)cy + R) * W + ((int)cx + R), dkey((double)w[2] - (double)o[2]));
}

// one block: the query's bin values q[n_bins] (one byte each) and ring keys qk[n_ring]
__global__ void __launch_bounds__(DESC_T) pl_query_desc_kernel(Binning b, const unsigned long long* __restrict__ qg, int R,
                                                               uint8_t* __restrict__ q, uint16_t* __restrict__ qk) {
  __shared__ uint32_t lv[MALIO_PLACE_MAX_BINS];
  for (uint32_t k = threadIdx.x; k < b.n_bins; k += DESC_T) lv[k] = 0;
  __syncthreads();
  const int W = 2 * R + 1;
  walk(b, lv, [&](int ox, int oy, double& z) {
    const unsigned long long k = qg[(size_t)(oy + R) * W + (ox + R)];
    if (!k) return false;
    z = dkey_inv(k);
    return true;
  });
  __syncthreads();
  occlude(b, lv);
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < b.n_bins; k += DESC_T) q[k] = (uint8_t)lv[k];
  for (uint32_t r = threadIdx.x; r < b.n_ring; r += DESC_T) {
    uint32_t s = 0;
    for (uint32_t c = 0; c < b.n_sector; ++c) s += lv[r * b.n_sector + c];
    qk[r] = (uint16_t)s;
  }
}

// ---------------------------------------------------------------------------------------------------- ranking kernels
__global__ void __launch_bounds__(256) pl_stage1_kernel(const uint16_t* __restrict__ rk, uint32_t n_pos, uint32_t n_ring,
                                                        const uint16_t* __restrict__ qk, unsigned long long* __restrict__ key) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n_pos) return;
  uint32_t d = 0;
  for (uint32_t r = 0; r < n_ring; ++r) {
    const int v = (int)rk[(size_t)p * n_ring + r] - (int)qk[r];
    d += (uint32_t)(v < 0 ? -v : v);
  }
  key[p] = ((unsigned long long)d << 32) | p;
}

// block t: the stage-1 survivor of rank t; warps over shifts, lanes over bins
__global__ void __launch_bounds__(ST2_T) pl_stage2_kernel(const unsigned long long* __restrict__ sorted, uint32_t n_ring, uint32_t n_sector,
                                                          const uint8_t* __restrict__ q, const uint8_t* __restrict__ nib, uint32_t bpp,
                                                          const int2* __restrict__ cols, const double* __restrict__ zs,
                                                          Stage2Out* __restrict__ out) {
  __shared__ uint8_t sq[MALIO_PLACE_MAX_BINS], sd[MALIO_PLACE_MAX_BINS];
  __shared__ unsigned long long best[ST2_T / 32];
  const unsigned long long key = sorted[blockIdx.x];
  const uint32_t p = (uint32_t)key;
  const uint32_t nb = n_ring * n_sector;
  for (uint32_t k = threadIdx.x; k < nb; k += ST2_T) {
    sq[k] = q[k];
    const uint8_t v = nib[(size_t)p * bpp + (k >> 1)];
    sd[k] = (k & 1u) ? (uint8_t)(v >> 4) : (uint8_t)(v & 15u);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long mine = ~0ull;
  for (uint32_t s = warp; s < n_sector; s += ST2_T / 32) {
    uint32_t d = 0;
    for (uint32_t k = lane; k < nb; k += 32) {
      const uint32_t r = k / n_sector, c = k - r * n_sector;
      uint32_t cs = c + s;
      if (cs >= n_sector) cs -= n_sector;
      const int v = (int)sq[k] - (int)sd[r * n_sector + cs];
      d += (uint32_t)(v < 0 ? -v : v);
    }
    d = __reduce_add_sync(0xffffffffu, d);
    const unsigned long long kk = ((unsigned long long)d << 32) | s;
    mine = kk < mine ? kk : mine;
  }
  if (lane == 0) best[warp] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long b = best[0];
    for (int w = 1; w < ST2_T / 32; ++w) b = best[w] < b ? best[w] : b;
    const int2 c = cols[p];
    out[blockIdx.x] = Stage2Out{p, (uint32_t)(key >> 32), (uint32_t)(b >> 32), (uint32_t)b, c.x, c.y, zs[p]};
  }
}

}  // namespace

namespace malio_place {

// ---------------------------------------------------------------------------------------------------- host
struct PlaceDb {
  malio_place_args args{};
  uint64_t n = 0;
  uint32_t bpp = 0, n_bins = 0, n_st = 0, R = 0;
  DeviceBuffer<StEntry> d_st;
  DeviceBuffer<int2> d_cols;
  DeviceBuffer<double> d_zs;
  DeviceBuffer<uint8_t> d_nib;
  DeviceBuffer<uint16_t> d_rk;
  size_t bytes() const { return d_st.bytes() + d_cols.bytes() + d_zs.bytes() + d_nib.bytes() + d_rk.bytes(); }
  // the database of the loaded prior (n_prior points), built whole
  int init(malio_handle* h, DeviceState* D, const malio_place_args* a, const float4* prior, uint32_t n_prior, malio_place_db_report* rep);
};

}  // namespace malio_place

namespace {

using malio_place::PlaceDb;

int64_t floor_div(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// malio_b200.h step 1 and the caps of step 2, host double arithmetic without contraction
void make_table(const malio_place_args& a, std::vector<StEntry>& st, uint32_t& R) {
  const uint32_t S = a.n_sector, Q = S / 4;
  R = (uint32_t)std::ceil(a.r_max / a.cell);
  std::vector<double> rad2(a.n_ring);
  for (uint32_t k = 1; k < a.n_ring; ++k) {
    const double rk = a.r_max * (double)k / (double)a.n_ring;
    rad2[k] = rk * rk;
  }
  std::vector<double> bx(Q), by(Q);
  for (uint32_t j = 1; j < Q; ++j) {
    const double phi = 2.0 * M_PI * (double)j / (double)S;
    bx[j] = std::cos(phi);
    by[j] = std::sin(phi);
    if (8 * j == S) bx[j] = by[j] = std::sqrt(0.5);
  }
  std::vector<uint8_t> cap(a.n_ring, 15);
  if (a.fov_up < M_PI / 2) {
    const double tf = std::tan(a.fov_up);
    for (uint32_t r = 0; r < a.n_ring; ++r) {
      const double rho = a.r_max * (double)r / (double)a.n_ring;
      const double z = rho * tf;
      uint32_t l = 1;
      if (z >= a.z_lo) {
        double t = std::floor((z - a.z_lo) / a.dz);
        t = t < 0.0 ? 0.0 : (t > 14.0 ? 14.0 : t);
        l = 1u + (uint32_t)t;
      }
      cap[r] = (uint8_t)l;
    }
  }
  const double r2max = a.r_max * a.r_max;
  st.clear();
  for (int oy = -(int)R; oy <= (int)R; ++oy)
    for (int ox = -(int)R; ox <= (int)R; ++ox) {
      if (ox == 0 && oy == 0) continue;
      const double x = (double)ox * a.cell, y = (double)oy * a.cell;
      const double r2 = x * x + y * y;
      if (!(r2 < r2max)) continue;
      uint32_t ring = 0;
      for (uint32_t k = 1; k < a.n_ring; ++k) ring += r2 >= rad2[k];
      uint32_t q;
      double u, v;
      if (x > 0 && y >= 0) { q = 0; u = x; v = y; }
      else if (x <= 0 && y > 0) { q = 1; u = y; v = -x; }
      else if (x < 0 && y <= 0) { q = 2; u = -x; v = -y; }
      else { q = 3; u = -y; v = x; }
      uint32_t sec = q * Q;
      for (uint32_t j = 1; j < Q; ++j) sec += bx[j] * v - by[j] * u >= 0.0;
      st.push_back(StEntry{(int16_t)ox, (int16_t)oy, (uint16_t)(ring * S + sec), cap[ring], 0});
    }
}

int check_args(malio_handle* h, const malio_place_args* a) {
  auto pos = [](double v) { return std::isfinite(v) && v > 0.0; };
  bool ok = pos(a->cell) && pos(a->step) && pos(a->r_max) && pos(a->dz) && std::isfinite(a->sensor_height) && std::isfinite(a->z_lo) &&
            !std::isnan(a->fov_up) && a->block_level <= 15 && a->n_ring > 0 && a->n_sector > 0 && a->n_sector % 4 == 0 &&
            (uint64_t)a->n_ring * a->n_sector <= MALIO_PLACE_MAX_BINS;
  if (ok) {
    const double m = std::round(a->step / a->cell);
    ok = m >= 1.0 && m < 65536.0 && m * a->cell == a->step && a->r_max / a->cell <= (double)MALIO_PLACE_MAX_RADIUS_CELLS;
  }
  if (!ok) {
    h->err = "malio_place_db_build: cell, step, r_max, dz finite and > 0; step an integer multiple of cell; n_ring > 0; n_sector a "
             "positive multiple of 4; n_ring x n_sector <= MALIO_PLACE_MAX_BINS; r_max / cell <= MALIO_PLACE_MAX_RADIUS_CELLS; "
             "sensor_height, z_lo finite; fov_up not NaN; block_level <= 15";
    return MALIO_ERR_INVALID_ARG;
  }
  return MALIO_OK;
}

// the build's scratch, released (after the drain in db_build) before it returns
struct BuildScratch {
  DeviceBuffer<int> d_small;
  DeviceBuffer<uint32_t> d_gmax, d_gmin, d_flag, d_off;
  DeviceBuffer<char> d_temp;
  size_t bytes() const { return d_small.bytes() + d_gmax.bytes() + d_gmin.bytes() + d_flag.bytes() + d_off.bytes() + d_temp.bytes(); }
};

int build(malio_handle* h, DeviceState* D, const malio_place_args* a, const float4* prior, uint32_t n_prior, PlaceDb& P, BuildScratch& S,
          malio_place_db_report* rep) {
  cudaStream_t st = D->stream;
  std::vector<StEntry> tab;
  uint32_t R;
  make_table(*a, tab, R);
  P.args = *a;
  P.R = R;
  P.n_st = (uint32_t)tab.size();
  P.n_bins = a->n_ring * a->n_sector;
  P.bpp = (P.n_bins + 1) / 2;
  if (int rc = P.d_st.allocate(h, st, tab.size() ? tab.size() : 1)) return rc;
  CUDA_TRY(cudaMemcpyAsync(P.d_st, tab.data(), tab.size() * sizeof(StEntry), cudaMemcpyHostToDevice, st));
  D->ctr.h2d_bytes += tab.size() * sizeof(StEntry);
  malio_place_db_report r{};
  r.n_stencil = P.n_st;
  r.bytes_per_position = (uint32_t)(sizeof(int2) + sizeof(double) + P.bpp + 2 * a->n_ring);
  if (n_prior) {
    if (int rc = S.d_small.allocate(h, st, 5)) return rc;
    const int init[5] = {0, INT_MAX, INT_MAX, INT_MIN, INT_MIN};
    CUDA_TRY(cudaMemcpyAsync(S.d_small, init, sizeof(init), cudaMemcpyHostToDevice, st));
    pl_bbox_kernel<<<(n_prior + 255) / 256, 256, 0, st>>>(prior, n_prior, a->cell, S.d_small);
    CUDA_TRY(cudaGetLastError());
    int small[5];
    CUDA_TRY(cudaMemcpyAsync(small, S.d_small, sizeof(small), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    D->ctr.kernel_launches += 1;
    D->ctr.h2d_bytes += sizeof(init);
    D->ctr.d2h_bytes += sizeof(small);
    if (small[0] & FLAG_RANGE) { h->err = "malio_place_db_build: a prior point's column index lies outside +-2^30 (cell too small)"; return MALIO_ERR_CAPACITY; }
    const int ilo = small[1], jlo = small[2];
    const uint64_t nx = (uint64_t)((int64_t)small[3] - ilo + 1), ny = (uint64_t)((int64_t)small[4] - jlo + 1);
    const long double gbytes = (long double)nx * ny * 8.0L;
    if (gbytes > (long double)MALIO_PLACE_MAX_GRID_BYTES || nx >= (1ull << 31) || ny >= (1ull << 31)) {
      h->err = "malio_place_db_build: the column grids need " + std::to_string((double)gbytes) + " bytes over " + std::to_string(nx) +
               " x " + std::to_string(ny) + " columns (limit MALIO_PLACE_MAX_GRID_BYTES): a coarser cell or a smaller prior";
      return MALIO_ERR_CAPACITY;
    }
    r.grid_nx = (uint32_t)nx;
    r.grid_ny = (uint32_t)ny;
    if (int rc = malio_buf::allocate_group(h, st, {{S.d_gmax, nx * ny}, {S.d_gmin, nx * ny}})) return rc;
    CUDA_TRY(cudaMemsetAsync(S.d_gmax, 0, nx * ny * 4, st));
    CUDA_TRY(cudaMemsetAsync(S.d_gmin, 0xFF, nx * ny * 4, st));
    pl_fold_kernel<<<(n_prior + 255) / 256, 256, 0, st>>>(prior, n_prior, a->cell, ilo, jlo, (uint32_t)nx, S.d_gmax, S.d_gmin);
    D->ctr.kernel_launches += 1;
    // the lattice: columns whose indices are multiples of m, inside the box
    const int64_t m = (int64_t)std::llround(a->step / a->cell);
    const int64_t ia = -floor_div(-(int64_t)ilo, m), ib = floor_div(small[3], m);
    const int64_t ja = -floor_div(-(int64_t)jlo, m), jb = floor_div(small[4], m);
    const uint64_t lx = ib >= ia ? (uint64_t)(ib - ia + 1) : 0, ly = jb >= ja ? (uint64_t)(jb - ja + 1) : 0;
    const uint64_t nl = lx * ly;
    if (nl) {
      const uint32_t gi0 = (uint32_t)(ia * m - ilo), gj0 = (uint32_t)(ja * m - jlo);
      if (int rc = malio_buf::allocate_group(h, st, {{S.d_flag, nl + 1}, {S.d_off, nl + 1}})) return rc;
      size_t t = 0;
      uint32_t* un = nullptr;
      CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t, un, un, (int)(nl + 1), st));
      if (int rc = S.d_temp.allocate(h, st, t)) return rc;
      pl_flag_kernel<<<(unsigned)((nl + 1 + 255) / 256), 256, 0, st>>>(S.d_gmax, (uint32_t)nx, gi0, gj0, (uint32_t)m, (uint32_t)lx,
                                                                        (uint32_t)nl, S.d_flag);
      CUDA_TRY(cub::DeviceScan::ExclusiveSum(S.d_temp.data(), t, S.d_flag.data(), S.d_off.data(), (int)(nl + 1), st));
      uint32_t npos = 0;
      CUDA_TRY(cudaMemcpyAsync(&npos, S.d_off + nl, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      D->ctr.kernel_launches += 2;
      D->ctr.d2h_bytes += sizeof(uint32_t);
      const long double dbytes = (long double)npos * r.bytes_per_position;
      if (dbytes > (long double)MALIO_PLACE_MAX_DB_BYTES) {
        h->err = "malio_place_db_build: the database needs " + std::to_string((double)dbytes) + " bytes for " + std::to_string(npos) +
                 " positions (limit MALIO_PLACE_MAX_DB_BYTES): a larger step or fewer bins";
        return MALIO_ERR_CAPACITY;
      }
      if (npos) {
        if (int rc = malio_buf::allocate_group(h, st, {{P.d_cols, npos}, {P.d_zs, npos}, {P.d_nib, (size_t)npos * P.bpp},
                                                       {P.d_rk, (size_t)npos * a->n_ring}}))
          return rc;
        pl_scatter_kernel<<<(unsigned)((nl + 255) / 256), 256, 0, st>>>(S.d_gmin, S.d_off, (uint32_t)nx, ilo, jlo, gi0, gj0, (uint32_t)m,
                                                                         (uint32_t)lx, (uint32_t)nl, a->sensor_height, P.d_cols, P.d_zs);
        const Binning b{P.d_st, P.n_st, a->n_ring, a->n_sector, P.n_bins, a->z_lo, a->dz, a->block_level};
        pl_db_desc_kernel<<<npos, DESC_T, 0, st>>>(b, S.d_gmax, ilo, jlo, (uint32_t)nx, (uint32_t)ny, P.d_cols, P.d_zs, P.bpp, P.d_nib, P.d_rk);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamSynchronize(st));
        D->ctr.kernel_launches += 2;
      }
      P.n = npos;
    }
  }
  r.n_positions = P.n;
  r.device_bytes = P.bytes();
  r.scratch_bytes = S.bytes();
  *rep = r;
  return MALIO_OK;
}

// the resident scan against the database: query descriptor, stages 1-2 (malio_b200.h, steps 4-5); out[0 .. n1) by stage-1 rank
struct QueryScratch {
  DeviceBuffer<unsigned long long> d_qg, d_key, d_sorted;
  DeviceBuffer<uint8_t> d_q;
  DeviceBuffer<uint16_t> d_qk;
  DeviceBuffer<Stage2Out> d_out;
  DeviceBuffer<char> d_temp;
  size_t bytes() const {
    return d_qg.bytes() + d_key.bytes() + d_sorted.bytes() + d_q.bytes() + d_qk.bytes() + d_out.bytes() + d_temp.bytes();
  }
};

int rank(malio_handle* h, DeviceState* D, const PlaceDb& P, const malio_pass_state* s, uint32_t n1, QueryScratch& S, uint8_t* q,
         std::vector<Stage2Out>& out) {
  cudaStream_t st = D->stream;
  const malio_place_args& a = P.args;
  const uint32_t W = 2 * P.R + 1;
  if (int rc = S.d_qg.allocate(h, st, (size_t)W * W)) return rc;
  if (int rc = S.d_q.allocate(h, st, P.n_bins)) return rc;
  if (int rc = S.d_qk.allocate(h, st, a.n_ring)) return rc;
  CUDA_TRY(cudaMemsetAsync(S.d_qg, 0, (size_t)W * W * sizeof(unsigned long long), st));
  malio_pass_state s0 = *s;
  s0.pos[0] = s0.pos[1] = s0.pos[2] = 0.0;
  const PassConst pc = make_pass_const(h, D, &s0);
  if (D->N) {
    pl_query_cols_kernel<<<(D->N + 255) / 256, 256, 0, st>>>(D->d_pts, D->N, pc, a.cell, (int)P.R, S.d_qg);
    D->ctr.kernel_launches += 1;
  }
  const Binning b{P.d_st, P.n_st, a.n_ring, a.n_sector, P.n_bins, a.z_lo, a.dz, a.block_level};
  pl_query_desc_kernel<<<1, DESC_T, 0, st>>>(b, S.d_qg, (int)P.R, S.d_q, S.d_qk);
  D->ctr.kernel_launches += 1;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(q, S.d_q, P.n_bins, cudaMemcpyDeviceToHost, st));
  D->ctr.d2h_bytes += P.n_bins;
  if (n1) {
    const uint32_t np = (uint32_t)P.n;
    if (int rc = malio_buf::allocate_group(h, st, {{S.d_key, np}, {S.d_sorted, np}})) return rc;
    if (int rc = S.d_out.allocate(h, st, n1)) return rc;
    size_t t = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortKeys(nullptr, t, S.d_key.data(), S.d_sorted.data(), (int)np, 0, 64, st));
    if (int rc = S.d_temp.allocate(h, st, t)) return rc;
    pl_stage1_kernel<<<(np + 255) / 256, 256, 0, st>>>(P.d_rk, np, a.n_ring, S.d_qk, S.d_key);
    CUDA_TRY(cub::DeviceRadixSort::SortKeys(S.d_temp.data(), t, S.d_key.data(), S.d_sorted.data(), (int)np, 0, 64, st));
    pl_stage2_kernel<<<n1, ST2_T, 0, st>>>(S.d_sorted, a.n_ring, a.n_sector, S.d_q, P.d_nib, P.bpp, P.d_cols, P.d_zs, S.d_out);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 3;   // stage 1, the sort (counted as one), stage 2
    out.resize(n1);
    CUDA_TRY(cudaMemcpyAsync(out.data(), S.d_out, n1 * sizeof(Stage2Out), cudaMemcpyDeviceToHost, st));
    D->ctr.d2h_bytes += n1 * sizeof(Stage2Out);
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return MALIO_OK;
}

// Eigen's _transformVector, the device's q_rot, on the host
void q_rot_host(const double q[4], const double v[3], double o[3]) {
  const double qv[3] = {q[1], q[2], q[3]};
  double uv[3] = {qv[1] * v[2] - qv[2] * v[1], qv[2] * v[0] - qv[0] * v[2], qv[0] * v[1] - qv[1] * v[0]};
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  const double c2[3] = {qv[1] * uv[2] - qv[2] * uv[1], qv[2] * uv[0] - qv[0] * uv[2], qv[0] * uv[1] - qv[1] * uv[0]};
  o[0] = v[0] + q[0] * uv[0] + c2[0];
  o[1] = v[1] + q[0] * uv[1] + c2[1];
  o[2] = v[2] + q[0] * uv[2] + c2[2];
}

}  // namespace

namespace malio_place {

int PlaceDb::init(malio_handle* h, DeviceState* D, const malio_place_args* a, const float4* prior, uint32_t n_prior,
                  malio_place_db_report* rep) {
  BuildScratch S;
  const int rc = build(h, D, a, prior, n_prior, *this, S, rep);
  CUDA_TRY(cudaStreamSynchronize(D->stream));   // before the scratch goes back
  return rc;
}

int db_build(malio_handle* h, const malio_place_args* a, malio_place_db_report* rep) {
  release(h->place, h->dev->stream);
  if (int rc = check_args(h, a)) return rc;
  const float* prior = nullptr;
  uint32_t n_prior = 0;
  if (malio_prior::points(h, &prior, &n_prior) != MALIO_OK) { h->err = "malio_place_db_build before malio_prior_map_load"; return MALIO_ERR_STATE; }
  PlaceDb* P;
  DeviceState* D;
  return acquire(h, h->place, P, D, a, reinterpret_cast<const float4*>(prior), n_prior, rep);
}

int db_info(malio_handle* h, uint64_t* n_positions, uint64_t* device_bytes) {
  const PlaceDb* P = h->place.get();
  if (n_positions) *n_positions = P ? P->n : 0;
  if (device_bytes) *device_bytes = P ? P->bytes() : 0;
  return MALIO_OK;
}

int db_download(malio_handle* h, int32_t* cols, double* z_s, uint8_t* nib, uint16_t* rk, uint64_t cap, uint64_t* n) {
  const PlaceDb* P = h->place.get();
  if (!P) { h->err = "malio_place_db_download before malio_place_db_build"; return MALIO_ERR_STATE; }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  *n = P->n;
  const uint64_t m = cap < P->n ? cap : P->n;
  if (m) {
    cudaStream_t st = D->stream;
    if (cols) CUDA_TRY(cudaMemcpyAsync(cols, P->d_cols, m * sizeof(int2), cudaMemcpyDeviceToHost, st));
    if (z_s) CUDA_TRY(cudaMemcpyAsync(z_s, P->d_zs, m * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (nib) CUDA_TRY(cudaMemcpyAsync(nib, P->d_nib, m * P->bpp, cudaMemcpyDeviceToHost, st));
    if (rk) CUDA_TRY(cudaMemcpyAsync(rk, P->d_rk, m * P->args.n_ring * sizeof(uint16_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
  }
  return MALIO_OK;
}

int relocalize_global(malio_handle* h, const malio_pass_state* s, const malio_global_args* a, malio_global_report* rep) {
  bool finite = std::isfinite(a->yaw_step) && a->yaw_step > 0.0;
  for (int i = 0; i < 4; ++i) finite = finite && std::isfinite(s->rot[i]);
  if (a->k1 == 0 || a->k1 > MALIO_PLACE_MAX_K1 || a->k2 == 0 || a->k2 > a->k1 || a->k2 > MALIO_PLACE_MAX_K2 || !finite) {
    h->err = "malio_relocalize_global: 0 < k2 <= k1, k1 <= MALIO_PLACE_MAX_K1, k2 <= MALIO_PLACE_MAX_K2, yaw_step finite and > 0, "
             "s.rot finite";
    return MALIO_ERR_INVALID_ARG;
  }
  DeviceState* D = h->dev.get();
  const float* prior = nullptr;
  uint32_t n_prior = 0;
  if (malio_prior::points(h, &prior, &n_prior) != MALIO_OK) { h->err = "malio_relocalize_global before malio_prior_map_load"; return MALIO_ERR_STATE; }
  const PlaceDb* P = h->place.get();
  if (!P) { h->err = "malio_relocalize_global before malio_place_db_build"; return MALIO_ERR_STATE; }
  if (!D->scan_ready) { h->err = "malio_relocalize_global before a scan upload"; return MALIO_ERR_STATE; }
  if (D->comm) { h->err = "malio_relocalize_global: a communicator is attached (each rank holds only its block of the scan)"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t S = P->args.n_sector;
  std::unique_ptr<malio_global_report> r(new malio_global_report{});   // (off the stack); written to *rep only on success
  r->verify.res = a->res;
  r->verify.half_xy = a->half_xy;
  r->verify.half_z = a->half_z;
  r->verify.yaw_step = a->yaw_step;
  const double win = 1.5 * (2.0 * M_PI / (double)S);
  const double nh = std::ceil(win / a->yaw_step);
  r->verify.n_yaw = nh < 1e6 ? 2u * (uint32_t)nh + 1u : 0u;   // 0: refused by malio_relocalize below
  r->verify.yaw_lo = -(double)(r->verify.n_yaw / 2) * a->yaw_step;
  r->n_stage1 = (uint32_t)std::min<uint64_t>(a->k1, P->n);
  r->n_candidates = std::min<uint32_t>(a->k2, r->n_stage1);
  std::vector<Stage2Out> out;
  const auto t0 = std::chrono::steady_clock::now();
  int rc;
  size_t peak;
  {
    QueryScratch Q;
    rc = rank(h, D, *P, s, r->n_stage1, Q, r->query, out);
    peak = Q.bytes();
    CUDA_TRY(cudaStreamSynchronize(D->stream));
  }
  const auto t1 = std::chrono::steady_clock::now();
  if (rc) return rc;
  for (uint32_t t = 0; t < r->n_stage1; ++t) { r->stage1[t] = out[t].p; r->stage1_d1[t] = out[t].d1; }
  std::sort(out.begin(), out.end(), [](const Stage2Out& x, const Stage2Out& y) { return x.d2 != y.d2 ? x.d2 < y.d2 : x.p < y.p; });
  std::memcpy(r->rot, s->rot, sizeof(r->rot));
  std::memcpy(r->pos, s->pos, sizeof(r->pos));
  bool have = false;
  for (uint32_t k = 0; k < r->n_candidates; ++k) {
    const Stage2Out& o = out[k];
    malio_global_candidate& c = r->cand[k];
    c.position = o.p; c.shift = o.shift; c.d1 = o.d1; c.d2 = o.d2; c.col[0] = o.i; c.col[1] = o.j; c.z_s = o.z_s;
    // the guess: rot = q_yaw(theta) (x) s.rot (malio_relocalize's product), the slot-0 origin at the position's sensor
    const double theta = 2.0 * M_PI * (double)o.shift / (double)S;
    const double cth = std::cos(theta / 2.0), sth = std::sin(theta / 2.0);
    const double w0 = s->rot[0], x0 = s->rot[1], y0 = s->rot[2], z0 = s->rot[3];
    malio_pass_state g = *s;
    g.rot[0] = cth * w0 - sth * z0;
    g.rot[1] = cth * x0 - sth * y0;
    g.rot[2] = cth * y0 + sth * x0;
    g.rot[3] = cth * z0 + sth * w0;
    double e[3];
    q_rot_host(g.rot, s->ext[0].t, e);
    const double target[3] = {((double)o.i + 0.5) * P->args.cell, ((double)o.j + 0.5) * P->args.cell, o.z_s};
    for (int i = 0; i < 3; ++i) g.pos[i] = target[i] - e[i];
    std::memcpy(c.guess_rot, g.rot, sizeof(c.guess_rot));
    std::memcpy(c.guess_pos, g.pos, sizeof(c.guess_pos));
    malio_reloc_report rr{};
    rc = malio_reloc::relocalize(h, &g, &r->verify, &rr);
    if (rc) return rc;
    std::memcpy(c.rot, rr.rot, sizeof(c.rot));
    std::memcpy(c.pos, rr.pos, sizeof(c.pos));
    c.score = rr.score;
    c.n_points = rr.n_points;
    peak = std::max<size_t>(peak, rr.device_bytes);
    if (!have || rr.score > r->score) {
      have = true;
      r->best_rank = k;
      r->score = rr.score;
      r->n_points = rr.n_points;
      std::memcpy(r->rot, rr.rot, sizeof(r->rot));
      std::memcpy(r->pos, rr.pos, sizeof(r->pos));
    }
  }
  const auto t2 = std::chrono::steady_clock::now();
  r->ms_rank = std::chrono::duration<double, std::milli>(t1 - t0).count();
  r->ms_verify = std::chrono::duration<double, std::milli>(t2 - t1).count();
  r->device_bytes = peak;
  *rep = *r;
  return MALIO_OK;
}

}  // namespace malio_place

// relocalization without a position guess (malio_b200.h, after malio_relocalize)
extern "C" int malio_place_db_build(malio_handle* h, const malio_place_args* a, malio_place_db_report* rep) {
  if (!h || !a || !rep) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_place::db_build(h, a, rep);
}
extern "C" int malio_place_db_info(malio_handle* h, uint64_t* n_positions, uint64_t* device_bytes) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_place::db_info(h, n_positions, device_bytes);
}
extern "C" int malio_place_db_download(malio_handle* h, int32_t* cols, double* z_s, uint8_t* nibbles, uint16_t* ring_keys, uint64_t cap,
                                       uint64_t* n) {
  if (!h || !n) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_place::db_download(h, cols, z_s, nibbles, ring_keys, cap, n);
}
extern "C" int malio_relocalize_global(malio_handle* h, const malio_pass_state* s, const malio_global_args* a, malio_global_report* rep) {
  if (!h || !s || !a || !rep) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_place::relocalize_global(h, s, a, rep);
}
