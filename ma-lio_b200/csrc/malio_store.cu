// malio_store.cu — the session's dense scans kept on the device, sm_90a, so that the voxel map can be rebuilt later under
// corrected states, another leaf or other carve settings (malio_world_voxel_rebuild in malio_voxmap.cu folds them again).
// Per scan: the rows malio_world_accumulate registers (slots 0..L-1 in slot order, each in its buffer order) as {x, y, z} in
// the LiDAR frame, 12 B a point, bits unchanged, in device blocks of MALIO_STORE_BLOCK_POINTS points that a scan never
// crosses; and a host record (malio_stored_scan) with everything the registration reads besides the points: the state, the
// temporal compensation of the last scan upload and the slot tags.
//   st_pack_kernel      the undistorted 20-byte rows of the slots -> 12-byte rows of a block (malio_scan_store_add)
//   st_register_kernel  a stored scan through body_to_world: the bits world_kernel gives for it (malio_scan_store_register_device)
#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <vector>

#include "malio_device.cuh"

using namespace malio_devstate;

namespace malio_store {

struct Block {
  DeviceBuffer<float> xyz;   // capacity x 3 floats
  uint64_t used = 0;         // points stored
};
struct Stored {
  malio_stored_scan rec;
  uint32_t block;
  uint64_t row, rows;        // first point in the block, points
};

struct StoreState {
  std::vector<Block> blocks;   // grown by appending: a block is never copied or moved on the device
  std::vector<Stored> scans;
  uint64_t points = 0;
  int init(malio_handle*, DeviceState*) { return MALIO_OK; }
};

}  // namespace malio_store

namespace {

using malio_store::Block;
using malio_store::StoreState;
using malio_store::Stored;

constexpr uint64_t MAX_SCAN_POINTS = 0x7FFFFFFFull;   // one scan's rows are indexed by uint32 in the fold

// the slots of one scan: slot of point p is the l with first[l] <= p < first[l + 1]
struct Slots {
  const float* ud[MALIO_MAX_LIDAR];   // the undistorted n x 5 rows (st_pack_kernel only)
  float tag[MALIO_MAX_LIDAR];
  uint32_t first[MALIO_MAX_LIDAR + 1];
  int L;
};
__device__ __forceinline__ int slot_of(const Slots& c, uint32_t p) {
  int l = 0;
  while (l + 1 < c.L && p >= c.first[l + 1]) ++l;
  return l;
}

__global__ void __launch_bounds__(256) st_pack_kernel(Slots c, uint32_t n, float* __restrict__ out) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n) return;
  const int l = slot_of(c, p);
  const float* r = c.ud[l] + 5 * (size_t)(p - c.first[l]);
  float* o = out + 3 * (size_t)p;
  o[0] = r[0]; o[1] = r[1]; o[2] = r[2];
}

__global__ void __launch_bounds__(256) st_register_kernel(const float* __restrict__ xyz, Slots c, PassConst pc, uint32_t n,
                                                          float4* __restrict__ out) {
  const uint32_t p = blockIdx.x * 256u + threadIdx.x;
  if (p >= n) return;
  const int l = slot_of(c, p);
  const float* r = xyz + 3 * (size_t)p;
  float w[3];
  body_to_world(pc, l, r[0], r[1], r[2], w);
  out[p] = make_float4(w[0], w[1], w[2], c.tag[l]);
}

// where n more points go: the last block when they fit, else a new block of max(n, MALIO_STORE_BLOCK_POINTS) points (nothing
// is copied; a failed allocation leaves the store as it was)
int room(malio_handle* h, StoreState* S, uint64_t n, uint32_t* block, uint64_t* row) {
  if (!S->blocks.empty()) {
    const Block& b = S->blocks.back();
    if (n == 0 || b.used + n <= b.xyz.size() / 3) {
      *block = (uint32_t)(S->blocks.size() - 1);
      *row = b.used;
      return MALIO_OK;
    }
  } else if (n == 0) {
    *block = 0;
    *row = 0;
    return MALIO_OK;
  }
  const uint64_t cap = n > MALIO_STORE_BLOCK_POINTS ? n : MALIO_STORE_BLOCK_POINTS;
  Block b;
  if (const cudaError_t e = b.xyz.allocate_empty(cap * 3 * sizeof(float))) {
    cudaGetLastError();
    h->err = std::string("scan store: cannot allocate a block of ") + std::to_string(cap) + " points: " + cudaGetErrorString(e);
    return MALIO_ERR_CUDA;
  }
  S->blocks.push_back(std::move(b));
  *block = (uint32_t)(S->blocks.size() - 1);
  *row = 0;
  return MALIO_OK;
}

// the record's scan in its block: n points from `row` on
void append(StoreState* S, const malio_stored_scan& rec, uint32_t block, uint64_t row, uint64_t n) {
  if (n) S->blocks[block].used = row + n;
  S->scans.push_back(Stored{rec, block, row, n});
  S->points += n;
}

Slots slots_of(const malio_stored_scan& rec, int L) {
  Slots c{};
  c.L = L;
  uint32_t at = 0;
  for (int l = 0; l < L; ++l) { c.tag[l] = rec.slot_tag[l]; c.first[l] = at; at += rec.n_points[l]; }
  c.first[L] = at;
  return c;
}

}  // namespace

namespace malio_store {

uint64_t count(const malio_handle* h) { return h->store ? h->store->scans.size() : 0; }

View view(const malio_handle* h, uint64_t k) {
  const Stored& s = h->store->scans[k];
  const float* base = s.rows ? h->store->blocks[s.block].xyz.data() + 3 * s.row : nullptr;
  return View{&s.rec, base, s.rows, s.block};
}

int add(malio_handle* h, const malio_pass_state* s, const float* slot_tag, double time, uint64_t* n_scans) {
  StoreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->store, S, D)) return rc;
  const int L = h->cfg.params.n_lidar;
  const float* ud[MALIO_MAX_LIDAR] = {nullptr, nullptr, nullptr};
  uint32_t m[MALIO_MAX_LIDAR] = {0, 0, 0};
  if (int rc = malio_pre::world_dense_source(h, ud, m)) return rc;
  malio_stored_scan rec{};
  rec.time = time;
  rec.state = *s;
  for (int l = 1; l < MALIO_MAX_LIDAR; ++l) rec.temporal_comp[l - 1] = D->tcomp[l];
  uint64_t n = 0;
  for (int l = 0; l < L; ++l) { rec.slot_tag[l] = slot_tag[l]; rec.n_points[l] = m[l]; n += m[l]; }
  if (n > MAX_SCAN_POINTS) { h->err = "scan store: more than 2^31 - 1 points in one scan"; return MALIO_ERR_CAPACITY; }
  uint32_t block = 0;
  uint64_t row = 0;
  if (int rc = room(h, S, n, &block, &row)) return rc;
  if (n) {
    Slots c = slots_of(rec, L);
    for (int l = 0; l < L; ++l) c.ud[l] = ud[l];
    const uint32_t nn = (uint32_t)n;
    st_pack_kernel<<<(nn + 255) / 256, 256, 0, D->stream>>>(c, nn, S->blocks[block].xyz + 3 * row);
    CUDA_TRY(cudaGetLastError());
    D->ctr.kernel_launches += 1;
  }
  append(S, rec, block, row, n);
  if (n_scans) *n_scans = S->scans.size();
  return MALIO_OK;
}

int put(malio_handle* h, const malio_stored_scan* rec, const float* xyz, uint64_t* n_scans) {
  StoreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->store, S, D)) return rc;
  const int L = h->cfg.params.n_lidar;
  uint64_t n = 0;
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
    if (l >= L && rec->n_points[l]) { h->err = "scan store put: n_points must be 0 beyond the handle's L"; return MALIO_ERR_INVALID_ARG; }
    n += rec->n_points[l];
  }
  if (n > MAX_SCAN_POINTS) { h->err = "scan store put: more than 2^31 - 1 points in one scan"; return MALIO_ERR_INVALID_ARG; }
  if (n && !xyz) { h->err = "scan store put: xyz is NULL for a scan with points"; return MALIO_ERR_INVALID_ARG; }
  uint32_t block = 0;
  uint64_t row = 0;
  if (int rc = room(h, S, n, &block, &row)) return rc;
  if (n) {
    const size_t bytes = (size_t)n * 3 * sizeof(float);
    CUDA_TRY(cudaMemcpyAsync(S->blocks[block].xyz + 3 * row, xyz, bytes, cudaMemcpyHostToDevice, D->stream));
    CUDA_TRY(cudaStreamSynchronize(D->stream));   // the caller may reuse xyz once the call returns
    D->ctr.h2d_bytes += bytes;
  }
  append(S, *rec, block, row, n);
  if (n_scans) *n_scans = S->scans.size();
  return MALIO_OK;
}

int get(malio_handle* h, uint64_t k, malio_stored_scan* rec, float* xyz, uint64_t cap, uint64_t* n_out) {
  StoreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->store, S, D)) return rc;
  if (k >= S->scans.size()) {
    h->err = "scan store get: scan " + std::to_string(k) + " beyond the store (" + std::to_string(S->scans.size()) + " scans)";
    return MALIO_ERR_INVALID_ARG;
  }
  const View v = view(h, k);
  *n_out = v.rows;
  if (xyz && cap < v.rows) {
    h->err = "scan store get: cap " + std::to_string(cap) + " below the scan's " + std::to_string(v.rows) + " points (nothing read)";
    return MALIO_ERR_CAPACITY;
  }
  if (rec) *rec = *v.rec;
  if (!xyz || v.rows == 0) return MALIO_OK;
  const size_t bytes = (size_t)v.rows * 3 * sizeof(float);
  CUDA_TRY(cudaMemcpyAsync(xyz, v.xyz, bytes, cudaMemcpyDeviceToHost, D->stream));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  D->ctr.d2h_bytes += bytes;
  return MALIO_OK;
}

int register_device(malio_handle* h, uint64_t k, const malio_pass_state* s, float* out, uint64_t cap, uint64_t* n_out,
                    cudaStream_t caller) {
  StoreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->store, S, D)) return rc;
  if (k >= S->scans.size()) {
    h->err = "scan store register: scan " + std::to_string(k) + " beyond the store (" + std::to_string(S->scans.size()) + " scans)";
    return MALIO_ERR_INVALID_ARG;
  }
  const View v = view(h, k);
  const uint64_t kk = v.rows < cap ? v.rows : cap;
  if (out && kk) {
    if (int rc = check_device_ptr(h, D, out, "malio_scan_store_register_device out", 16, "the points are stored as float4")) return rc;
  }
  *n_out = v.rows;
  if (!out || kk == 0) return MALIO_OK;
  if (int rc = caller_enter(h, D, caller)) return rc;
  if (int rc = enqueue_register(h, k, s, kk, out)) return rc;
  return caller_leave(h, D, caller);
}

int enqueue_register(malio_handle* h, uint64_t k, const malio_pass_state* s, uint64_t n, float* out) {
  DeviceState* D = h->dev.get();
  const View v = view(h, k);
  if (n == 0) return MALIO_OK;
  malio_rigid tc[MALIO_MAX_LIDAR];
  tc[0] = D->tcomp[0];
  for (int l = 1; l < MALIO_MAX_LIDAR; ++l) tc[l] = v.rec->temporal_comp[l - 1];
  const PassConst pc = make_pass_const(h, D, s ? s : &v.rec->state, tc);
  const uint32_t nn = (uint32_t)n;
  st_register_kernel<<<(nn + 255) / 256, 256, 0, D->stream>>>(v.xyz, slots_of(*v.rec, h->cfg.params.n_lidar), pc, nn,
                                                             reinterpret_cast<float4*>(out));
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

int info(malio_handle* h, uint64_t* n_scans, uint64_t* n_points, uint64_t* device_bytes) {
  const StoreState* S = h->store.get();
  uint64_t bytes = 0;
  if (S)
    for (const Block& b : S->blocks) bytes += b.xyz.bytes();
  if (n_scans) *n_scans = S ? S->scans.size() : 0;
  if (n_points) *n_points = S ? S->points : 0;
  if (device_bytes) *device_bytes = bytes;
  return MALIO_OK;
}

}  // namespace malio_store

// the scan store (malio_b200.h, next to malio_world_voxel_rebuild)
extern "C" int malio_scan_store_add(malio_handle* h, const malio_pass_state* s, const float* slot_tag, double time, uint64_t* n_scans) {
  if (!h || !s) return MALIO_ERR_INVALID_ARG;
  if (!slot_tag) { h->err = "scan store add: the dense cloud needs slot_tag"; return MALIO_ERR_INVALID_ARG; }
  MALIO_SETTLE(h);
  return malio_store::add(h, s, slot_tag, time, n_scans);
}
extern "C" int malio_scan_store_put(malio_handle* h, const malio_stored_scan* rec, const float* xyz, uint64_t* n_scans) {
  if (!h || !rec) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_store::put(h, rec, xyz, n_scans);
}
extern "C" int malio_scan_store_get(malio_handle* h, uint64_t k, malio_stored_scan* rec, float* xyz, uint64_t cap, uint64_t* n_out) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!n_out || (cap && !xyz)) return MALIO_ERR_INVALID_ARG;
  return malio_store::get(h, k, rec, xyz, cap, n_out);
}
extern "C" int malio_scan_store_register_device(malio_handle* h, uint64_t k, const malio_pass_state* s, float* d_out, uint64_t cap,
                                                uint64_t* n_out, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!n_out || (cap && !d_out)) return MALIO_ERR_INVALID_ARG;
  return malio_store::register_device(h, k, s, d_out, cap, n_out, (cudaStream_t)stream);
}
extern "C" int malio_scan_store_info(malio_handle* h, uint64_t* n_scans, uint64_t* n_points, uint64_t* device_bytes) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_store::info(h, n_scans, n_points, device_bytes);
}
extern "C" int malio_scan_store_clear(malio_handle* h) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  CUDA_TRY(malio_buf::release(h->store, D->stream));   // a register_device may still read the blocks
  return MALIO_OK;
}
