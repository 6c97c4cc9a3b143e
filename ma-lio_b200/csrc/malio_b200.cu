// malio_b200.cu — handle lifecycle and per-scan data movement of libmalio_b200.so, sm_90a: create / destroy, the scan
// upload (from host or device memory) and its per-scan reset, the downloads in caller order (to host or device memory),
// stand-alone k-NN queries from host or device memory (the search itself is in malio_knn.cu) and map_incremental's per-point
// decision.  The measurement pass is in malio_pass.cu.
// Compiled with -fmad=false like the rest of the library (bit parity with the reference's non-FMA x86-64 build).
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "malio_internal.h"
#include "malio_device.cuh"

using namespace malio_devstate;
namespace {

// per-scan state back to "nothing searched yet": point_selected_surf = 0, normal_y = 0, Nearest_Points empty, k-NN list
// counters 0 — one launch instead of four memsets (this sits at the head of every scan)
__global__ void reset_scan_kernel(uint32_t cap, uint8_t* __restrict__ sel, float* __restrict__ normal_y,
                                  uint32_t* __restrict__ nn_idx, uint32_t* __restrict__ gstats) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 4) gstats[2 + i] = 0;
  if (i < cap) {
    sel[i] = 0;
    normal_y[i] = 0.f;
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) nn_idx[(size_t)j * cap + i] = 0xFFFFFFFFu;
  }
}
// ------------------------------------------------------------------ next to the path: map_incremental's decision
// laserMapping.cpp:398-446 per point, from device-resident data: normal_y and Nearest_Points (indices into the snapshot)
// of the last pass, the scan point and the state after the update.  pointBodyToWorld (:134-147) has its own operation
// order (no detour through the LiDAR-0 frame), restated exactly by body_to_world (malio_device.cuh).  Outputs in caller order.
__global__ void map_incr_kernel(const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm, uint32_t N,
                                PassConst pc, const float4* __restrict__ mpts, const uint32_t* __restrict__ nn_idx,
                                const float* __restrict__ normal_y, double cov_threshold, double fs, int ekf_inited,
                                uint8_t* __restrict__ cls_out, float* __restrict__ world_out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const uint32_t i = perm ? perm[p] : p;
  uint8_t cls = MALIO_MAP_SKIP;
  float w[3] = {0.f, 0.f, 0.f};
  if (!((double)normal_y[p] > cov_threshold)) {                                                 // :406
    const malio_scan_pt pt = pts[p];
    body_to_world(pc, pt.lidar, pt.x, pt.y, pt.z, w);                                           // :134-147
    uint32_t id[MALIO_K];
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) { id[j] = nn_idx[(size_t)j * N + p]; cnt += id[j] != 0xFFFFFFFFu; }
    if (cnt > 0 && ekf_inited) {                                                                // :411
      float mid[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) mid[k] = (float)(floor((double)w[k] / fs) * fs + 0.5 * fs);   // :417-419
      const float dist = (w[0] - mid[0]) * (w[0] - mid[0]) + (w[1] - mid[1]) * (w[1] - mid[1]) + (w[2] - mid[2]) * (w[2] - mid[2]);
      const float4 n0 = __ldg(mpts + id[0]);
      if ((double)fabsf(n0.x - mid[0]) > 0.5 * fs && (double)fabsf(n0.y - mid[1]) > 0.5 * fs && (double)fabsf(n0.z - mid[2]) > 0.5 * fs) {
        cls = MALIO_MAP_ADD_NO_DOWNSAMPLE;                                                      // :421-425
      } else {
        bool need_add = true;
        if (cnt >= MALIO_K) {                                                                   // :428-429
#pragma unroll
          for (int j = 0; j < MALIO_K; ++j) {
            const float4 q = __ldg(mpts + id[j]);
            const float dj = (q.x - mid[0]) * (q.x - mid[0]) + (q.y - mid[1]) * (q.y - mid[1]) + (q.z - mid[2]) * (q.z - mid[2]);
            if (need_add && dj < dist) need_add = false;                                        // :430-434
          }
        }
        cls = need_add ? MALIO_MAP_ADD : MALIO_MAP_DROP;
      }
    } else {
      cls = MALIO_MAP_ADD;                                                                      // :439-440
    }
  }
  cls_out[i] = cls;
  if (world_out) { world_out[3 * (size_t)i] = w[0]; world_out[3 * (size_t)i + 1] = w[1]; world_out[3 * (size_t)i + 2] = w[2]; }
}

// position space -> caller order
__global__ void scatter_aux_kernel(const uint32_t* __restrict__ perm, uint32_t N, const float* __restrict__ normal_y,
                                   const uint32_t* __restrict__ nn_idx, const float* __restrict__ nn_d2,
                                   const uint8_t* __restrict__ sel, const float4* __restrict__ world,
                                   float* __restrict__ o_ny, uint32_t* __restrict__ o_idx, float* __restrict__ o_d2,
                                   uint8_t* __restrict__ o_sel, float* __restrict__ o_world) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const uint32_t i = perm ? perm[p] : p;
  if (o_ny) o_ny[i] = normal_y[p];
  if (o_sel) o_sel[i] = sel[p];
  if (o_world) { const float4 w = world[p]; o_world[3 * (size_t)i] = w.x; o_world[3 * (size_t)i + 1] = w.y; o_world[3 * (size_t)i + 2] = w.z; }
  if (o_idx) {
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) o_idx[(size_t)i * MALIO_K + j] = nn_idx[(size_t)j * N + p];
  }
  if (o_d2) {
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) o_d2[(size_t)i * MALIO_K + j] = nn_d2[(size_t)j * N + p];
  }
}

// malio_upload_scan_from_device's record check, upload_scan's host sweep on device memory: word 3 of a malio_scan_pt is
// lidar | table_idx << 16, and lidar must be < L.  A warp with a bad record ORs 1 into *bad.  The records are read as words:
// the caller's buffer need only be 4-byte aligned.
__global__ void scan_lidar_check_kernel(const uint32_t* __restrict__ words, uint32_t n, uint32_t L, uint32_t* __restrict__ bad) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool b = i < n && (words[4 * (size_t)i + 3] & 0xFFFFu) >= L;
  if (__any_sync(0xFFFFFFFFu, b) && (threadIdx.x & 31u) == 0) atomicOr(bad, 1u);
}

}  // namespace

// ------------------------------------------------------------------ device-memory entry points
namespace malio_devstate {
int check_device_ptr(malio_handle* h, const DeviceState* D, const void* p, const char* what) {
  if (!p) { h->err = std::string(what) + ": NULL"; return MALIO_ERR_INVALID_ARG; }
  if (reinterpret_cast<uintptr_t>(p) & 3u) { h->err = std::string(what) + ": not 4-byte aligned"; return MALIO_ERR_INVALID_ARG; }
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();   // not sticky: clear it so that it does not surface in a later call
    h->err = std::string(what) + ": not a CUDA pointer";
    return MALIO_ERR_INVALID_ARG;
  }
  if (a.type == cudaMemoryTypeManaged) { h->err = std::string(what) + ": managed memory is not accepted (use cudaMalloc'ed memory)"; return MALIO_ERR_INVALID_ARG; }
  if (a.type != cudaMemoryTypeDevice) { h->err = std::string(what) + ": host memory (the *_device calls take device memory)"; return MALIO_ERR_INVALID_ARG; }
  if (a.device != D->device) { h->err = std::string(what) + ": memory of another device than the handle's"; return MALIO_ERR_INVALID_ARG; }
  return MALIO_OK;
}
int check_device_ptrs(malio_handle* h, const DeviceState* D, std::initializer_list<DevicePtrArg> args) {
  for (const DevicePtrArg& a : args)
    if (a.p) { if (int rc = check_device_ptr(h, D, a.p, a.what)) return rc; }
  return MALIO_OK;
}

int caller_enter(malio_handle* h, DeviceState* D, cudaStream_t caller) {
  CUDA_TRY(cudaEventRecord(D->ev_caller_in, caller));
  CUDA_TRY(cudaStreamWaitEvent(D->stream, D->ev_caller_in, 0));
  return MALIO_OK;
}
int caller_leave(malio_handle* h, DeviceState* D, cudaStream_t caller) {
  CUDA_TRY(cudaEventRecord(D->ev_caller_out, D->stream));
  CUDA_TRY(cudaStreamWaitEvent(caller, D->ev_caller_out, 0));
  return MALIO_OK;
}
}  // namespace malio_devstate

namespace {
// h->deferred of malio_knn_device: wait for its statistics, fold the fast-path counters in, report a traversal fault
int settle_knn_device(malio_handle* h) {
  DeviceState* D = h->dev.get();
  h->deferred = nullptr;
  CUDA_TRY(cudaSetDevice(D->device));
  CUDA_TRY(cudaEventSynchronize(D->ev_deferred));
  if (D->deferred_grid) { D->ctr.knn_fallback_queries += D->h_gstats[3]; D->ctr.knn_ring2_queries += D->h_gstats[5]; }
  return knn_fault(h, D);
}
}  // namespace

namespace malio_dev {

int create(malio_handle* h) {
  h->dev = malio_owner<DeviceState>(new DeviceState);   // a state left half-built by a failure below goes through destroy()
  DeviceState* D = h->dev.get();
  D->device = h->cfg.device;
  int ndev = 0;
  CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (ndev <= 0 || D->device >= ndev) { h->err = "no such CUDA device"; return MALIO_ERR_CUDA; }
  CUDA_TRY(cudaSetDevice(D->device));
  cudaDeviceProp prop{};
  CUDA_TRY(cudaGetDeviceProperties(&prop, D->device));
  D->sm_count = prop.multiProcessorCount;
  CUDA_TRY(cudaStreamCreateWithFlags(&D->stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&D->stream2, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&D->stream3, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_h2d, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_refit, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_cov, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_sorted, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_tau, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_caller_in, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_caller_out, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_deferred, cudaEventDisableTiming));
  for (auto& e : D->ev) CUDA_TRY(cudaEventCreate(&e));
  const cudaStream_t st = D->stream;
  if (int rc = D->d_counters.allocate(h, st, 4)) return rc;
  CUDA_TRY(cudaMemset(D->d_counters, 0, 4 * sizeof(uint32_t)));
  if (int rc = D->d_mmkey.allocate(h, st, 8)) return rc;
  {
    const unsigned long long init[8] = {dkey(1000.0), dkey(-0.0), dkey(9999.0), dkey(-0.0), dkey(1000.0), dkey(-0.0), dkey(9999.0), dkey(-0.0)};
    CUDA_TRY(cudaMemcpy(D->d_mmkey, init, sizeof(init), cudaMemcpyHostToDevice));
  }
  if (int rc = D->d_res.allocate(h, st, MALIO_RED_DOUBLES)) return rc;
  if (int rc = D->d_cand.allocate(h, st, 4)) return rc;   // [0] candidates, [1..3] multi-GPU exchange waits (ns, ns, passes)
  CUDA_TRY(cudaMemset(D->d_cand, 0, 4 * sizeof(unsigned long long)));
  if (int rc = D->d_gstats.allocate(h, st, 8)) return rc;
  CUDA_TRY(cudaMemset(D->d_gstats, 0, 8 * sizeof(uint32_t)));
  if (int rc = D->d_hist.allocate(h, st, SORT_BINS)) return rc;
  if (int rc = D->d_offs.allocate(h, st, SORT_BINS)) return rc;
  if (int rc = D->d_cursor.allocate(h, st, SORT_BINS)) return rc;
  if (int rc = D->d_btot.allocate(h, st, SCAN_BLOCKS)) return rc;
  CUDA_TRY(cudaMemset(D->d_hist, 0, SORT_BINS * sizeof(uint32_t)));
  if (int rc = D->d_rows.allocate(h, st, (size_t)ROWS_DOUBLES * (1 + MAIL_MAX_WORLD))) return rc;   // own rows | gathered rows of all ranks
  // pinned + mapped: [0, RED) result | +0..3 min/max keys | +4..7 k-NN list statistics | +8 pass sequence flag | +16.. rows
  if (int rc = D->h_res.allocate(h, MALIO_RED_DOUBLES + 16 + MALIO_MAX_DOF * 25, cudaHostAllocMapped)) return rc;
  std::memset(D->h_res, 0, (MALIO_RED_DOUBLES + 16) * sizeof(double));
  CUDA_TRY(cudaHostGetDevicePointer((void**)&D->h_res_dev, D->h_res.data(), 0));
  D->h_gstats = reinterpret_cast<uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 4);
  std::memset(D->h_gstats, 0, 8 * sizeof(uint32_t));
  if (int rc = pass_init(h, D)) return rc;
  if (const char* e = getenv("MALIO_KNN_CELL")) { D->env_knn_cell = (float)atof(e); D->env_knn_cell_set = true; }
  D->host_prof = getenv("MALIO_HOST_PROF") != nullptr;
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) { D->tcomp[l] = malio_rigid{{1, 0, 0, 0}, {0, 0, 0}}; }
  return MALIO_OK;
}

void destroy(malio_handle* h) {
  DeviceState* D = h->dev.get();
  if (!D) return;
  cudaSetDevice(D->device);
  if (D->stream) cudaStreamSynchronize(D->stream);   // an enqueued call (malio_knn_device) may still use the buffers below
  h->deferred = nullptr;
  release(h->pre, D->stream);
  release(h->voxmap, D->stream);
  release(h->place, D->stream);
  release(h->prior, D->stream);
  release(h->mapst, D->stream);
  if (D->host_prof && D->host_passes)
    fprintf(stderr, "[malio] passes %llu: host launch %.1f us/pass, host wait-for-device %.1f us/pass\n",
            (unsigned long long)D->host_passes, D->host_launch_us / D->host_passes, D->host_wait_us / D->host_passes);
  comm_destroy(D);
  release(h->dev, D->stream);
}

static int ensure_point_buffers(malio_handle* h, DeviceState* D, uint32_t n) {
  if (n <= D->d_pts.size()) return MALIO_OK;
  uint32_t cap = n + n / 8 + 1024;
  if (cap < h->cfg.max_points) cap = h->cfg.max_points;
  const size_t capK = (size_t)cap * MALIO_K;
  return malio_buf::allocate_group(h, D->stream, {{D->d_pts, cap}, {D->d_pts_sorted, cap}, {D->d_perm, cap}, {D->d_keys16, cap},
                                                  {D->d_tmp_ids, cap}, {D->d_nn_idx, capK}, {D->d_nn_d2, capK}, {D->d_sel, cap},
                                                  {D->d_world, cap}, {D->d_plane, cap}, {D->d_ucov, cap}, {D->d_tau, cap},
                                                  {D->d_tau2, cap}, {D->d_pd2, cap}, {D->d_rows12, (size_t)cap * 12}, {D->d_lid8, cap},
                                                  {D->d_normal_y, cap}, {D->d_o_ny, cap}, {D->d_o_idx, capK}, {D->d_o_d2, capK},
                                                  {D->d_o_sel, cap}, {D->d_o_world, (size_t)cap * 3}, {D->d_fb_list, cap}});
}

int upload_scan_from(malio_handle* h, ScanSource from, const malio_scan_pt* pts, uint32_t n, const malio_pose_entry* table,
                     cudaMemcpyKind table_kind, const uint32_t* table_off, const malio_rigid* tcomp, cudaStream_t caller) {
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  const int L = h->cfg.params.n_lidar;
  for (int l = 0; l < L; ++l)
    if (table_off[l + 1] < table_off[l] + 2) { h->err = "pose table of each LiDAR needs >= 2 entries"; return MALIO_ERR_INVALID_ARG; }
  const bool on_device = from == SCAN_DEVICE && n > 0;   // no record to read: nothing on `caller`
  // pt.lidar indexes per-LiDAR tables on the device: reject ids outside [0, L) before anything changes
  if (from == SCAN_HOST) {   // one vectorisable sweep
    uint32_t bad = 0;
    for (uint32_t i = 0; i < n; ++i) bad |= (uint32_t)(pts[i].lidar >= (uint16_t)L);
    if (bad) { h->err = "scan point with lidar id >= n_lidar"; return MALIO_ERR_INVALID_ARG; }
  } else if (on_device) {
    if (int rc = check_device_ptr(h, D, pts, "malio_upload_scan_from_device pts")) return rc;
    if (!D->d_scan_check) { if (int rc = D->d_scan_check.allocate(h, D->stream, 1)) return rc; }
    if (!D->h_scan_check) { if (int rc = D->h_scan_check.allocate(h, 1)) return rc; }
    if (int rc = caller_enter(h, D, caller)) return rc;
    CUDA_TRY(cudaMemsetAsync(D->d_scan_check, 0, sizeof(uint32_t), D->stream));
    scan_lidar_check_kernel<<<(n + 255) / 256, 256, 0, D->stream>>>(reinterpret_cast<const uint32_t*>(pts), n, (uint32_t)L,
                                                                    D->d_scan_check);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(D->h_scan_check, D->d_scan_check, sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    D->ctr.kernel_launches += 1;
    if (*D->h_scan_check) { h->err = "scan point with lidar id >= n_lidar"; return MALIO_ERR_INVALID_ARG; }
  }
  if (int rc = ensure_point_buffers(h, D, n > 0 ? n : 1)) return rc;
  const uint32_t n_tab = table_off[L];
  if (n_tab > D->d_table.size() / TABLE_DOUBLES) {
    if (int rc = D->d_table.allocate(h, D->stream, (size_t)(n_tab + 64) * TABLE_DOUBLES)) return rc;
  }
  if (n && from != SCAN_ROOM)
    CUDA_TRY(cudaMemcpyAsync(D->d_pts, pts, (size_t)n * sizeof(malio_scan_pt), on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                             D->stream));
  if (on_device) { if (int rc = caller_leave(h, D, caller)) return rc; }   // the copy is the last read of the caller's records
  CUDA_TRY(cudaMemcpyAsync(D->d_table, table, (size_t)n_tab * sizeof(malio_pose_entry), table_kind, D->stream));
  const uint32_t cap = (uint32_t)D->d_pts.size();
  reset_scan_kernel<<<(cap + 255) / 256, 256, 0, D->stream>>>(cap, D->d_sel, D->d_normal_y, D->d_nn_idx, D->d_gstats);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  for (int l = 0; l <= MALIO_MAX_LIDAR; ++l) D->table_off[l] = (l <= L) ? table_off[l] : table_off[L];
  for (int l = 1; l < L; ++l) D->tcomp[l] = tcomp[l - 1];
  D->N = n; D->scan_ready = true; D->perm_valid = false; D->tau_valid = false; D->pass_done = false;
  if (from == SCAN_HOST) D->ctr.h2d_bytes += (uint64_t)n * sizeof(malio_scan_pt);
  if (table_kind == cudaMemcpyHostToDevice) D->ctr.h2d_bytes += (uint64_t)n_tab * sizeof(malio_pose_entry);
  return MALIO_OK;
}

int upload_scan(malio_handle* h, const malio_scan_pt* pts, uint32_t n, const malio_pose_entry* table,
                const uint32_t* table_off, const malio_rigid* tcomp) {
  return upload_scan_from(h, SCAN_HOST, pts, n, table, cudaMemcpyHostToDevice, table_off, tcomp, nullptr);
}

int rearm_scan(malio_handle* h) {
  DeviceState* D = h->dev.get();
  if (!D->scan_ready) { h->err = "rearm_scan before upload_scan"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t cap = (uint32_t)D->d_pts.size();
  reset_scan_kernel<<<(cap + 255) / 256, 256, 0, D->stream>>>(cap, D->d_sel, D->d_normal_y, D->d_nn_idx, D->d_gstats);
  CUDA_TRY(cudaGetLastError());
  D->perm_valid = false; D->tau_valid = false; D->pass_done = false;
  return MALIO_OK;
}

int set_timing(malio_handle* h, int enable) {
  h->dev->timing = enable != 0;
  return MALIO_OK;
}

int get_counters(malio_handle* h, malio_counters* out) {
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  unsigned long long c[4] = {0, 0, 0, 0};
  CUDA_TRY(cudaMemcpy(c, D->d_cand, sizeof(c), cudaMemcpyDeviceToHost));
  D->ctr.knn_candidates = c[0];
  D->ctr.exchange_min_wait_ms = (double)c[1] * 1e-6;
  D->ctr.exchange_sum_wait_ms = (double)c[2] * 1e-6;
  D->ctr.exchange_passes = c[3];
  D->ctr.knn_tie_queries = D->h_gstats[7];
  *out = D->ctr;
  return MALIO_OK;
}

// download_aux's scatter from position space into caller order, into those of the five outputs that are not NULL: host arrays
// (on_device false) through the d_o_* staging buffers, which download_aux copies out when D->N > 0, or the caller's device
// arrays, ordered on `caller`
static int scatter_aux_to(malio_handle* h, float* normal_y, uint32_t* nn_idx, float* nn_d2, uint8_t* sel, float* world, bool on_device,
                          cudaStream_t caller) {
  DeviceState* D = h->dev.get();
  if (!D->pass_done) { h->err = "download_aux before measure"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t N = D->N;
  if (N == 0) return MALIO_OK;
  if (on_device) {
    if (int rc = check_device_ptrs(h, D, {{normal_y, "malio_download_aux_device normal_y"}, {nn_idx, "malio_download_aux_device nn_idx"},
                                          {nn_d2, "malio_download_aux_device nn_sqdist"}, {sel, "malio_download_aux_device selected"},
                                          {world, "malio_download_aux_device world"}}))
      return rc;
    if (int rc = caller_enter(h, D, caller)) return rc;
  } else {
    normal_y = normal_y ? D->d_o_ny.data() : nullptr; nn_idx = nn_idx ? D->d_o_idx.data() : nullptr; nn_d2 = nn_d2 ? D->d_o_d2.data() : nullptr;
    sel = sel ? D->d_o_sel.data() : nullptr; world = world ? D->d_o_world.data() : nullptr;
  }
  const uint32_t* perm = (h->cfg.sort_queries && D->perm_valid) ? D->d_perm.data() : nullptr;
  scatter_aux_kernel<<<(N + 255) / 256, 256, 0, D->stream>>>(perm, N, D->d_normal_y, D->d_nn_idx, D->d_nn_d2, D->d_sel, D->d_world,
                                                             normal_y, nn_idx, nn_d2, sel, world);
  CUDA_TRY(cudaGetLastError());
  if (on_device) { if (int rc = caller_leave(h, D, caller)) return rc; }
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

int download_aux(malio_handle* h, float* normal_y, uint32_t* nn_idx, float* nn_d2, uint8_t* sel, float* world) {
  if (int rc = scatter_aux_to(h, normal_y, nn_idx, nn_d2, sel, world, false, nullptr)) return rc;
  DeviceState* D = h->dev.get();
  const uint32_t N = D->N;
  if (N == 0) return MALIO_OK;
  if (normal_y) CUDA_TRY(cudaMemcpyAsync(normal_y, D->d_o_ny, (size_t)N * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  if (nn_idx) CUDA_TRY(cudaMemcpyAsync(nn_idx, D->d_o_idx, (size_t)N * MALIO_K * sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
  if (nn_d2) CUDA_TRY(cudaMemcpyAsync(nn_d2, D->d_o_d2, (size_t)N * MALIO_K * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  if (sel) CUDA_TRY(cudaMemcpyAsync(sel, D->d_o_sel, (size_t)N, cudaMemcpyDeviceToHost, D->stream));
  if (world) CUDA_TRY(cudaMemcpyAsync(world, D->d_o_world, (size_t)N * 3 * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  D->ctr.d2h_bytes += (uint64_t)N * ((normal_y ? 4 : 0) + (nn_idx ? 20 : 0) + (nn_d2 ? 20 : 0) + (sel ? 1 : 0) + (world ? 12 : 0));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}

// the stand-alone search of nq > 0 queries on the committed map: the point buffers grown, the sort, the search and the
// caller-order scatter of the lists.  Host call (on_device false): the queries go through d_queries, the lists into the d_o_*
// staging buffers, and ev[0] / ev[1] bracket the search kernels (knn_ms, ms_device).  Device call: the queries are read and the
// lists written where the caller keeps them, ordered on `caller`.  The scatter is counted by the callers.
static int knn_search(malio_handle* h, DeviceState* D, const float* q, uint32_t nq, uint32_t* idx, float* d2, bool on_device,
                      cudaStream_t caller) {
  if (int rc = ensure_point_buffers(h, D, nq)) return rc;
  if (!on_device && nq > D->d_queries.size() / 3) {
    if (int rc = D->d_queries.allocate(h, D->stream, (size_t)(nq + 1024) * 3)) return rc;
  }
  D->scan_ready = false;   // point buffers are shared with the scan path
  D->pass_done = false;
  if (on_device) {
    if (int rc = caller_enter(h, D, caller)) return rc;
  } else {
    CUDA_TRY(cudaMemcpyAsync(D->d_queries, q, (size_t)nq * 3 * sizeof(float), cudaMemcpyHostToDevice, D->stream));
    q = nullptr;   // sort_queries / run_knn: D->d_queries
    idx = idx ? D->d_o_idx.data() : nullptr;
    d2 = d2 ? D->d_o_d2.data() : nullptr;
  }
  PassConst pc{};
  const uint32_t* perm = nullptr;
  if (h->cfg.sort_queries) {
    if (int rc = sort_queries<1>(h, D, nq, pc, 0, q)) return rc;
    perm = D->d_perm;
  }
  CUDA_TRY(cudaMemsetAsync(D->d_gstats + 2, 0, 4 * sizeof(uint32_t), D->stream));
  if (!on_device) CUDA_TRY(cudaEventRecord(D->ev[0], D->stream));
  if (int rc = run_knn<1>(h, D, nq, nullptr, perm, pc, 0.f, q)) return rc;
  if (!on_device) CUDA_TRY(cudaEventRecord(D->ev[1], D->stream));
  scatter_aux_kernel<<<(nq + 255) / 256, 256, 0, D->stream>>>(perm, nq, nullptr, D->d_nn_idx, D->d_nn_d2, nullptr,
                                                               nullptr, nullptr, idx, d2, nullptr, nullptr);
  CUDA_TRY(cudaGetLastError());
  if (on_device) { if (int rc = caller_leave(h, D, caller)) return rc; }
  return MALIO_OK;
}

int knn(malio_handle* h, const float* q, uint32_t nq, uint32_t* idx, float* d2, float* ms_out) {
  DeviceState* D = h->dev.get();
  if (h->mapst) { if (int rc = malio_map::commit(h)) return rc; }
  if (!D->map_ready) { h->err = "knn before upload_map"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  if (nq == 0) return MALIO_OK;
  if (int rc = knn_search(h, D, q, nq, idx, d2, false, nullptr)) return rc;
  if (idx) CUDA_TRY(cudaMemcpyAsync(idx, D->d_o_idx, (size_t)nq * MALIO_K * sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
  if (d2) CUDA_TRY(cudaMemcpyAsync(d2, D->d_o_d2, (size_t)nq * MALIO_K * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  if (int rc = fetch_knn_stats(h, D, D->stream)) return rc;
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  CUDA_TRY(cudaGetLastError());
  if (int rc = knn_fault(h, D)) return rc;
  float ms = 0.f;
  cudaEventElapsedTime(&ms, D->ev[0], D->ev[1]);
  if (ms_out) *ms_out = ms;
  D->ctr.kernel_launches += 1;   // scatter (the sort and the k-NN count their own)
  if (D->grid_on) { D->ctr.knn_fallback_queries += D->h_gstats[3]; D->ctr.knn_ring2_queries += D->h_gstats[5]; }
  D->ctr.knn_launches += 1; D->ctr.knn_queries += nq; D->ctr.knn_ms += ms;
  D->ctr.h2d_bytes += (uint64_t)nq * 12;
  D->ctr.d2h_bytes += (uint64_t)nq * ((idx ? 20 : 0) + (d2 ? 20 : 0));
  return MALIO_OK;
}

// malio_knn on device memory, ordered on the caller's stream.  Returns after enqueueing; the statistics malio_knn waits for are
// copied behind the search and folded in by the next call on the handle (settle_knn_device).
int knn_device(malio_handle* h, const float* q, uint32_t nq, uint32_t* idx, float* d2, cudaStream_t caller) {
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  if (nq) {
    if (int rc = check_device_ptr(h, D, q, "malio_knn_device queries")) return rc;
    if (int rc = check_device_ptr(h, D, idx, "malio_knn_device nn_idx")) return rc;
    if (int rc = check_device_ptr(h, D, d2, "malio_knn_device nn_sqdist")) return rc;
  }
  if (!D->map_ready) { h->err = "knn before upload_map"; return MALIO_ERR_STATE; }
  if (nq == 0) return MALIO_OK;
  if (h->mapst) { if (int rc = malio_map::commit(h)) return rc; }
  if (int rc = knn_fault(h, D)) return rc;   // this map already overflowed a traversal stack: no search on it is trusted
  if (int rc = knn_search(h, D, q, nq, idx, d2, true, caller)) return rc;
  if (int rc = fetch_knn_stats(h, D, D->stream)) return rc;   // behind the caller's event: the caller does not wait for it
  CUDA_TRY(cudaEventRecord(D->ev_deferred, D->stream));
  D->deferred_grid = D->grid_on;
  h->deferred = settle_knn_device;
  D->ctr.kernel_launches += 1;   // scatter (the sort and the k-NN count their own)
  D->ctr.knn_launches += 1; D->ctr.knn_queries += nq;
  return MALIO_OK;
}

// map_incremental's decision per point of the last pass, in caller order, into cls (N bytes) and world (N x 3 floats, may be
// NULL): host arrays (on_device false) through the d_o_sel / d_o_world staging buffers of download_aux, which map_incremental
// copies out when D->N > 0, or the caller's device arrays, ordered on `caller`
static int map_incr_to(malio_handle* h, const malio_pass_state* s, double fs, int ekf_inited, uint8_t* cls, float* world, bool on_device,
                       cudaStream_t caller) {
  DeviceState* D = h->dev.get();
  if (!D->pass_done) { h->err = "map_incremental before measure"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t N = D->N;
  if (N == 0) return MALIO_OK;
  const bool sorted = h->cfg.sort_queries && D->perm_valid;
  const PassConst pc = make_pass_const(h, D, s);
  if (on_device) {
    if (int rc = check_device_ptr(h, D, cls, "malio_map_incremental_device cls")) return rc;
    if (int rc = check_device_ptrs(h, D, {{world, "malio_map_incremental_device world"}})) return rc;
    if (int rc = caller_enter(h, D, caller)) return rc;
  } else {
    cls = D->d_o_sel;
    world = world ? D->d_o_world.data() : nullptr;
  }
  map_incr_kernel<<<(N + 255) / 256, 256, 0, D->stream>>>(sorted ? D->d_pts_sorted.data() : D->d_pts.data(), sorted ? D->d_perm.data() : nullptr, N, pc,
                                                           D->d_mpts, D->d_nn_idx, D->d_normal_y, h->cfg.params.cov_threshold, fs,
                                                           ekf_inited, cls, world);
  CUDA_TRY(cudaGetLastError());
  if (on_device) { if (int rc = caller_leave(h, D, caller)) return rc; }
  D->ctr.kernel_launches += 1;
  return MALIO_OK;
}

int map_incremental(malio_handle* h, const malio_pass_state* s, double fs, int ekf_inited, uint8_t* cls, float* world) {
  if (int rc = map_incr_to(h, s, fs, ekf_inited, cls, world, false, nullptr)) return rc;
  DeviceState* D = h->dev.get();
  const uint32_t N = D->N;
  if (N == 0) return MALIO_OK;
  CUDA_TRY(cudaMemcpyAsync(cls, D->d_o_sel, (size_t)N, cudaMemcpyDeviceToHost, D->stream));
  if (world) CUDA_TRY(cudaMemcpyAsync(world, D->d_o_world, (size_t)N * 3 * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  D->ctr.d2h_bytes += (uint64_t)N * (1 + (world ? 12 : 0));
  return MALIO_OK;
}

}  // namespace malio_dev

extern "C" int malio_knn_device(malio_handle* h, const float* d_queries, uint32_t n_queries, uint32_t* d_nn_idx,
                                float* d_nn_sqdist, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_dev::knn_device(h, d_queries, n_queries, d_nn_idx, d_nn_sqdist, (cudaStream_t)stream);
}

// the wrappers check what malio_upload_scan / _download_aux / _map_incremental check on the host; the device pointers are
// checked inside, once the point count is known
extern "C" int malio_upload_scan_from_device(malio_handle* h, const malio_scan_pt* d_pts, uint32_t n_pts, const malio_pose_entry* table,
                                             const uint32_t* table_off, const malio_rigid* temporal_comp, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!table || !table_off) return MALIO_ERR_INVALID_ARG;
  if (h->cfg.params.n_lidar > 1 && !temporal_comp) { h->err = "temporal_comp required for L > 1"; return MALIO_ERR_INVALID_ARG; }
  return malio_dev::upload_scan_from(h, malio_dev::SCAN_DEVICE, d_pts, n_pts, table, cudaMemcpyHostToDevice, table_off, temporal_comp,
                                     (cudaStream_t)stream);
}
extern "C" int malio_download_aux_device(malio_handle* h, float* d_normal_y, uint32_t* d_nn_idx, float* d_nn_sqdist,
                                         uint8_t* d_selected, float* d_world, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_dev::scatter_aux_to(h, d_normal_y, d_nn_idx, d_nn_sqdist, d_selected, d_world, true, (cudaStream_t)stream);
}
extern "C" int malio_map_incremental_device(malio_handle* h, const malio_pass_state* s, double filter_size_map, int ekf_inited,
                                            uint8_t* d_cls, float* d_world, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!s || !(filter_size_map > 0.0)) return MALIO_ERR_INVALID_ARG;
  return malio_dev::map_incr_to(h, s, filter_size_map, ekf_inited, d_cls, d_world, true, (cudaStream_t)stream);
}
