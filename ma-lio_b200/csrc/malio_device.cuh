// malio_device.cuh — device-side state of one handle, the device math and constants shared by the CUDA translation units
// of libmalio_b200.so, and the host functions they call in each other.  The units (no relocatable device code: each one
// launches only its own kernels):
//   malio_knn.cu      the k-NN search and the map it searches (snapshot upload, cell-list index, query sort)
//   malio_pass.cu     the measurement pass (plane fit, gate, reduction, the fused pass_kernel and its multi-GPU exchange)
//   malio_b200.cu     handle lifecycle and per-scan data movement (create / destroy, scan upload, downloads)
//   malio_preproc.cu  undistortion, voxel grid, world registration
//   malio_mapops.cu   the device-resident map and its Add_Points / Delete_Point_Boxes replay
//   malio_voxmap.cu   the saved map as a voxel map
//   malio_prior.cu    localization in a prior map: the prior's tile store and the local-map window over it
//   malio_reloc.cu    relocalization in a loaded prior: branch-and-bound over yaws and a position lattice
//   malio_place.cu    relocalization without a position guess: place descriptors of the prior, ranked, each checked by malio_reloc
#ifndef MALIO_DEVICE_CUH_
#define MALIO_DEVICE_CUH_

#include <cuda_runtime.h>
#include <nccl.h>

#include <cstdint>
#include <cstring>
#include <initializer_list>
#include <string>

#include "malio_buffer.h"
#include "malio_internal.h"

namespace malio_devstate {

using malio_buf::acquire;
using malio_buf::DeviceBuffer;
using malio_buf::PinnedBuffer;
using malio_buf::release;

#define CUDA_TRY(expr)                                                                     \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      h->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                          \
      return MALIO_ERR_CUDA;                                                               \
    }                                                                                      \
  } while (0)

constexpr int KNN_THREADS = 64;
constexpr int PLANE_THREADS = 64;
constexpr int GATE_THREADS = 256;
constexpr int RED_THREADS = 128;          // one tile = 128 points
constexpr int RED_HS_STRIDE = 13;         // doubles per staged row of a*J12/rho (12 + 1: odd stride, conflict-free)
constexpr int RED_HX_STRIDE = 17;         // doubles per staged row of [a*J12 | z | rho*a*J12_0..2] (16 + 1)
constexpr int RED_TASKS = 9;              // upper-triangular 4x4 blocks of the 12 x 16 compact system
constexpr int RED_KS = 14;                // row-splits per task: 9 x 14 = 126 of the 128 threads work
constexpr int RED_SMEM_DOUBLES = RED_THREADS * (RED_HS_STRIDE + RED_HX_STRIDE) + RED_TASKS * RED_KS * 16;   // staging + flush scratch
constexpr int TABLE_DOUBLES = 52;         // malio_pose_entry
constexpr int SORT_BINS = 1 << 16;        // counting sort of the queries (malio_knn.cu): bins ...
constexpr int SCAN_BLOCKS = 64;           // ... and blocks of its prefix scan
constexpr uint32_t FAULT_STACK_OVERFLOW = 1u;   // d_gstats[6]: a traversal stack overflowed (snapshot deeper than declared)

struct PassConst {
  double rot[4], pos[3];
  double eq[MALIO_MAX_LIDAR][4], et[MALIO_MAX_LIDAR][3];   // extrinsics (state)
  double cq[MALIO_MAX_LIDAR][4], ct[MALIO_MAX_LIDAR][3];   // temporal compensation, index l (entry 0 unused)
  uint32_t table_off[MALIO_MAX_LIDAR + 1];
  int L;
  int ext_en;
  // rotation matrices (row-major) of the conjugates, filled by the host once per pass: the Jacobian rows are matrix-vector
  // products with them (9 FP64 instructions each instead of ~33 for a quaternion sandwich; FP64 issue is what bounds the gate)
  double RsT[9];                       // R(s.rot)^T
  double ReT[MALIO_MAX_LIDAR][9];      // R(offset_R_l)^T
  double RcT[MALIO_MAX_LIDAR][9];      // R(temporal_comp_l)^T  (entry 0 unused)
};

// ------------------------------------------------------------------ small device algebra (mirrors Eigen's op order)
__device__ __forceinline__ void cross3(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
// Quaternion * vector as Eigen's _transformVector: v + w*uv + qv x uv, uv = 2 (qv x v); q = (w,x,y,z)
__device__ __forceinline__ void q_rot(const double q[4], const double v[3], double o[3]) {
  const double qv[3] = {q[1], q[2], q[3]};
  double uv[3], c2[3];
  cross3(qv, v, uv);
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  cross3(qv, uv, c2);
  o[0] = v[0] + q[0] * uv[0] + c2[0];
  o[1] = v[1] + q[0] * uv[1] + c2[1];
  o[2] = v[2] + q[0] * uv[2] + c2[2];
}
__device__ __forceinline__ void q_rot_conj(const double q[4], const double v[3], double o[3]) {
  const double qc[4] = {q[0], -q[1], -q[2], -q[3]};
  q_rot(qc, v, o);
}
// laserMapping.cpp:569-579: point in its LiDAR frame -> LiDAR-0 body frame b, IMU frame m, world g
__device__ __forceinline__ void transform_point(const PassConst& pc, float px, float py, float pz, int lid,
                                                double b[3], double m[3], double g[3]) {
  b[0] = px; b[1] = py; b[2] = pz;
  if (lid != 0) {
    double a[3], t[3], d[3];
    q_rot(pc.eq[lid], b, a);
    a[0] += pc.et[lid][0]; a[1] += pc.et[lid][1]; a[2] += pc.et[lid][2];
    q_rot(pc.cq[lid], a, t);
    d[0] = (t[0] + pc.ct[lid][0]) - pc.et[0][0];
    d[1] = (t[1] + pc.ct[lid][1]) - pc.et[0][1];
    d[2] = (t[2] + pc.ct[lid][2]) - pc.et[0][2];
    q_rot_conj(pc.eq[0], d, b);
  }
  q_rot(pc.eq[0], b, m);
  m[0] += pc.et[0][0]; m[1] += pc.et[0][1]; m[2] += pc.et[0][2];
  q_rot(pc.rot, m, g);
  g[0] += pc.pos[0]; g[1] += pc.pos[1]; g[2] += pc.pos[2];
}
// order-preserving map double <-> uint64 (so that min/max can use integer atomics: exact and order-independent)
__host__ __device__ __forceinline__ unsigned long long dkey(double v) {
  unsigned long long b;
  memcpy(&b, &v, 8);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double dkey_inv(unsigned long long k) {
  const unsigned long long b = (k & 0x8000000000000000ull) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
  double v;
  memcpy(&v, &b, 8);
  return v;
}

// pointBodyToWorld / RGBpointBodyToWorld (laserMapping.cpp:134-163) in the reference's own operation order (no detour through
// the LiDAR-0 frame), in double, rounded to float at the end:
//   lid == 0:  p_w = rot (q_E[0] p + t_E[0]) + pos
//   lid != 0:  p_w = rot (q_C[lid-1] (q_E[lid] p + t_E[lid]) + t_C[lid-1]) + pos      (PassConst keeps q_C[lid-1] at cq[lid])
// One function for map_incr_kernel and world_kernel, so that both give the same bits.
__device__ __forceinline__ void body_to_world(const PassConst& pc, int lid, float x, float y, float z, float w[3]) {
  const double pb[3] = {(double)x, (double)y, (double)z};
  double a[3], g[3];
  q_rot(pc.eq[lid], pb, a);
  a[0] += pc.et[lid][0]; a[1] += pc.et[lid][1]; a[2] += pc.et[lid][2];
  if (lid != 0) {                                                                               // :142, :157
    double b[3];
    q_rot(pc.cq[lid], a, b);
    a[0] = b[0] + pc.ct[lid][0]; a[1] = b[1] + pc.ct[lid][1]; a[2] = b[2] + pc.ct[lid][2];
  }
  q_rot(pc.rot, a, g);
  w[0] = (float)(g[0] + pc.pos[0]); w[1] = (float)(g[1] + pc.pos[1]); w[2] = (float)(g[2] + pc.pos[2]);
}

struct ParamConst {
  float plane_th, knn_max_sqdist;
  double cov_threshold, point_cov_max, point_cov_min, plane_cov_max, plane_cov_min, range_min, range_max;
};

struct GridConst {
  float ox, oy, oz, inv_h, h;
  int nx, ny, nz;        // cells per axis (un-padded)
  int px, py;            // padded pitches: nx + 2*GRID_PAD, ny + 2*GRID_PAD
  uint32_t ncell;        // padded cell count
};
constexpr int GRID_PAD = 3;          // empty border cells: queries up to one cell outside the box still take the fast path
constexpr int GRID_CHUNK = 4096;          // cells per scan block (1024 threads x 4)
constexpr float GRID_MARGIN = 0.005f;     // in cells: >> rounding of (x - o) * inv_h (< 1e-3 cells for < 4096 cells/axis)
__host__ __device__ __forceinline__ uint32_t grid_cell_index(const GridConst& G, int cx, int cy, int cz) {
  return (uint32_t)(((cz + GRID_PAD) * G.py + (cy + GRID_PAD)) * G.px + (cx + GRID_PAD));
}

constexpr int MAIL_MAX_WORLD = 8;
constexpr int ROWS_DOUBLES = MALIO_MAX_DOF * 25 + 8;   // rows of the degenerate branch (25 doubles each) | row count | padding
constexpr int MAIL_MIN_BYTES = 64;        // u64 keys[4] | u32 count | u32 seq (byte 40)
constexpr int MAIL_SUM_BYTES = 3584;      // double res[MALIO_RED_DOUBLES] | u32 seq (byte 3480)
constexpr int MAIL_SUM_SEQ_OFF = 3480;
static_assert(MALIO_RED_DOUBLES * 8 <= MAIL_SUM_SEQ_OFF, "mailbox slot too small");
constexpr int MAIL_PARITY_BYTES = MAIL_MAX_WORLD * (MAIL_MIN_BYTES + MAIL_SUM_BYTES);
constexpr int MAIL_BYTES = 2 * MAIL_PARITY_BYTES;
struct DeviceState {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;            // box rebuild of the compact upload runs beside the scan's first kernels
  cudaStream_t stream3 = nullptr;            // copy stream for the map-side weights of the compact upload
  cudaEvent_t ev_h2d = nullptr, ev_refit = nullptr; bool refit_pending = false;
  cudaEvent_t ev_cov = nullptr;
  cudaEvent_t ev_sorted = nullptr, ev_tau = nullptr;   // point-covariance traces run beside the first search of a scan
  cudaEvent_t ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // [5] after sort, [6] after knn kernel
  // calls on device memory ordered on the caller's stream (malio_knn_device, malio_map_*_device): ev_caller_in is recorded on
  // the caller's stream and waited for by this handle's, ev_caller_out the other way round; ev_deferred follows the copy of the
  // search statistics the next entry point folds in (settle_deferred), deferred_grid whether that search ran on the cell list
  cudaEvent_t ev_caller_in = nullptr, ev_caller_out = nullptr, ev_deferred = nullptr; bool deferred_grid = false;
  // malio_upload_scan_from_device: the record check's flag word and its pinned host copy (allocated on first use)
  DeviceBuffer<uint32_t> d_scan_check; PinnedBuffer<uint32_t> h_scan_check;
  malio_counters ctr{};
  bool timing = true;   // per-pass CUDA-event timing (malio_set_timing)
  double host_launch_us = 0, host_wait_us = 0; uint64_t host_passes = 0;   // MALIO_HOST_PROF=1 prints them at destroy
  // map
  DeviceBuffer<float4> d_nodes; DeviceBuffer<float> d_cov;   // 64-byte tree records (4 float4 each); map-side weights
  DeviceBuffer<float4> d_mpts;         // compact mirror: point + link of every node, 16 B stride; its size sizes the cell lists
  DeviceBuffer<uint32_t> d_parent, d_arrived;   // box rebuild of the compact upload
  uint32_t n_nodes = 0, depth = 0;
  // device-resident map mode (malio_mapops.cu): d_mpts / d_cov / d_ids are slots of a point set (link word = deleted bit only),
  // there are no 64-byte tree records and the search never walks a tree.  slot_store is a mode, not a size: false once a
  // snapshot upload has taken d_mpts / d_cov, so that the next grow_slots re-creates the slot store
  bool tree_free = false; DeviceBuffer<int32_t> d_ids; bool slot_store = false;
  // scan (caller order) + internal order; the point buffers share one capacity, d_pts' size
  DeviceBuffer<malio_scan_pt> d_pts; uint32_t N = 0;
  DeviceBuffer<malio_scan_pt> d_pts_sorted;   // the scan in internal (position) order
  DeviceBuffer<uint32_t> d_perm; bool perm_valid = false;
  DeviceBuffer<uint16_t> d_keys16; DeviceBuffer<uint32_t> d_hist, d_offs, d_cursor, d_btot, d_tmp_ids;   // counting sort
  DeviceBuffer<double> d_table;
  uint32_t table_off[MALIO_MAX_LIDAR + 1] = {0, 0, 0, 0};
  malio_rigid tcomp[MALIO_MAX_LIDAR];
  bool scan_ready = false, map_ready = false, pass_done = false;
  // per point, position space
  DeviceBuffer<uint32_t> d_nn_idx; DeviceBuffer<float> d_nn_d2; DeviceBuffer<uint8_t> d_sel;
  DeviceBuffer<float4> d_world, d_plane; DeviceBuffer<double> d_ucov, d_tau; DeviceBuffer<float> d_normal_y;
  DeviceBuffer<double2> d_tau2; DeviceBuffer<float> d_pd2; bool tau_valid = false;
  DeviceBuffer<double> d_rows12; DeviceBuffer<uint8_t> d_lid8;
  // aux staging (caller order)
  DeviceBuffer<float> d_o_ny; DeviceBuffer<uint32_t> d_o_idx; DeviceBuffer<float> d_o_d2; DeviceBuffer<uint8_t> d_o_sel; DeviceBuffer<float> d_o_world;
  // reductions
  DeviceBuffer<uint32_t> d_counters;   // [3] rows rows_kernel found (download_rows); [0..2] unused
  DeviceBuffer<unsigned long long> d_mmkey;   // 2 parities x 4 keys
  int parity = 0, last_parity = 0;
  DeviceBuffer<double> d_block_red; uint32_t red_grid = 0;
  DeviceBuffer<double> d_res;          // MALIO_RED_DOUBLES
  DeviceBuffer<double> d_rows;         // MALIO_MAX_DOF x 25
  PinnedBuffer<double> h_res;          // pinned, mapped: res | mm(4) | cnt
  PassConst last_pc{};
  // stand-alone queries
  DeviceBuffer<float> d_queries;
  // cell-list index over the live snapshot points (k-NN fast path)
  bool grid_on = false; GridConst grid{}; float grid_h = 0.f;
  DeviceBuffer<uint32_t> d_cell_start, d_cell_cnt, d_cell_of, d_ctot, d_cbase;
  DeviceBuffer<float4> d_cell_pts;
  DeviceBuffer<uint32_t> d_fb_list;          // positions the fast path could not settle (-> exact traversal)
  DeviceBuffer<unsigned long long> d_cand;   // [0] candidates scanned by the cell-list scans since create (summed only while timing is on)
  // [0] occupied cells, [1] live points, [2] fb count, [3] fb count of the last search, [4] ring-2 queries, [5] ring-2 queries
  // of the last search, [6] traversal fault bits (FAULT_STACK_OVERFLOW; cleared only by a map upload), [7] tie queries
  DeviceBuffer<uint32_t> d_gstats;
  uint32_t* h_gstats = nullptr;            // pinned mirror (8 words, carved out of h_res)
  // fused pass (single cooperative launch per measurement pass)
  bool fused = true; int pass_max_blocks = 0, pass_max_blocks_generic = 0;
  int trace_passes = 0; float env_knn_cell = -1.f; bool env_knn_cell_set = false; bool host_prof = false;   // environment switches, read once in create()
  DeviceBuffer<uint32_t> d_bar; uint32_t bar_base[3] = {0, 0, 0}; uint32_t seq = 0;
  double* h_res_dev = nullptr;     // device-side address of the mapped host result buffer
  DeviceBuffer<unsigned long long> d_dbg; int trace_left = 0;
  // multi-GPU
  ncclComm_t comm = nullptr; int rank = 0, world = 1;
  // d_mail: this rank's mailbox; mail_peer: every rank's, the peers' opened with cudaIpcOpenMemHandle (closed by comm_destroy)
  bool p2p = false; DeviceBuffer<unsigned char> d_mail; unsigned char* mail_peer[MAIL_MAX_WORLD] = {nullptr};

  // the streams and events of a state create() made, whole or in part; the owner has drained `stream` (the buffers go back
  // after this body)
  ~DeviceState() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    for (cudaStream_t s : {stream2, stream3}) if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    for (cudaEvent_t e : {ev_h2d, ev_refit, ev_cov, ev_sorted, ev_tau, ev_caller_in, ev_caller_out, ev_deferred}) if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
  }
};

// ---- host functions one unit calls in another
// malio_knn.cu.  MODE 0: the scan's points through pc, MODE 1: stand-alone world-frame queries, n x 3 floats in `queries`
// (device memory; NULL = D->d_queries).
// keys + counting sort of n queries into D->d_perm; lid_major: LiDAR id as the major key (large scans, see count_kernel)
template <int MODE>
int sort_queries(malio_handle* h, DeviceState* D, uint32_t n, const PassConst& pc, int lid_major, const float* queries = nullptr);
template <int MODE>
int run_knn(malio_handle* h, DeviceState* D, uint32_t n, const malio_scan_pt* pts_in, const uint32_t* perm,
            const PassConst& pc, float max_sqdist, const float* queries = nullptr);
// d_gstats[2..7] of the last search -> h_gstats[2..7], enqueued on st
int fetch_knn_stats(malio_handle* h, DeviceState* D, cudaStream_t st);
// MALIO_ERR_TREE_TOO_DEEP if a traversal of this handle overflowed its stack since the last map upload (h_gstats[6])
int knn_fault(malio_handle* h, const DeviceState* D);
// malio_b200.cu: the device-memory entry points.
// MALIO_OK when p is 4-byte aligned device memory of D's device (cudaMalloc / a memory pool: what torch allocates); NULL, host,
// pinned, managed or another device's memory -> MALIO_ERR_INVALID_ARG with h->err naming `what`
int check_device_ptr(malio_handle* h, const DeviceState* D, const void* p, const char* what);
// check_device_ptr on each pointer of the list that is not NULL (NULL: that output is not asked for), in list order
struct DevicePtrArg { const void* p; const char* what; };
int check_device_ptrs(malio_handle* h, const DeviceState* D, std::initializer_list<DevicePtrArg> args);
// D->stream waits for everything enqueued on the caller's stream so far / the caller's stream waits for D->stream
int caller_enter(malio_handle* h, DeviceState* D, cudaStream_t caller);
int caller_leave(malio_handle* h, DeviceState* D, cudaStream_t caller);
// malio_pass.cu
PassConst make_pass_const(const malio_handle* h, const DeviceState* D, const malio_pass_state* s);
int pass_init(malio_handle* h, DeviceState* D);   // part of create(): per-block result slots, pass_kernel launch limits
void comm_destroy(DeviceState* D);

}  // namespace malio_devstate

// malio_b200.cu: the scan upload of every entry point that sets the scan.  The n records come from
//   SCAN_HOST    host memory (malio_upload_scan*): checked by a host sweep, copied H2D
//   SCAN_DEVICE  the caller's device memory (malio_upload_scan_from_device), ordered on `caller`: checked where they are, the
//                host waiting for the verdict so that a bad scan changes nothing, then copied D2D into d_pts, because the
//                passes keep reading d_pts over several malio_measure calls while the caller may reuse its buffer
//   SCAN_ROOM    nowhere: d_pts gets room for n records, which the caller fills on the handle's stream (malio_preproc.cu's
//                merged scan)
// table_kind: where `table` lives, host memory or this device's (malio_upload_scan_resident)
namespace malio_dev {
enum ScanSource { SCAN_HOST, SCAN_DEVICE, SCAN_ROOM };
int upload_scan_from(malio_handle* h, ScanSource from, const malio_scan_pt* pts, uint32_t n, const malio_pose_entry* table,
                     cudaMemcpyKind table_kind, const uint32_t* table_off, const malio_rigid* tcomp, cudaStream_t caller);
}

#endif  // MALIO_DEVICE_CUH_
