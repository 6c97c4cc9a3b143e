// malio_device.cuh — device-side state of one handle and the constants shared by the CUDA translation units of
// libmalio_b200.so (malio_b200.cu: k-NN / pass kernels and the per-scan entry points; malio_preproc.cu: undistortion and
// voxel grid; malio_mapops.cu: the device-resident map and its Add_Points / Delete_Point_Boxes replay).
#ifndef MALIO_DEVICE_CUH_
#define MALIO_DEVICE_CUH_

#include <cuda_runtime.h>
#include <nccl.h>

#include <cstdint>
#include <string>

#include "malio_internal.h"

namespace malio_devstate {

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

// Quaternion * vector as Eigen's _transformVector: v + w*uv + qv x uv, uv = 2 (qv x v); q = (w,x,y,z).  The same operations,
// in the same order, as malio_b200.cu's q_rot.
__device__ __forceinline__ void eigen_q_rot(const double q[4], const double v[3], double o[3]) {
  const double uv0 = q[2] * v[2] - q[3] * v[1], uv1 = q[3] * v[0] - q[1] * v[2], uv2 = q[1] * v[1] - q[2] * v[0];
  const double u[3] = {uv0 + uv0, uv1 + uv1, uv2 + uv2};
  const double c0 = q[2] * u[2] - q[3] * u[1], c1 = q[3] * u[0] - q[1] * u[2], c2 = q[1] * u[1] - q[2] * u[0];
  o[0] = v[0] + q[0] * u[0] + c0;
  o[1] = v[1] + q[0] * u[1] + c1;
  o[2] = v[2] + q[0] * u[2] + c2;
}

// pointBodyToWorld / RGBpointBodyToWorld (laserMapping.cpp:134-163) in the reference's own operation order (no detour through
// the LiDAR-0 frame), in double, rounded to float at the end:
//   lid == 0:  p_w = rot (q_E[0] p + t_E[0]) + pos
//   lid != 0:  p_w = rot (q_C[lid-1] (q_E[lid] p + t_E[lid]) + t_C[lid-1]) + pos      (PassConst keeps q_C[lid-1] at cq[lid])
// One function for map_incr_kernel and world_kernel, so that both give the same bits.
__device__ __forceinline__ void body_to_world(const PassConst& pc, int lid, float x, float y, float z, float w[3]) {
  const double pb[3] = {(double)x, (double)y, (double)z};
  double a[3], g[3];
  eigen_q_rot(pc.eq[lid], pb, a);
  a[0] += pc.et[lid][0]; a[1] += pc.et[lid][1]; a[2] += pc.et[lid][2];
  if (lid != 0) {                                                                               // :142, :157
    double b[3];
    eigen_q_rot(pc.cq[lid], a, b);
    a[0] = b[0] + pc.ct[lid][0]; a[1] = b[1] + pc.ct[lid][1]; a[2] = b[2] + pc.ct[lid][2];
  }
  eigen_q_rot(pc.rot, a, g);
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
  malio_counters ctr{};
  bool timing = true;   // per-pass CUDA-event timing (malio_set_timing)
  double host_launch_us = 0, host_wait_us = 0; uint64_t host_passes = 0;   // MALIO_HOST_PROF=1 prints them at destroy
  // map
  float4* d_nodes = nullptr; float* d_cov = nullptr;
  float4* d_mpts = nullptr;            // compact mirror: point + link of every node, 16 B stride
  uint32_t *d_parent = nullptr, *d_arrived = nullptr;   // box rebuild of the compact upload
  uint32_t n_nodes = 0, cap_nodes = 0, depth = 0;
  // device-resident map mode (malio_mapops.cu): d_mpts / d_cov / d_ids are slots of a point set (link word = deleted bit only),
  // there are no 64-byte tree records and the search never walks a tree
  bool tree_free = false; int32_t* d_ids = nullptr; uint32_t cap_slots = 0;
  // scan (caller order) + internal order
  malio_scan_pt* d_pts = nullptr; uint32_t N = 0, capN = 0;
  malio_scan_pt* d_pts_sorted = nullptr;   // the scan in internal (position) order
  uint32_t* d_perm = nullptr; bool perm_valid = false;
  uint16_t* d_keys16 = nullptr; uint32_t *d_hist = nullptr, *d_offs = nullptr, *d_cursor = nullptr, *d_btot = nullptr, *d_tmp_ids = nullptr;   // counting sort
  double* d_table = nullptr; uint32_t cap_table = 0;
  uint32_t table_off[MALIO_MAX_LIDAR + 1] = {0, 0, 0, 0};
  malio_rigid tcomp[MALIO_MAX_LIDAR];
  bool scan_ready = false, map_ready = false, pass_done = false, searched_once = false;
  // per point, position space
  uint32_t* d_nn_idx = nullptr; float* d_nn_d2 = nullptr; uint8_t* d_sel = nullptr;
  float4 *d_world = nullptr, *d_plane = nullptr; double *d_ucov = nullptr, *d_tau = nullptr; float* d_normal_y = nullptr;
  double2* d_tau2 = nullptr; float* d_pd2 = nullptr; bool tau_valid = false;
  double* d_rows12 = nullptr; uint8_t* d_lid8 = nullptr;
  // aux staging (caller order)
  float* d_o_ny = nullptr; uint32_t* d_o_idx = nullptr; float* d_o_d2 = nullptr; uint8_t* d_o_sel = nullptr; float* d_o_world = nullptr;
  // reductions
  double* d_block_mm = nullptr; uint32_t* d_block_cnt = nullptr; uint32_t cap_blocks = 0;
  uint32_t* d_counters = nullptr;   // [0] plane, [1] reduce, [2] n_eff local, [3] n_rows
  unsigned long long* d_mmkey = nullptr;   // 2 parities x 4 keys (+ counts in d_counters[4+parity])
  int parity = 0, last_parity = 0;
  double* d_block_red = nullptr; uint32_t red_grid = 0;
  double* d_res = nullptr;          // MALIO_RED_DOUBLES
  double* d_rows = nullptr;         // MALIO_MAX_DOF x 25
  double* h_res = nullptr;          // pinned: res | mm(4) | cnt
  PassConst last_pc{};
  // stand-alone queries
  float* d_queries = nullptr; uint32_t capQ = 0;
  // cell-list index over the live snapshot points (k-NN fast path)
  bool grid_on = false; GridConst grid{}; float grid_h = 0.f;
  uint32_t *d_cell_start = nullptr, *d_cell_cnt = nullptr, *d_cell_of = nullptr, *d_ctot = nullptr, *d_cbase = nullptr;
  uint32_t cap_cells = 0, cap_cell_pts = 0;
  float4* d_cell_pts = nullptr;
  uint32_t* d_fb_list = nullptr;          // positions the fast path could not settle (-> exact traversal)
  unsigned long long* d_cand = nullptr;   // [0] candidates scanned by the cell-list scans since create (summed only while timing is on)
  uint32_t* d_gstats = nullptr;           // [0] occupied cells, [1] live points, [2] fb count, [3] fb count of the last search, [4] ring-2 queries
  uint32_t* h_gstats = nullptr;            // pinned mirror (8 words, carved out of h_res)
  // fused pass (single cooperative launch per measurement pass)
  bool fused = true; int pass_max_blocks = 0, pass_max_blocks_generic = 0;
  int trace_passes = 0; float env_knn_cell = -1.f; bool env_knn_cell_set = false; bool host_prof = false;   // environment switches, read once in create()
  uint32_t* d_bar = nullptr; uint32_t bar_base[3] = {0, 0, 0}; uint32_t seq = 0;
  double* h_res_dev = nullptr;     // device-side address of the mapped host result buffer
  unsigned long long* d_dbg = nullptr; int trace_left = 0;
  // multi-GPU
  ncclComm_t comm = nullptr; int rank = 0, world = 1;
  bool p2p = false; unsigned char* d_mail = nullptr; unsigned char* mail_peer[MAIL_MAX_WORLD] = {nullptr};
};

template <class T>
int ensure(malio_handle* h, T*& ptr, size_t count) {
  if (ptr) { cudaFree(ptr); ptr = nullptr; }
  CUDA_TRY(cudaMalloc((void**)&ptr, count * sizeof(T)));
  return MALIO_OK;
}

}  // namespace malio_devstate

#endif  // MALIO_DEVICE_CUH_
