// malio_preproc.cu — the two stages immediately before the hot path (SURVEY.md §8f), sm_90a:
//   N2  ImuProcess::UndistortPcl's per-raw-point loop        src/IMU_Processing.hpp:468-508
//       BsplineSE3::get_pose                                  src/BsplineSE3.cpp:84-118, quat_ops.h:150-257
//   N3  pcl::VoxelGrid down-sampling + merge into the scan    src/laserMapping.cpp:968-983
// and the one after the update that reads their clouds again:
//       publish_frame_world + the saved map (pcl_wait_save)   src/laserMapping.cpp:448-489, 1083-1091
// Compiled with -fmad=false like the rest of the library: every double expression is evaluated with the IEEE operations
// the reference's x86-64 build uses, in its order.
//
// N2 on the device.  (1) log_se3(Inv(P_k) P_{k+1}) depends on the control points only: one thread per control-point pair
// computes it once per call (the reference recomputes three of them per point).  (2) One thread per raw point: bounding
// control points by binary search in shared memory, three exp_se3, the pose product, Eigen's matrix->quaternion
// conversion, the compensation of :492, and need_i = how many entries of the IMU-covariance list lie above the point's
// time.  (3) The reference walks that list with AT MOST ONE pop per point (:476-486), last point first:
//        pops_s = min(need_s, pops_{s-1} + 1)   =>   pops_s = s + min(1, min_{j<=s}(need_j - j))
// a min-plus prefix scan over the reversed point order, done by one block (chunked Hillis-Steele in shared memory);
// intensity = pops - 1, and every increase of pops marks the point whose pose seeds a table entry.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "malio_compound.h"
#include "malio_device.cuh"

using namespace malio_devstate;

namespace malio_pre {

struct PreLidar {
  uint32_t n = 0;                     // raw / undistorted points; the buffers below hold d_raw's size of them
  DeviceBuffer<malio_raw_pt> d_raw;
  DeviceBuffer<float> d_ud;           // n x 5: x, y, z, intensity (= idx as float, 0 where untouched), curvature
  DeviceBuffer<int32_t> d_need;
  DeviceBuffer<int32_t> d_idx;
  DeviceBuffer<uint8_t> d_ok;
  DeviceBuffer<double> d_pose;        // n x 7: the spline pose of every point (zeros where get_pose failed, and at point 0)
  DeviceBuffer<int32_t> d_pop;        // MALIO_MAX_COV + 1: pop points of the last malio_undistort (last = count)
  bool ud_valid = false;              // d_ud holds the result of a completed malio_undistort (possibly of 0 points)
  // what malio_scan_uncertainty needs of that call besides the device buffers
  uint32_t n_cov = 0, n_pops = 0;
  int32_t cov_pointer = -1;
  malio_rigid lt_imu_frame{};
  // voxel grid
  uint32_t n_ds = 0;
  DeviceBuffer<float> d_ds;           // n_ds x 5
  bool ds_valid = false;
};
struct PreState {
  cudaStream_t stream = nullptr;
  PreLidar lid[MALIO_MAX_LIDAR];
  DeviceBuffer<double> d_ct, d_cT, d_seglog, d_covt;
  // malio_scan_uncertainty: imu_cov (MALIO_MAX_COV x 36) and its one output buffer (table | temporal_comp | lidar_uncertainty)
  DeviceBuffer<double> d_ucov;
  DeviceBuffer<char> d_uout;
  // voxel scratch
  DeviceBuffer<float> d_vin;                          // host-provided input staged on the device
  DeviceBuffer<uint32_t> d_vidx, d_vtmp, d_vorder;    // per point
  DeviceBuffer<uint32_t> d_vcnt, d_voff, d_vocc, d_vcur;   // per cell
  DeviceBuffer<uint32_t> d_ctot, d_cbase;             // chunk totals / bases of the two cell scans (2 x 65536)
  DeviceBuffer<uint32_t> d_bounds;    // 6 order-preserving keys + out count
  DeviceBuffer<uint32_t> d_order_bad; // malio_undistort_device: raw_order_check_kernel's flag word
  // pinned, 8 words: the voxel grid's bounds and counts in [0..5]; malio_undistort_device's order flag and pop count in [6..7]
  PinnedBuffer<uint32_t> h_small;
  // the table malio_scan_uncertainty* left at the head of d_uout, for malio_upload_scan_resident: its offsets, the rigid part
  // of the temporal compensations, and whether it still describes the slots (any malio_undistort* since then clears it)
  bool table_resident = false;
  uint32_t res_table_off[MALIO_MAX_LIDAR + 1] = {0, 0, 0, 0};
  malio_rigid res_tcomp[MALIO_MAX_LIDAR] = {};
  // publish_frame_world / pcd_save (world registration): {x, y, z, intensity} per point
  DeviceBuffer<float4> d_wstage;      // malio_world_register's result before its one D2H copy
  DeviceBuffer<float4> d_acc; uint64_t n_acc = 0;   // pcl_wait_save (laserMapping.cpp:475), device-resident
  PinnedBuffer<float4> h_bounce;      // pinned, malio_pcd::CHUNK points: malio_world_save_pcd's D2H staging

  int init(malio_handle* h, DeviceState* D) {
    stream = D->stream;   // same stream as the scan path: malio_upload_scan_device is ordered after the voxel grid
    if (int rc = d_ct.allocate(h, stream, MALIO_MAX_CTRL)) return rc;
    if (int rc = d_cT.allocate(h, stream, (size_t)MALIO_MAX_CTRL * 16)) return rc;
    if (int rc = d_seglog.allocate(h, stream, (size_t)MALIO_MAX_CTRL * 6)) return rc;
    if (int rc = d_covt.allocate(h, stream, MALIO_MAX_COV)) return rc;
    if (int rc = d_bounds.allocate(h, stream, 8)) return rc;
    if (int rc = d_order_bad.allocate(h, stream, 1)) return rc;
    if (int rc = d_ctot.allocate(h, stream, 2 * 65536)) return rc;
    if (int rc = d_cbase.allocate(h, stream, 2 * 65536)) return rc;
    return h_small.allocate(h, 8);
  }
};

}  // namespace malio_pre

namespace {

using malio_pre::PreLidar;
using malio_pre::PreState;

// ------------------------------------------------------------------ quat_ops.h restated for the device
__host__ __device__ inline void mul3(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
// 4x4 homogeneous product in Eigen's coefficient order (k ascending, the bottom row 0 0 0 1 included)
__host__ __device__ inline void mul4(const double* A, const double* B, double* C) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = A[4 * i] * B[j];
      for (int k = 1; k < 4; ++k) s += A[4 * i + k] * B[4 * k + j];
      C[4 * i + j] = s;
    }
}
// quat_ops.h:150-187
__host__ __device__ inline void log_so3(const double R[9], double omega[3]) {
  const double R11 = R[0], R12 = R[1], R13 = R[2], R21 = R[3], R22 = R[4], R23 = R[5], R31 = R[6], R32 = R[7], R33 = R[8];
  const double tr = R11 + R22 + R33;
  const double PI = 3.14159265358979323846;
  if (tr + 1.0 < 1e-10) {
    if (fabs(R33 + 1.0) > 1e-5) {
      const double f = PI / sqrt(2.0 + 2.0 * R33);
      omega[0] = f * R13; omega[1] = f * R23; omega[2] = f * (1.0 + R33);
    } else if (fabs(R22 + 1.0) > 1e-5) {
      const double f = PI / sqrt(2.0 + 2.0 * R22);
      omega[0] = f * R12; omega[1] = f * (1.0 + R22); omega[2] = f * R32;
    } else {
      const double f = PI / sqrt(2.0 + 2.0 * R11);
      omega[0] = f * (1.0 + R11); omega[1] = f * R21; omega[2] = f * R31;
    }
  } else {
    double magnitude;
    const double tr_3 = tr - 3.0;
    if (tr_3 < -1e-7) {
      const double theta = acos((tr - 1.0) / 2.0);
      magnitude = theta / (2.0 * sin(theta));
    } else {
      magnitude = 0.5 - tr_3 / 12.0;
    }
    omega[0] = magnitude * (R32 - R23); omega[1] = magnitude * (R13 - R31); omega[2] = magnitude * (R21 - R12);
  }
}
// quat_ops.h:190-220
__host__ __device__ inline void exp_se3(const double vec[6], double mat[16]) {
  const double w0 = vec[0], w1 = vec[1], w2 = vec[2];
  const double theta = sqrt(w0 * w0 + w1 * w1 + w2 * w2);
  const double K[9] = {0, -w2, w1, w2, 0, -w0, -w1, w0, 0};
  double A, B, Cc;
  if (theta < 1e-7) { A = 1; B = 0.5; Cc = 1.0 / 6.0; }
  else { A = sin(theta) / theta; B = (1 - cos(theta)) / (theta * theta); Cc = (1 - A) / (theta * theta); }
  double K2[9];
  mul3(K, K, K2);
  double V[9];
  for (int i = 0; i < 9; ++i) {
    const double I = (i % 4 == 0) ? 1.0 : 0.0;
    V[i] = I + B * K[i] + Cc * K2[i];
    const double r = I + A * K[i] + B * K2[i];
    mat[4 * (i / 3) + (i % 3)] = r;
  }
  for (int i = 0; i < 3; ++i) mat[4 * i + 3] = V[3 * i] * vec[3] + V[3 * i + 1] * vec[4] + V[3 * i + 2] * vec[5];
  mat[12] = 0; mat[13] = 0; mat[14] = 0; mat[15] = 1;
}
// quat_ops.h:223-243
__host__ __device__ inline void log_se3(const double mat[16], double out[6]) {
  const double R[9] = {mat[0], mat[1], mat[2], mat[4], mat[5], mat[6], mat[8], mat[9], mat[10]};
  double w[3];
  log_so3(R, w);
  const double T[3] = {mat[3], mat[7], mat[11]};
  const double t = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  out[0] = w[0]; out[1] = w[1]; out[2] = w[2];
  if (t < 1e-10) { out[3] = T[0]; out[4] = T[1]; out[5] = T[2]; return; }
  const double a[3] = {w[0] / t, w[1] / t, w[2] / t};
  const double W[9] = {0, -a[2], a[1], a[2], 0, -a[0], -a[1], a[0], 0};
  const double Tan = tan(0.5 * t);
  double WT[3], WWT[3];
  for (int i = 0; i < 3; ++i) WT[i] = W[3 * i] * T[0] + W[3 * i + 1] * T[1] + W[3 * i + 2] * T[2];
  for (int i = 0; i < 3; ++i) WWT[i] = W[3 * i] * WT[0] + W[3 * i + 1] * WT[1] + W[3 * i + 2] * WT[2];
  for (int i = 0; i < 3; ++i) out[3 + i] = T[i] - (0.5 * t) * WT[i] + (1 - t / (2. * Tan)) * WWT[i];
}
// quat_ops.h:252-257
__host__ __device__ inline void inv_se3(const double T[16], double Ti[16]) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Ti[4 * i + j] = T[4 * j + i];
  for (int i = 0; i < 3; ++i) Ti[4 * i + 3] = -(Ti[4 * i] * T[3] + Ti[4 * i + 1] * T[7] + Ti[4 * i + 2] * T[11]);
  Ti[12] = 0; Ti[13] = 0; Ti[14] = 0; Ti[15] = 1;
}
// Eigen 3.3 QuaternionBase::operator=(rotation matrix) -> (w, x, y, z); m row-major 3x3
__host__ __device__ inline void quat_from_R(const double m[9], double q[4]) {
  double t = m[0] + m[4] + m[8];
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (m[7] - m[5]) * t;
    q[2] = (m[2] - m[6]) * t;
    q[3] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m[4 * i] - m[4 * j] - m[4 * k] + 1.0);
    double qv[3];
    qv[i] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[3 * k + j] - m[3 * j + k]) * t;
    qv[j] = (m[3 * j + i] + m[3 * i + j]) * t;
    qv[k] = (m[3 * k + i] + m[3 * i + k]) * t;
    q[1] = qv[0]; q[2] = qv[1]; q[3] = qv[2];
  }
}
// Eigen Quaternion * Vector3 (_transformVector), q = (w,x,y,z)
__host__ __device__ inline void q_rot(const double q[4], const double v[3], double o[3]) {
  const double uv0 = 2 * (q[2] * v[2] - q[3] * v[1]), uv1 = 2 * (q[3] * v[0] - q[1] * v[2]), uv2 = 2 * (q[1] * v[1] - q[2] * v[0]);
  const double c0 = q[2] * uv2 - q[3] * uv1, c1 = q[3] * uv0 - q[1] * uv2, c2 = q[1] * uv1 - q[2] * uv0;
  o[0] = v[0] + q[0] * uv0 + c0;
  o[1] = v[1] + q[0] * uv1 + c1;
  o[2] = v[2] + q[0] * uv2 + c2;
}
// BsplineSE3::find_bounding_control_points (BsplineSE3.cpp:120-231) on the ascending key array; i0..i3 on success
__host__ __device__ inline bool find_bounding(const double* ct, int n, double ts, int& i0, int& i1, int& i2, int& i3) {
  int lo = 0, hi = n;                 // lower_bound: first key >= ts
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (ct[mid] < ts) lo = mid + 1; else hi = mid; }
  const int lb = lo;
  lo = lb; hi = n;                    // upper_bound: first key > ts
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (ct[mid] <= ts) lo = mid + 1; else hi = mid; }
  const int ub = lo;
  bool older = false;
  i1 = -1;
  if (lb != n) {
    if (ct[lb] == ts) { i1 = lb; older = true; }
    else if (lb != 0) { i1 = lb - 1; older = true; }
  }
  if (!older || ub == n) return false;
  i2 = ub;
  if (i1 == 0) return false;
  i0 = i1 - 1; i3 = i2 + 1;
  return i3 != n;
}
// the spline pose from the per-pair logarithms (seglog[k] = log_se3(Inv(P_k) P_{k+1}))
__host__ __device__ inline bool spline_pose(const double* ct, const double* cT, const double* seglog, int n, double ts, double q[4], double p[3]) {
  int i0, i1, i2, i3;
  if (!find_bounding(ct, n, ts, i0, i1, i2, i3)) return false;
  const double t1 = ct[i1], t2 = ct[i2];
  const double DT = (t2 - t1);
  const double u = (ts - t1) / DT;
  const double b0 = 1.0 / 6.0 * (5 + 3 * u - 3 * u * u + u * u * u);
  const double b1 = 1.0 / 6.0 * (1 + 3 * u + 3 * u * u - 2 * u * u * u);
  const double b2 = 1.0 / 6.0 * (u * u * u);
  double l[6], A[16], m1[16], m2[16];
  for (int k = 0; k < 6; ++k) l[k] = b0 * seglog[6 * i0 + k];
  exp_se3(l, A);
  mul4(cT + 16 * i0, A, m1);
  for (int k = 0; k < 6; ++k) l[k] = b1 * seglog[6 * i1 + k];
  exp_se3(l, A);
  mul4(m1, A, m2);
  for (int k = 0; k < 6; ++k) l[k] = b2 * seglog[6 * i2 + k];
  exp_se3(l, A);
  mul4(m2, A, m1);
  const double R[9] = {m1[0], m1[1], m1[2], m1[4], m1[5], m1[6], m1[8], m1[9], m1[10]};
  quat_from_R(R, q);
  p[0] = m1[3]; p[1] = m1[7]; p[2] = m1[11];
  return true;
}

__global__ void seglog_kernel(const double* __restrict__ cT, int n, double* __restrict__ seglog) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k + 1 >= n) return;
  double ai[16], rel[16], l[6];
  inv_se3(cT + 16 * k, ai);
  mul4(ai, cT + 16 * (k + 1), rel);
  log_se3(rel, l);
  for (int j = 0; j < 6; ++j) seglog[6 * k + j] = l[j];
}

struct UdConst {
  double beg_time;
  double eq[4], et[3], lq[4], lt[3];
  int n_ctrl, n_cov, cov_pointer;
};
constexpr int UD_THREADS = 128;
__global__ void __launch_bounds__(UD_THREADS)
undistort_kernel(const malio_raw_pt* __restrict__ raw, uint32_t n, UdConst c, const double* __restrict__ ct,
                 const double* __restrict__ cT, const double* __restrict__ seglog, const double* __restrict__ covt,
                 float* __restrict__ ud, int32_t* __restrict__ need, uint8_t* __restrict__ ok, double* __restrict__ pose) {
  extern __shared__ double s_mem[];
  double* s_ct = s_mem;                       // n_ctrl
  double* s_cov = s_ct + c.n_ctrl;            // n_cov
  for (int k = threadIdx.x; k < c.n_ctrl; k += UD_THREADS) s_ct[k] = ct[k];
  for (int k = threadIdx.x; k < c.n_cov; k += UD_THREADS) s_cov[k] = covt[k];
  __syncthreads();
  const uint32_t i = blockIdx.x * UD_THREADS + threadIdx.x;
  if (i >= n) return;
  const malio_raw_pt pt = raw[i];
  float ox = pt.x, oy = pt.y, oz = pt.z;
  uint8_t flag = 0;
  int32_t nd = 0;
  if (i > 0) {                                // the reference's loop stops before begin(): point 0 is never touched
    const double point_t = (double)pt.curvature / double(1000) + c.beg_time;                   // :474
    double q[4], p[3];
    if (spline_pose(s_ct, cT, seglog, c.n_ctrl, point_t, q, p)) {                               // :475
      flag = 1;
      const double P_i[3] = {(double)pt.x, (double)pt.y, (double)pt.z};
      const double T_ei[3] = {p[0] - c.lt[0], p[1] - c.lt[1], p[2] - c.lt[2]};
      const double eqc[4] = {c.eq[0], -c.eq[1], -c.eq[2], -c.eq[3]}, lqc[4] = {c.lq[0], -c.lq[1], -c.lq[2], -c.lq[3]};
      double a[3], b[3], cc[3], d[3];
      q_rot(c.eq, P_i, a);                                                                      // :492
      a[0] += c.et[0]; a[1] += c.et[1]; a[2] += c.et[2];
      q_rot(q, a, b);
      b[0] += T_ei[0]; b[1] += T_ei[1]; b[2] += T_ei[2];
      q_rot(lqc, b, cc);
      cc[0] -= c.et[0]; cc[1] -= c.et[1]; cc[2] -= c.et[2];
      q_rot(eqc, cc, d);
      ox = (float)d[0]; oy = (float)d[1]; oz = (float)d[2];
      if (pose) { double* o = pose + 7 * (size_t)i; o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3]; o[4] = p[0]; o[5] = p[1]; o[6] = p[2]; }
    } else if (pose) {
      double* o = pose + 7 * (size_t)i;
      for (int k = 0; k < 7; ++k) o[k] = 0.0;
    }
    // entries k <= cov_pointer of the (ascending) list with time > point_t: what the walk may still pop at this point
    int lo = 0, hi = c.cov_pointer + 1;
    if (hi > c.n_cov) hi = c.n_cov;
    const int top = hi;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_cov[mid] <= point_t) lo = mid + 1; else hi = mid; }
    nd = top - lo;
  } else if (pose) {
    double* o = pose;
    for (int k = 0; k < 7; ++k) o[k] = 0.0;
  }
  float* o5 = ud + 5 * (size_t)i;
  o5[0] = ox; o5[1] = oy; o5[2] = oz; o5[4] = pt.curvature;   // [3] = intensity, written by the scan kernel
  need[i] = nd;
  ok[i] = flag;
}

// reverse-order min-plus scan (see the file header): one block, chunks of SCAN_T points, carry = running prefix minimum
constexpr int SCAN_T = 1024;
__global__ void __launch_bounds__(SCAN_T)
idx_scan_kernel(const int32_t* __restrict__ need, const uint8_t* __restrict__ ok, uint32_t n, float* __restrict__ ud,
                int32_t* __restrict__ idx_out, int32_t* __restrict__ pop_point, int n_cov) {
  __shared__ int32_t s_v[SCAN_T];
  __shared__ int32_t s_carry;
  if (threadIdx.x == 0) s_carry = 1;          // min(1, ...): pops_s <= s + 1
  for (int k = threadIdx.x; k <= n_cov; k += SCAN_T) pop_point[k] = (k == n_cov) ? 0 : -1;
  __syncthreads();
  const uint32_t steps = n > 0 ? n - 1 : 0;   // s = 0 .. n-2  <->  i = n-1 .. 1
  for (uint32_t base = 0; base < steps; base += SCAN_T) {
    const uint32_t s = base + threadIdx.x;
    const bool valid = s < steps;
    const uint32_t i = valid ? (n - 1 - s) : 0;
    int32_t v = valid ? (need[i] - (int32_t)s) : INT32_MAX;
    s_v[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < SCAN_T; o <<= 1) {    // inclusive prefix minimum
      const int32_t t = (threadIdx.x >= (unsigned)o) ? s_v[threadIdx.x - o] : INT32_MAX;
      __syncthreads();
      v = min(v, t);
      s_v[threadIdx.x] = v;
      __syncthreads();
    }
    const int32_t carry = s_carry;
    const int32_t m = min(carry, v);
    const int32_t m_prev = (threadIdx.x == 0) ? carry : min(carry, s_v[threadIdx.x - 1]);
    if (valid) {
      const int32_t pops = (int32_t)s + m;                                  // after processing this point
      const int32_t pops_prev = (s == 0) ? 0 : (int32_t)(s - 1) + m_prev;   // before it
      if (pops > pops_prev && pops - 1 < n_cov) pop_point[pops - 1] = (int32_t)i;
      const bool touched = ok[i] != 0;
      idx_out[i] = touched ? pops - 1 : INT32_MIN;                          // :496 only where spline_flag != 0
      ud[5 * (size_t)i + 3] = touched ? (float)(pops - 1) : 0.f;
    }
    __syncthreads();
    if (threadIdx.x == SCAN_T - 1) s_carry = m;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (n > 0) { idx_out[0] = INT32_MIN; ud[3] = 0.f; }
    const int32_t total = steps ? (int32_t)(steps - 1) + s_carry : 0;
    pop_point[n_cov] = total < 0 ? 0 : total;
  }
}

// malio_undistort_device's time-order check, malio_undistort's host loop on device memory: point i >= 1 is out of order when
// its time is below its predecessor's (the same comparison, so a NaN time passes exactly where the host loop lets it pass).
// A warp with such a point ORs 1 into *bad.  Only the time word of each 16-byte record is read.
__global__ void __launch_bounds__(256) raw_order_check_kernel(const malio_raw_pt* __restrict__ raw, uint32_t n, uint32_t* __restrict__ bad) {
  const uint32_t i = blockIdx.x * 256u + threadIdx.x;
  const bool b = i >= 1 && i < n && raw[i].curvature < raw[i - 1].curvature;
  if (__any_sync(0xFFFFFFFFu, b) && (threadIdx.x & 31u) == 0) atomicOr(bad, 1u);
}

// ------------------------------------------------------------------ N3: voxel grid
__device__ __forceinline__ uint32_t fkey(float f) {   // order-preserving float -> uint32
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ inline float fkey_inv(uint32_t k) {
  const uint32_t b = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
  float f;
  memcpy(&f, &b, 4);
  return f;
}
__global__ void __launch_bounds__(256) vg_bounds_kernel(const float* __restrict__ in, uint32_t n, uint32_t* __restrict__ keys) {
  // getMinMax3D over the finite points: grid-stride, one set of atomics per block
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n; i += gridDim.x * 256u) {
    const float x = in[5 * (size_t)i], y = in[5 * (size_t)i + 1], z = in[5 * (size_t)i + 2];
    if (isfinite(x) && isfinite(y) && isfinite(z)) {
      lo[0] = fminf(lo[0], x); hi[0] = fmaxf(hi[0], x); lo[1] = fminf(lo[1], y); hi[1] = fmaxf(hi[1], y); lo[2] = fminf(lo[2], z); hi[2] = fmaxf(hi[2], z);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
      hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
    }
  __shared__ float s_lo[8][3], s_hi[8][3];
  if ((threadIdx.x & 31) == 0) for (int k = 0; k < 3; ++k) { s_lo[threadIdx.x >> 5][k] = lo[k]; s_hi[threadIdx.x >> 5][k] = hi[k]; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < 8; ++w) for (int k = 0; k < 3; ++k) { lo[k] = fminf(lo[k], s_lo[w][k]); hi[k] = fmaxf(hi[k], s_hi[w][k]); }
    if (lo[0] <= hi[0]) for (int k = 0; k < 3; ++k) { atomicMin(keys + k, fkey(lo[k])); atomicMax(keys + 3 + k, fkey(hi[k])); }
  }
}
struct VgConst { float il; int minb[3]; long long dx, dxy; };
__global__ void vg_count_kernel(const float* __restrict__ in, uint32_t n, VgConst c, uint32_t* __restrict__ vidx,
                                uint32_t* __restrict__ cnt) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = in[5 * (size_t)i], y = in[5 * (size_t)i + 1], z = in[5 * (size_t)i + 2];
  if (!(isfinite(x) && isfinite(y) && isfinite(z))) { vidx[i] = 0xFFFFFFFFu; return; }
  // static_cast<int>(std::floor(p.x * inverse_leaf_size_[0]) - static_cast<float>(min_b_[0]))   (voxel_grid.hpp)
  const int a = (int)(floorf(x * c.il) - (float)c.minb[0]);
  const int b = (int)(floorf(y * c.il) - (float)c.minb[1]);
  const int d = (int)(floorf(z * c.il) - (float)c.minb[2]);
  const uint32_t v = (uint32_t)((long long)a + (long long)b * c.dx + (long long)d * c.dxy);
  vidx[i] = v;
  atomicAdd(cnt + v, 1u);
}
// exclusive scan of count[] (-> off) and of (count != 0) (-> occ) over `cells` entries: chunk-local pass, chunk totals,
// add-back (two quantities side by side)
constexpr int VS_T = 1024, VS_PER = 4, VS_CHUNK = VS_T * VS_PER;
__global__ void __launch_bounds__(VS_T) vg_scan_local_kernel(const uint32_t* __restrict__ cnt, uint64_t cells, uint32_t* __restrict__ off,
                                                             uint32_t* __restrict__ occ, uint32_t* __restrict__ ctot) {
  __shared__ uint32_t s_a[32], s_b[32];
  const uint64_t base = ((uint64_t)blockIdx.x * VS_T + threadIdx.x) * VS_PER;
  uint32_t v[VS_PER], sa = 0, sb = 0;
#pragma unroll
  for (int k = 0; k < VS_PER; ++k) { v[k] = (base + k < cells) ? cnt[base + k] : 0u; sa += v[k]; sb += v[k] != 0; }
  uint32_t ia = sa, ib = sb;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o);
    if ((threadIdx.x & 31) >= (unsigned)o) { ia += ta; ib += tb; }
  }
  if ((threadIdx.x & 31) == 31) { s_a[threadIdx.x >> 5] = ia; s_b[threadIdx.x >> 5] = ib; }
  __syncthreads();
  if (threadIdx.x < 32) {
    const uint32_t wa = s_a[threadIdx.x], wb = s_b[threadIdx.x];
    uint32_t xa = wa, xb = wb;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ta = __shfl_up_sync(0xffffffffu, xa, o), tb = __shfl_up_sync(0xffffffffu, xb, o);
      if (threadIdx.x >= (unsigned)o) { xa += ta; xb += tb; }
    }
    s_a[threadIdx.x] = xa - wa; s_b[threadIdx.x] = xb - wb;
    if (threadIdx.x == 31) { ctot[2 * blockIdx.x] = xa; ctot[2 * blockIdx.x + 1] = xb; }
  }
  __syncthreads();
  uint32_t ra = s_a[threadIdx.x >> 5] + ia - sa, rb = s_b[threadIdx.x >> 5] + ib - sb;
#pragma unroll
  for (int k = 0; k < VS_PER; ++k) {
    if (base + k < cells) { off[base + k] = ra; occ[base + k] = rb; }
    ra += v[k]; rb += v[k] != 0;
  }
}
__global__ void __launch_bounds__(1024) vg_scan_tot_kernel(const uint32_t* __restrict__ ctot, uint32_t nchunk, uint32_t* __restrict__ cbase,
                                                           uint32_t* __restrict__ totals) {
  // nchunk <= 65536: each of 1024 threads owns 64 consecutive chunks
  __shared__ uint32_t s_a[32], s_b[32];
  uint32_t sa = 0, sb = 0;
  const uint32_t b0 = threadIdx.x * 64;
  for (uint32_t k = 0; k < 64; ++k) { const uint32_t c = b0 + k; if (c < nchunk) { sa += ctot[2 * c]; sb += ctot[2 * c + 1]; } }
  uint32_t ia = sa, ib = sb;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o);
    if ((threadIdx.x & 31) >= (unsigned)o) { ia += ta; ib += tb; }
  }
  if ((threadIdx.x & 31) == 31) { s_a[threadIdx.x >> 5] = ia; s_b[threadIdx.x >> 5] = ib; }
  __syncthreads();
  uint32_t wa = 0, wb = 0;
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) { wa += s_a[w]; wb += s_b[w]; }
  uint32_t ra = wa + ia - sa, rb = wb + ib - sb;
  for (uint32_t k = 0; k < 64; ++k) {
    const uint32_t c = b0 + k;
    if (c < nchunk) { cbase[2 * c] = ra; cbase[2 * c + 1] = rb; ra += ctot[2 * c]; rb += ctot[2 * c + 1]; }
  }
  if (threadIdx.x == 1023) { totals[0] = ra; totals[1] = rb; }   // points binned, occupied voxels
}
__global__ void __launch_bounds__(VS_T) vg_scan_add_kernel(uint32_t* __restrict__ off, uint32_t* __restrict__ occ, uint64_t cells,
                                                           const uint32_t* __restrict__ cbase) {
  const uint64_t base = ((uint64_t)blockIdx.x * VS_T + threadIdx.x) * VS_PER;
  const uint32_t a = cbase[2 * blockIdx.x], b = cbase[2 * blockIdx.x + 1];
#pragma unroll
  for (int k = 0; k < VS_PER; ++k) if (base + k < cells) { off[base + k] += a; occ[base + k] += b; }
}
__global__ void vg_scatter_kernel(const uint32_t* __restrict__ vidx, uint32_t n, const uint32_t* __restrict__ off,
                                  uint32_t* __restrict__ cursor, uint32_t* __restrict__ tmp) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = vidx[i];
  if (v == 0xFFFFFFFFu) return;
  tmp[off[v] + atomicAdd(cursor + v, 1u)] = i;
}
// each point finds its rank among its voxel-mates by input index (deterministic order inside a voxel) ...
__global__ void vg_rank_kernel(const uint32_t* __restrict__ vidx, uint32_t n, const uint32_t* __restrict__ off,
                               const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ tmp, uint32_t* __restrict__ order) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = vidx[i];
  if (v == 0xFFFFFFFFu) return;
  const uint32_t o = off[v], c = cnt[v];
  uint32_t r = 0;
  for (uint32_t j = 0; j < c; ++j) r += (tmp[o + j] < i) ? 1u : 0u;
  order[o + r] = i;
}
// ... and the first point of every voxel sums the voxel's run sequentially (float, ascending input index: the order a
// stable sort would give PCL's centroid accumulator) and writes the centroid at the voxel's rank among the occupied ones
__global__ void vg_centroid_kernel(const float* __restrict__ in, const uint32_t* __restrict__ vidx, uint32_t n,
                                   const uint32_t* __restrict__ off, const uint32_t* __restrict__ cnt,
                                   const uint32_t* __restrict__ occ, const uint32_t* __restrict__ order,
                                   float* __restrict__ out, uint32_t out_cap) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = vidx[i];
  if (v == 0xFFFFFFFFu) return;
  const uint32_t o = off[v];
  if (order[o] != i) return;
  const uint32_t c = cnt[v], slot = occ[v];
  if (slot >= out_cap) return;
  float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (uint32_t j = 0; j < c; ++j) {
    const float* p = in + 5 * (size_t)order[o + j];
#pragma unroll
    for (int f = 0; f < 5; ++f) acc[f] += p[f];
  }
  const float cf = (float)c;
#pragma unroll
  for (int f = 0; f < 5; ++f) out[5 * (size_t)slot + f] = acc[f] / cf;
}
__global__ void merge_scan_kernel(const float* __restrict__ ds, uint32_t n, uint16_t lidar, malio_scan_pt* __restrict__ dst) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = ds + 5 * (size_t)i;
  malio_scan_pt o;
  o.x = p[0]; o.y = p[1]; o.z = p[2];
  o.lidar = lidar;                                   // laserMapping.cpp:976
  const int t = (int)p[3];                           // normal_x = averaged intensity (:975), int() at :694/:737
  o.table_idx = (uint16_t)(t < 0 ? 0 : (t > 65535 ? 65535 : t));
  dst[i] = o;
}

// ------------------------------------------------------------------ publish_frame_world: RGBpointBodyToWorld per point
// laserMapping.cpp:149-163 over one of publish_frame_world's two clouds (:452), output {x, y, z, intensity} (16 B) per point:
//   ud != NULL  dense (feats_undistort, :977-981): n x 5 undistorted records of LiDAR slot `slot`; lid = slot (:979),
//               intensity = the raw points' normal_y, one value per slot (`tag`, set by sync_packages, :321-322)
//   ud == NULL  down-sampled (feats_down_body): the scan in the library's position order; lid = its lidar field (:976),
//               intensity = normal_y of the last pass (:699, :730, :741); written in caller order through perm
__global__ void world_kernel(const float* __restrict__ ud, int slot, float tag, const malio_scan_pt* __restrict__ pts,
                             const uint32_t* __restrict__ perm, const float* __restrict__ normal_y, uint32_t n, PassConst pc,
                             float4* __restrict__ out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  float w[3];
  if (ud) {
    const float* r = ud + 5 * (size_t)p;
    body_to_world(pc, slot, r[0], r[1], r[2], w);
    out[p] = make_float4(w[0], w[1], w[2], tag);
  } else {
    const malio_scan_pt pt = pts[p];
    body_to_world(pc, pt.lidar, pt.x, pt.y, pt.z, w);
    out[perm ? perm[p] : p] = make_float4(w[0], w[1], w[2], normal_y[p]);
  }
}

constexpr uint64_t WORLD_ACC_MIN = 1u << 16;   // first capacity of the accumulated cloud (points); it doubles from there

// d_wstage large enough for n points
int grow_wstage(malio_handle* h, PreState* S, uint64_t n) {
  if (n <= S->d_wstage.size()) return MALIO_OK;
  return S->d_wstage.allocate(h, S->stream, n + n / 8 + 1024);
}

// size of the cloud `source` registers, or a state error when it is not on the device
int world_count(malio_handle* h, PreState* S, DeviceState* D, int source, uint64_t& n) {
  n = 0;
  if (source == MALIO_WORLD_DENSE) {
    for (int l = 0; l < h->cfg.params.n_lidar; ++l) {
      if (!S->lid[l].ud_valid) { h->err = "world registration (dense): malio_undistort has not run on every LiDAR slot 0..L-1"; return MALIO_ERR_STATE; }
      n += S->lid[l].n;
    }
    return MALIO_OK;
  }
  if (!D->pass_done) { h->err = "world registration (down-sampled): no measurement pass on the current scan"; return MALIO_ERR_STATE; }
  n = D->N;
  return MALIO_OK;
}

// enqueue the registration of `source` into dst[0 .. n) on the handle's stream
int world_launch(malio_handle* h, PreState* S, DeviceState* D, const malio_pass_state* s, int source, const float* slot_tag,
                 float4* dst) {
  const PassConst pc = make_pass_const(h, D, s);   // body_to_world reads the state and the temporal compensation
  if (source == MALIO_WORLD_DENSE) {
    uint64_t at = 0;
    for (int l = 0; l < h->cfg.params.n_lidar; ++l) {
      const uint32_t m = S->lid[l].n;
      if (m) {
        world_kernel<<<(m + 255) / 256, 256, 0, S->stream>>>(S->lid[l].d_ud, l, slot_tag[l], nullptr, nullptr, nullptr, m, pc, dst + at);
        D->ctr.kernel_launches += 1;
      }
      at += m;
    }
  } else if (D->N) {
    const bool sorted = h->cfg.sort_queries && D->perm_valid;
    world_kernel<<<(D->N + 255) / 256, 256, 0, S->stream>>>(nullptr, 0, 0.f, sorted ? D->d_pts_sorted : D->d_pts,
                                                           sorted ? D->d_perm.data() : nullptr, D->d_normal_y, D->N, pc, dst);
    D->ctr.kernel_launches += 1;
  }
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}

// ------------------------------------------------------------------ N2, second half: the scan's pose-uncertainty lists
// IMU_Processing.hpp:474-523 and laserMapping.cpp:1028-1048 after malio_undistort has run on every slot.  One thread per
// (slot, pop k): uncertainty[num][k] from the spline pose undistort_kernel computed for the k-th pop point (:483, :487-492),
// then, unless it is the slot's last entry (:1035, :1040), its pose_unc entry.  Every slot has at least one thread; the
// slot's first thread writes temporal_comp[num - 1] (:518), which each thread of the slot computes for itself: the same code
// on the same inputs, so the same bits, and no second launch.
struct UncConst {
  malio_pose ext[MALIO_MAX_LIDAR];    // extrinsic[num] (:448)
  malio_pose ltl[MALIO_MAX_LIDAR];    // lt_lidar_frame[num] (:450, :471)
  const int32_t* pop[MALIO_MAX_LIDAR];
  const double* pose[MALIO_MAX_LIDAR];
  const uint8_t* ok[MALIO_MAX_LIDAR];
  int32_t cov_pointer[MALIO_MAX_LIDAR], n_pops[MALIO_MAX_LIDAR];
  uint32_t first[MALIO_MAX_LIDAR + 1];  // slot s owns threads [first[s], first[s + 1])
  uint32_t unc_off[MALIO_MAX_LIDAR], tab_off[MALIO_MAX_LIDAR];
  int L;
};
constexpr int UNC_THREADS = 64;
__global__ void __launch_bounds__(UNC_THREADS)
scan_unc_kernel(const UncConst c, const double* __restrict__ imu_cov, malio_pose_entry* __restrict__ tab, malio_pose* __restrict__ tc_out,
                malio_pose* __restrict__ unc) {
  using namespace malio_compound;
  const uint32_t g = blockIdx.x * UNC_THREADS + threadIdx.x;
  if (g >= c.first[c.L]) return;
  int num = 0;
  while (g >= c.first[num + 1]) ++num;
  const int k = (int)(g - c.first[num]);
  malio_pose tcomp{};
  if (num != 0) {
    compound_inv_pose_with_cov(&c.ltl[0], c.ltl[0].cov, &c.ltl[num], c.ltl[num].cov, &tcomp, tcomp.cov);   // :518
    if (k == 0) tc_out[num - 1] = tcomp;
  }
  if (k >= c.n_pops[num]) return;
  // the pose that compensated the pop point; where get_pose failed, the identity it sets up (BsplineSE3.cpp:93-95)
  const int32_t i = c.pop[num][k];
  double q[4] = {1.0, 0.0, 0.0, 0.0}, t[3] = {0.0, 0.0, 0.0};
  if (c.ok[num][i]) {
    const double* o = c.pose[num] + 7 * (size_t)i;
    for (int j = 0; j < 4; ++j) q[j] = o[j];
    for (int j = 0; j < 3; ++j) t[j] = o[4 + j];
  }
  malio_pose pt, pc{};
  pose_initial(&pt, t, q, imu_cov + 36 * (size_t)(c.cov_pointer[num] - k));                                   // :488
  compound_pose_with_cov(&pt, pt.cov, &c.ext[num], c.ext[num].cov, &pc, pc.cov);                              // :489
  compound_inv_pose_with_cov(&c.ltl[num], c.ltl[num].cov, &pc, pc.cov, &pc, pc.cov);                          // :490
  compound_inv_pose_with_cov(&c.ext[num], c.ext[num].cov, &pc, pc.cov, &pc, pc.cov);                          // :491
  unc[c.unc_off[num] + k] = pc;
  if (k < c.n_pops[num] - 1) pose_unc_entry(num, c.ext, &tcomp, &pc, &tab[c.tab_off[num] + k]);
}

// ---- malio_undistort and malio_undistort_device share three steps: the argument checks, the slot's preparation, the launches
int undistort_check_args(malio_handle* h, int lidar, const malio_undistort_args* a) {
  if (lidar < 0 || lidar >= MALIO_MAX_LIDAR) { h->err = "lidar slot out of range"; return MALIO_ERR_INVALID_ARG; }
  if (a->n_ctrl > MALIO_MAX_CTRL || a->n_cov > MALIO_MAX_COV) { h->err = "too many control points / covariance entries"; return MALIO_ERR_CAPACITY; }
  for (uint32_t k = 1; k < a->n_ctrl; ++k) if (!(a->ctrl_t[k] > a->ctrl_t[k - 1])) { h->err = "control-point times must ascend"; return MALIO_ERR_INVALID_ARG; }
  for (uint32_t k = 1; k < a->n_cov; ++k) if (!(a->imu_cov_t[k] >= a->imu_cov_t[k - 1])) { h->err = "imu_cov times must ascend"; return MALIO_ERR_INVALID_ARG; }
  if (a->cov_pointer < -1 || a->cov_pointer >= (int32_t)a->n_cov) { h->err = "cov_pointer outside the list"; return MALIO_ERR_INVALID_ARG; }
  return MALIO_OK;
}

// the slot takes the call's sizes and arguments and holds no valid result until the caller sets ud_valid; buffers grown for n
int undistort_prepare_slot(malio_handle* h, PreState* S, PreLidar& L, uint32_t n, const malio_undistort_args* a) {
  L.ud_valid = false;
  S->table_resident = false;   // the table in d_uout was built from this slot's previous undistortion
  if (n > L.d_raw.size()) {
    const uint32_t cap = n + n / 8 + 1024;
    if (int rc = malio_buf::allocate_group(h, S->stream, {{L.d_raw, cap}, {L.d_ud, (size_t)cap * 5}, {L.d_need, cap}, {L.d_idx, cap},
                                                          {L.d_ok, cap}, {L.d_pose, (size_t)cap * 7}}))
      return rc;
  }
  if (!L.d_pop) { if (int rc = L.d_pop.allocate(h, S->stream, MALIO_MAX_COV + 1)) return rc; }
  L.n = n;
  L.ds_valid = false;
  L.n_cov = a->n_cov;
  L.cov_pointer = a->cov_pointer;
  L.lt_imu_frame = a->lt_imu_frame;
  L.n_pops = 0;
  return MALIO_OK;
}

// control points and IMU times to the device, then the three kernels over d_raw[0 .. n), n > 0 (the slot's d_raw, or the
// caller's device array read in place); results in the slot's buffers
int undistort_launch(malio_handle* h, PreState* S, DeviceState* D, PreLidar& L, const malio_raw_pt* d_raw, uint32_t n,
                     const malio_undistort_args* a) {
  cudaStream_t st = S->stream;
  CUDA_TRY(cudaMemcpyAsync(S->d_ct, a->ctrl_t, a->n_ctrl * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(S->d_cT, a->ctrl_T, (size_t)a->n_ctrl * 16 * sizeof(double), cudaMemcpyHostToDevice, st));
  if (a->n_cov) CUDA_TRY(cudaMemcpyAsync(S->d_covt, a->imu_cov_t, a->n_cov * sizeof(double), cudaMemcpyHostToDevice, st));
  UdConst c{};
  c.beg_time = a->beg_time;
  std::memcpy(c.eq, a->extrinsic.q, sizeof(c.eq)); std::memcpy(c.et, a->extrinsic.t, sizeof(c.et));
  std::memcpy(c.lq, a->lt_imu_frame.q, sizeof(c.lq)); std::memcpy(c.lt, a->lt_imu_frame.t, sizeof(c.lt));
  c.n_ctrl = (int)a->n_ctrl; c.n_cov = (int)a->n_cov; c.cov_pointer = a->cov_pointer;
  if (a->n_ctrl > 1) seglog_kernel<<<(a->n_ctrl + 63) / 64, 64, 0, st>>>(S->d_cT, (int)a->n_ctrl, S->d_seglog);
  const size_t smem = (size_t)(a->n_ctrl + a->n_cov) * sizeof(double);
  undistort_kernel<<<(n + UD_THREADS - 1) / UD_THREADS, UD_THREADS, smem, st>>>(d_raw, n, c, S->d_ct, S->d_cT, S->d_seglog, S->d_covt,
                                                                                  L.d_ud, L.d_need, L.d_ok, L.d_pose);
  idx_scan_kernel<<<1, SCAN_T, 0, st>>>(L.d_need, L.d_ok, n, L.d_ud, L.d_idx, L.d_pop, (int)a->n_cov);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 3;
  D->ctr.h2d_bytes += (uint64_t)a->n_ctrl * 17 * 8 + (uint64_t)a->n_cov * 8;
  return MALIO_OK;
}

}  // namespace

namespace malio_pre {

int undistort(malio_handle* h, int lidar, const malio_raw_pt* pts, uint32_t n, const malio_undistort_args* a, float* xyz,
              int32_t* idx, uint8_t* ok, int32_t* pop_point, uint32_t* n_pops, double* pose) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  if (int rc = undistort_check_args(h, lidar, a)) return rc;
  PreLidar& L = S->lid[lidar];
  cudaStream_t st = S->stream;
  if (int rc = undistort_prepare_slot(h, S, L, n, a)) return rc;
  if (n == 0) { if (n_pops) *n_pops = 0; L.ud_valid = true; return MALIO_OK; }
  CUDA_TRY(cudaMemcpyAsync(L.d_raw, pts, (size_t)n * sizeof(malio_raw_pt), cudaMemcpyHostToDevice, st));
  D->ctr.h2d_bytes += (uint64_t)n * sizeof(malio_raw_pt);
  if (int rc = undistort_launch(h, S, D, L, L.d_raw, n, a)) return rc;
  std::vector<float> ud_host;
  if (xyz) ud_host.resize((size_t)n * 5);
  std::vector<int32_t> pops(a->n_cov + 1);
  if (xyz) CUDA_TRY(cudaMemcpyAsync(ud_host.data(), L.d_ud, (size_t)n * 5 * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (idx) CUDA_TRY(cudaMemcpyAsync(idx, L.d_idx, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (ok) CUDA_TRY(cudaMemcpyAsync(ok, L.d_ok, (size_t)n, cudaMemcpyDeviceToHost, st));
  if (pose) CUDA_TRY(cudaMemcpyAsync(pose, L.d_pose, (size_t)n * 7 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(pops.data(), L.d_pop, (a->n_cov + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (xyz) for (uint32_t i = 0; i < n; ++i) { xyz[3 * (size_t)i] = ud_host[5 * (size_t)i]; xyz[3 * (size_t)i + 1] = ud_host[5 * (size_t)i + 1]; xyz[3 * (size_t)i + 2] = ud_host[5 * (size_t)i + 2]; }
  if (pop_point) std::memcpy(pop_point, pops.data(), a->n_cov * sizeof(int32_t));
  if (n_pops) *n_pops = (uint32_t)pops[a->n_cov];
  L.n_pops = (uint32_t)pops[a->n_cov];
  D->ctr.d2h_bytes += (uint64_t)n * ((xyz ? 20 : 0) + (idx ? 4 : 0) + (ok ? 1 : 0) + (pose ? 56 : 0));
  L.ud_valid = true;
  return MALIO_OK;
}

// malio_undistort on a raw cloud in device memory, ordered on the caller's stream.  The cloud is read where it is by the order
// check and by undistort_kernel; the slot's d_raw is not used.  The check's verdict and the pop count are fetched together
// behind the kernels, so the host waits once.  That is safe on a cloud that turns out to be unordered: undistort_kernel treats
// every point on its own (need = entries of the list above the point's time, in [0, n_cov] whatever the order), and in
// idx_scan_kernel pops_s = s + min(1, min_{j<=s}(need_j - j)) lies in [0, need_s], so pop_point is written at pops - 1 < n_cov
// only and everything else at a point's own index.  Such a cloud leaves the slot without a valid result.
int undistort_device(malio_handle* h, int lidar, const malio_raw_pt* pts, uint32_t n, const malio_undistort_args* a, float* cloud,
                     int32_t* idx, uint8_t* ok, int32_t* pop_point, double* pose, uint32_t* n_pops, cudaStream_t caller) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  if (int rc = undistort_check_args(h, lidar, a)) return rc;
  if (n) {
    if (int rc = check_device_ptr(h, D, pts, "malio_undistort_device pts")) return rc;
    if (int rc = check_device_ptrs(h, D, {{cloud, "malio_undistort_device cloud"}, {idx, "malio_undistort_device idx"},
                                          {ok, "malio_undistort_device ok"}, {a->n_cov ? pop_point : nullptr, "malio_undistort_device pop_point"},
                                          {pose, "malio_undistort_device pose"}}))
      return rc;
  }
  PreLidar& L = S->lid[lidar];
  cudaStream_t st = S->stream;
  if (int rc = undistort_prepare_slot(h, S, L, n, a)) return rc;
  if (n == 0) { if (n_pops) *n_pops = 0; L.ud_valid = true; return MALIO_OK; }
  if (int rc = caller_enter(h, D, caller)) return rc;
  CUDA_TRY(cudaMemsetAsync(S->d_order_bad, 0, sizeof(uint32_t), st));
  raw_order_check_kernel<<<(n + 255) / 256, 256, 0, st>>>(pts, n, S->d_order_bad);
  D->ctr.kernel_launches += 1;
  if (int rc = undistort_launch(h, S, D, L, pts, n, a)) return rc;
  if (cloud) CUDA_TRY(cudaMemcpyAsync(cloud, L.d_ud, (size_t)n * 5 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (idx) CUDA_TRY(cudaMemcpyAsync(idx, L.d_idx, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  if (ok) CUDA_TRY(cudaMemcpyAsync(ok, L.d_ok, (size_t)n, cudaMemcpyDeviceToDevice, st));
  if (pop_point && a->n_cov) CUDA_TRY(cudaMemcpyAsync(pop_point, L.d_pop, a->n_cov * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  if (pose) CUDA_TRY(cudaMemcpyAsync(pose, L.d_pose, (size_t)n * 7 * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (int rc = caller_leave(h, D, caller)) return rc;   // the copies are the last access to the caller's arrays
  CUDA_TRY(cudaMemcpyAsync(S->h_small + 6, S->d_order_bad, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(S->h_small + 7, L.d_pop + a->n_cov, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (S->h_small[6]) { h->err = "malio_undistort: points must be sorted by curvature (IMU_Processing.hpp:232)"; return MALIO_ERR_INVALID_ARG; }
  L.n_pops = S->h_small[7];
  if (n_pops) *n_pops = L.n_pops;
  L.ud_valid = true;
  return MALIO_OK;
}

// the filter over d_in[0 .. n) (device memory: the slot's undistorted cloud, the staged host input or the caller's device
// array), shared by malio_voxel_grid and malio_voxel_grid_device.  Waits twice, for the grid geometry and for the output count
// (they size allocations), and returns with vg_centroid_kernel enqueued: the result is the slot's d_ds, n_ds rows.
static int voxel_grid_run(malio_handle* h, PreState* S, DeviceState* D, PreLidar& L, const float* d_in, uint32_t n, float leaf,
                          uint32_t* n_out) {
  cudaStream_t st = S->stream;
  L.ds_valid = false;
  L.n_ds = 0;
  if (n_out) *n_out = 0;
  if (n == 0) { L.ds_valid = true; return MALIO_OK; }
  if (n > S->d_vidx.size()) {
    const uint32_t cap = n + n / 8 + 1024;
    if (int rc = malio_buf::allocate_group(h, st, {{S->d_vidx, cap}, {S->d_vtmp, cap}, {S->d_vorder, cap}})) return rc;
  }
  // ---- bounds (getMinMax3D), then the grid geometry on the host exactly as PCL derives it
  const uint32_t init[6] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u, 0u};
  CUDA_TRY(cudaMemcpyAsync(S->d_bounds, init, sizeof(init), cudaMemcpyHostToDevice, st));
  vg_bounds_kernel<<<(n + 255) / 256 < 296u ? (n + 255) / 256 : 296u, 256, 0, st>>>(d_in, n, S->d_bounds);
  CUDA_TRY(cudaMemcpyAsync(S->h_small, S->d_bounds, 6 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  D->ctr.kernel_launches += 1;
  if (S->h_small[0] == 0xFFFFFFFFu) { L.ds_valid = true; return MALIO_OK; }   // no finite point
  VgConst c{};
  c.il = 1.0f / leaf;
  int maxb[3];
  for (int k = 0; k < 3; ++k) {
    const float lo = std::floor(fkey_inv(S->h_small[k]) * c.il), hi = std::floor(fkey_inv(S->h_small[3 + k]) * c.il);
    if (!(lo >= -2147483648.f && hi < 2147483648.f)) {   // x / leaf outside int (or infinite): PCL's int cast is undefined there
      h->err = "voxel_grid: leaf size too small for the cloud's coordinates (voxel index outside int)";
      return MALIO_ERR_CAPACITY;
    }
    c.minb[k] = (int)lo;
    maxb[k] = (int)hi;
  }
  const long long dx = (long long)maxb[0] - c.minb[0] + 1, dy = (long long)maxb[1] - c.minb[1] + 1, dz = (long long)maxb[2] - c.minb[2] + 1;
  const long long cells = dx * dy * dz;
  // PCL's per-axis index floor(x / leaf) - (float)min_b is a float subtraction: exact up to 2^24 voxels per axis, above that
  // it can round up to the axis' size and the point would be counted one cell past the grid
  if (dx > (1ll << 24) || dy > (1ll << 24) || dz > (1ll << 24)) {
    h->err = "voxel_grid: leaf size too small for the cloud's extent (more than 2^24 voxels along an axis)";
    return MALIO_ERR_CAPACITY;
  }
  if (cells <= 0 || cells > (1ll << 28)) {   // PCL gives up (returns the input) above INT_MAX voxels; the dense index here stops at 2^28
    h->err = "voxel_grid: leaf size too small for the cloud's extent (more than 2^28 voxels)";
    return MALIO_ERR_CAPACITY;
  }
  c.dx = dx; c.dxy = dx * dy;
  if ((uint64_t)cells > S->d_vcnt.size()) {
    const uint64_t cap = (uint64_t)cells + (uint64_t)cells / 4 + 4096;
    if (int rc = malio_buf::allocate_group(h, st, {{S->d_vcnt, cap}, {S->d_voff, cap}, {S->d_vocc, cap}, {S->d_vcur, cap}})) return rc;
  }
  const uint32_t nchunk = (uint32_t)((cells + VS_CHUNK - 1) / VS_CHUNK);   // <= 65536
  CUDA_TRY(cudaMemsetAsync(S->d_vcnt, 0, (size_t)cells * sizeof(uint32_t), st));
  CUDA_TRY(cudaMemsetAsync(S->d_vcur, 0, (size_t)cells * sizeof(uint32_t), st));
  vg_count_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_in, n, c, S->d_vidx, S->d_vcnt);
  vg_scan_local_kernel<<<nchunk, VS_T, 0, st>>>(S->d_vcnt, (uint64_t)cells, S->d_voff, S->d_vocc, S->d_ctot);
  vg_scan_tot_kernel<<<1, 1024, 0, st>>>(S->d_ctot, nchunk, S->d_cbase, S->d_bounds + 6);
  vg_scan_add_kernel<<<nchunk, VS_T, 0, st>>>(S->d_voff, S->d_vocc, (uint64_t)cells, S->d_cbase);
  vg_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(S->d_vidx, n, S->d_voff, S->d_vcur, S->d_vtmp);
  vg_rank_kernel<<<(n + 255) / 256, 256, 0, st>>>(S->d_vidx, n, S->d_voff, S->d_vcnt, S->d_vtmp, S->d_vorder);
  CUDA_TRY(cudaMemcpyAsync(S->h_small, S->d_bounds + 6, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  const uint32_t m = S->h_small[1];
  if (m > L.d_ds.size() / 5) { if (int rc = L.d_ds.allocate(h, st, (size_t)(m + m / 8 + 1024) * 5)) return rc; }
  vg_centroid_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_in, S->d_vidx, n, S->d_voff, S->d_vcnt, S->d_vocc, S->d_vorder, L.d_ds, m);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 7;
  L.n_ds = m;
  L.ds_valid = true;
  if (n_out) *n_out = m;
  return MALIO_OK;
}

// the slot's own cloud as the filter's input.  A slot whose last undistortion did not complete (an unordered cloud given to
// malio_undistort_device, a failed allocation) holds no cloud to filter; a slot never undistorted is an empty cloud.
static int voxel_slot_input(malio_handle* h, const PreLidar& L, const float*& d_in, uint32_t& n) {
  if (!L.ud_valid && L.n) { h->err = "voxel_grid: the slot's last undistortion did not complete (undistort it again)"; return MALIO_ERR_STATE; }
  n = L.n;
  d_in = L.d_ud;
  return MALIO_OK;
}

int voxel_grid(malio_handle* h, int lidar, const float* in, uint32_t n, float leaf, float* out, uint32_t out_cap, uint32_t* n_out) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  if (lidar < 0 || lidar >= MALIO_MAX_LIDAR || !(leaf > 0.f)) { h->err = "voxel_grid: bad lidar slot or leaf size"; return MALIO_ERR_INVALID_ARG; }
  PreLidar& L = S->lid[lidar];
  cudaStream_t st = S->stream;
  const float* d_in;
  if (in) {
    if (n > S->d_vin.size() / 5) { if (int rc = S->d_vin.allocate(h, st, (size_t)(n + 1024) * 5)) return rc; }
    if (n) CUDA_TRY(cudaMemcpyAsync(S->d_vin, in, (size_t)n * 5 * sizeof(float), cudaMemcpyHostToDevice, st));
    D->ctr.h2d_bytes += (uint64_t)n * 20;
    d_in = S->d_vin;
  } else if (int rc = voxel_slot_input(h, L, d_in, n)) {
    return rc;
  }
  if (int rc = voxel_grid_run(h, S, D, L, d_in, n, leaf, n_out)) return rc;
  if (out && L.n_ds) {
    const uint32_t k = L.n_ds < out_cap ? L.n_ds : out_cap;
    CUDA_TRY(cudaMemcpyAsync(out, L.d_ds, (size_t)k * 5 * sizeof(float), cudaMemcpyDeviceToHost, st));
    D->ctr.d2h_bytes += (uint64_t)k * 20;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return MALIO_OK;
}

// malio_voxel_grid with the explicit input and the output in device memory, ordered on the caller's stream.  The input is read
// where it is (nothing reads it after vg_centroid_kernel); the call returns with that kernel and the copy of the output enqueued.
int voxel_grid_device(malio_handle* h, int lidar, const float* in, uint32_t n, float leaf, float* out, uint32_t out_cap, uint32_t* n_out,
                      cudaStream_t caller) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  if (lidar < 0 || lidar >= MALIO_MAX_LIDAR || !(leaf > 0.f)) { h->err = "voxel_grid: bad lidar slot or leaf size"; return MALIO_ERR_INVALID_ARG; }
  PreLidar& L = S->lid[lidar];
  const float* d_in = in;
  if (!in) { if (int rc = voxel_slot_input(h, L, d_in, n)) return rc; }
  if (n) {
    if (int rc = check_device_ptrs(h, D, {{in, "malio_voxel_grid_device in"}, {out_cap ? out : nullptr, "malio_voxel_grid_device out"}}))
      return rc;
    if (int rc = caller_enter(h, D, caller)) return rc;
  }
  // an early return below (no finite point, MALIO_ERR_CAPACITY) comes after a wait for the last kernel that read `in`
  if (int rc = voxel_grid_run(h, S, D, L, d_in, n, leaf, n_out)) return rc;
  if (L.n_ds == 0) return MALIO_OK;
  const uint32_t k = L.n_ds < out_cap ? L.n_ds : out_cap;
  if (out && k) CUDA_TRY(cudaMemcpyAsync(out, L.d_ds, (size_t)k * 5 * sizeof(float), cudaMemcpyDeviceToDevice, S->stream));
  return caller_leave(h, D, caller);
}

// the slots' down-sampled clouds merged into the handle's scan.  table: host memory, or (table_on_device) the table
// malio_scan_uncertainty* left in d_uout, copied device-to-device
static int merge_scan(malio_handle* h, PreState* S, DeviceState* D, const malio_pose_entry* table, bool table_on_device,
                      const uint32_t* table_off, const malio_rigid* tcomp, uint32_t* n_total) {
  const int Ln = h->cfg.params.n_lidar;
  uint32_t total = 0;
  for (int l = 0; l < Ln; ++l) {
    if (!S->lid[l].ds_valid) { h->err = "upload_scan_device: no down-sampled cloud for a LiDAR (call malio_voxel_grid first)"; return MALIO_ERR_STATE; }
    total += S->lid[l].n_ds;
  }
  if (int rc = malio_dev::upload_scan_from(h, malio_dev::SCAN_ROOM, nullptr, total, table,
                                           table_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, table_off, tcomp, nullptr))
    return rc;
  uint32_t at = 0;
  for (int l = 0; l < Ln; ++l) {
    const uint32_t m = S->lid[l].n_ds;
    if (m) merge_scan_kernel<<<(m + 255) / 256, 256, 0, S->stream>>>(S->lid[l].d_ds, m, (uint16_t)l, D->d_pts + at);
    at += m;
  }
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(S->stream));
  D->ctr.kernel_launches += Ln;
  if (n_total) *n_total = total;
  return MALIO_OK;
}

int upload_scan_device(malio_handle* h, const malio_pose_entry* table, const uint32_t* table_off, const malio_rigid* tcomp,
                       uint32_t* n_total) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  return merge_scan(h, S, D, table, false, table_off, tcomp, n_total);
}

// malio_upload_scan_device with the table, its offsets and the temporal compensations of the last malio_scan_uncertainty*
int upload_scan_resident(malio_handle* h, uint32_t* n_total) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  if (!S->table_resident) {
    h->err = "upload_scan_resident: no pose table on the device (run malio_scan_uncertainty* after the last malio_undistort* of the scan)";
    return MALIO_ERR_STATE;
  }
  return merge_scan(h, S, D, (const malio_pose_entry*)S->d_uout.data(), true, S->res_table_off, S->res_tcomp, n_total);
}

// the registration of `source` for world_register: *n_out = its point count n, and the first k = min(n, cap) points go to
// `out`.  Host array (on_device false): world_kernel writes d_wstage, which world_register copies out when *k > 0.  Device
// array (16-byte aligned: world_kernel stores float4), ordered on `caller`: world_kernel writes it directly when all n points
// fit, and d_wstage otherwise, followed by a D2D copy of the first k points.
static int world_register_to(malio_handle* h, const malio_pass_state* s, int source, const float* slot_tag, float* out, uint32_t cap,
                             uint32_t* n_out, bool on_device, cudaStream_t caller, uint64_t* k_out) {
  *k_out = 0;
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  uint64_t n = 0;
  if (int rc = world_count(h, S, D, source, n)) return rc;
  if (n > 0xFFFFFFFFull) { h->err = "world registration: more than 2^32-1 points"; return MALIO_ERR_CAPACITY; }
  const uint64_t k = n < cap ? n : cap;
  if (on_device && out && k) {
    if (int rc = check_device_ptr(h, D, out, "malio_world_register_device out")) return rc;
    if (reinterpret_cast<uintptr_t>(out) & 15u) {
      h->err = "malio_world_register_device out: not 16-byte aligned (the points are stored as float4)";
      return MALIO_ERR_INVALID_ARG;
    }
  }
  *n_out = (uint32_t)n;
  if (!out || k == 0) return MALIO_OK;
  const bool whole = on_device && k == n;
  if (!whole) { if (int rc = grow_wstage(h, S, n)) return rc; }
  if (on_device) { if (int rc = caller_enter(h, D, caller)) return rc; }
  if (int rc = world_launch(h, S, D, s, source, slot_tag, whole ? reinterpret_cast<float4*>(out) : S->d_wstage)) return rc;
  if (on_device) {
    if (!whole) CUDA_TRY(cudaMemcpyAsync(out, S->d_wstage, (size_t)k * sizeof(float4), cudaMemcpyDeviceToDevice, S->stream));
    if (int rc = caller_leave(h, D, caller)) return rc;   // (S->stream is D->stream)
  }
  *k_out = k;
  return MALIO_OK;
}

int world_register(malio_handle* h, const malio_pass_state* s, int source, const float* slot_tag, float* out, uint32_t cap,
                   uint32_t* n_out) {
  uint64_t k = 0;
  if (int rc = world_register_to(h, s, source, slot_tag, out, cap, n_out, false, nullptr, &k)) return rc;
  if (k == 0) return MALIO_OK;
  PreState* S = h->pre.get();
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaMemcpyAsync(out, S->d_wstage, (size_t)k * sizeof(float4), cudaMemcpyDeviceToHost, S->stream));
  CUDA_TRY(cudaStreamSynchronize(S->stream));
  D->ctr.d2h_bytes += k * sizeof(float4);
  return MALIO_OK;
}

int world_accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, uint64_t* n_total) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  uint64_t n = 0;
  if (int rc = world_count(h, S, D, MALIO_WORLD_DENSE, n)) return rc;
  const uint64_t need = S->n_acc + n;
  if (need > S->d_acc.size()) {
    // geometric growth: a larger buffer, the old content copied over on the device, then the old one freed.  A failed
    // allocation leaves the accumulated cloud as it was.
    uint64_t c = S->d_acc.size() * 2;
    if (c < need) c = need;
    if (c < WORLD_ACC_MIN) c = WORLD_ACC_MIN;
    if (const cudaError_t e = malio_buf::grow_keep(S->stream, {{S->d_acc, c, S->n_acc}})) {
      h->err = std::string("world accumulate: cannot grow the cloud to ") + std::to_string(c) + " points: " + cudaGetErrorString(e);
      return MALIO_ERR_CUDA;
    }
  }
  if (n) {
    if (int rc = world_launch(h, S, D, s, MALIO_WORLD_DENSE, slot_tag, S->d_acc + S->n_acc)) return rc;
    CUDA_TRY(cudaStreamSynchronize(S->stream));
  }
  S->n_acc = need;
  if (n_total) *n_total = S->n_acc;
  return MALIO_OK;
}

// the dense cloud for the voxel map (malio_voxmap.cu): the undistorted clouds of slots 0..L-1 (n x 5 rows on the device) and
// their sizes, with world_count's state error
int world_dense_source(malio_handle* h, const float* ud[MALIO_MAX_LIDAR], uint32_t n[MALIO_MAX_LIDAR]) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  uint64_t total = 0;
  if (int rc = world_count(h, S, D, MALIO_WORLD_DENSE, total)) return rc;
  for (int l = 0; l < h->cfg.params.n_lidar; ++l) { ud[l] = S->lid[l].d_ud; n[l] = S->lid[l].n; }
  return MALIO_OK;
}

int world_save_pcd(malio_handle* h, const char* path, int clear) {
  PreState* S;
  DeviceState* D;
  if (int rc = acquire(h, h->pre, S, D)) return rc;
  if (S->n_acc == 0) { h->err = "world save: the accumulated cloud is empty (nothing is written)"; return MALIO_ERR_STATE; }
  if (!S->h_bounce) { if (int rc = S->h_bounce.allocate(h, malio_pcd::CHUNK)) return rc; }
  const int rc = malio_pcd::write_binary(path, S->n_acc, [&](uint64_t first, uint64_t cnt, const float** xyzi) {
    if (cudaMemcpyAsync(S->h_bounce, S->d_acc + first, cnt * sizeof(float4), cudaMemcpyDeviceToHost, S->stream) != cudaSuccess ||
        cudaStreamSynchronize(S->stream) != cudaSuccess)
      return (int)MALIO_ERR_CUDA;
    D->ctr.d2h_bytes += cnt * sizeof(float4);
    *xyzi = (const float*)S->h_bounce.data();
    return (int)MALIO_OK;
  }, h->err);
  if (rc == MALIO_OK && clear) S->n_acc = 0;   // pcl_wait_save->clear() (:485); the buffer is kept
  return rc;
}

// malio_scan_uncertainty, and with table == NULL malio_scan_uncertainty_resident: the table is built in d_uout either way and
// stays there for malio_upload_scan_resident; the resident call fetches the L - 1 temporal compensations only (the passes take
// them as kernel constants, and the host's sin / cos differ from the device's in the last place, so they are not recomputed),
// and table_off, temporal_comp may be NULL
int scan_uncertainty(malio_handle* h, const malio_scan_unc_args* a, malio_pose_entry* table, uint32_t table_cap, uint32_t* table_off,
                     malio_pose* temporal_comp, malio_pose* lidar_unc, uint32_t* lidar_unc_counts) {
  PreState* S = h->pre.get();
  uint32_t off_local[MALIO_MAX_LIDAR + 1];
  if (!table_off) table_off = off_local;
  const int Ln = h->cfg.params.n_lidar;
  UncConst c{};
  c.L = Ln;
  uint32_t n_unc = 0, n_tab = 0, n_thr = 0;
  for (int l = 0; l < Ln; ++l) {
    if (!S || !S->lid[l].ud_valid) { h->err = "scan_uncertainty: malio_undistort has not run on every LiDAR slot 0..L-1"; return MALIO_ERR_STATE; }
    const PreLidar& P = S->lid[l];
    if (P.n_cov != a->n_cov) { h->err = "scan_uncertainty: n_cov differs from the one malio_undistort of a slot saw"; return MALIO_ERR_INVALID_ARG; }
    if (l != 0 && P.cov_pointer < 0) { h->err = "scan_uncertainty: lt_lidar_frame of LiDAR >= 1 needs imu_cov[cov_pointer] (:471), cov_pointer is -1"; return MALIO_ERR_INVALID_ARG; }
    c.pop[l] = P.d_pop; c.pose[l] = P.d_pose; c.ok[l] = P.d_ok;
    c.cov_pointer[l] = P.cov_pointer;
    c.n_pops[l] = (int32_t)P.n_pops;
    c.first[l] = n_thr;
    c.unc_off[l] = n_unc;
    c.tab_off[l] = n_tab;
    table_off[l] = n_tab;
    n_thr += P.n_pops > 0 ? P.n_pops : 1;
    n_unc += P.n_pops;
    n_tab += P.n_pops > 1 ? P.n_pops - 1 : 0;                               // (int)size() - 1 entries, laserMapping.cpp:1035, :1040
  }
  c.first[Ln] = n_thr;
  table_off[Ln] = n_tab;
  if (table && n_tab > table_cap) {
    h->err = "scan_uncertainty: the table needs " + std::to_string(n_tab) + " entries (table_off[L]), table_cap is " + std::to_string(table_cap);
    return MALIO_ERR_CAPACITY;
  }
  for (int l = 0; l < Ln; ++l) {
    const PreLidar& P = S->lid[l];
    c.ext[l] = a->extrinsic[l];
    const double* cov = l == 0 ? a->uncertainty : a->imu_cov + 36 * (size_t)P.cov_pointer;   // :450 / :471
    malio_compound::pose_initial(&c.ltl[l], P.lt_imu_frame.t, P.lt_imu_frame.q, cov);
  }
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  cudaStream_t st = S->stream;
  const size_t tab_bytes = (size_t)n_tab * sizeof(malio_pose_entry);
  const size_t out_bytes = tab_bytes + (size_t)(Ln - 1 + (lidar_unc ? n_unc : 0)) * sizeof(malio_pose);
  if (!S->d_ucov) {   // sized for the largest lists: L x MALIO_MAX_COV pops, L - 1 compensations
    if (int rc = malio_buf::allocate_group(h, st, {{S->d_ucov, (size_t)MALIO_MAX_COV * 36},
                                                   {S->d_uout, (size_t)MALIO_MAX_LIDAR * MALIO_MAX_COV * (sizeof(malio_pose_entry) + sizeof(malio_pose)) +
                                                                   MALIO_MAX_LIDAR * sizeof(malio_pose)}}))
      return rc;
  }
  S->table_resident = false;
  if (a->n_cov) CUDA_TRY(cudaMemcpyAsync(S->d_ucov, a->imu_cov, (size_t)a->n_cov * 36 * sizeof(double), cudaMemcpyHostToDevice, st));
  malio_pose_entry* d_tab = (malio_pose_entry*)S->d_uout.data();
  malio_pose* d_tc = (malio_pose*)(S->d_uout.data() + tab_bytes);
  malio_pose* d_unc = d_tc + (Ln - 1);
  scan_unc_kernel<<<(n_thr + UNC_THREADS - 1) / UNC_THREADS, UNC_THREADS, 0, st>>>(c, S->d_ucov, d_tab, d_tc, d_unc);
  CUDA_TRY(cudaGetLastError());
  const size_t tc_bytes = (size_t)(Ln - 1) * sizeof(malio_pose);
  const size_t skip = table ? 0 : tab_bytes, fetch = table ? out_bytes : tc_bytes;
  std::vector<char> out(fetch);
  if (fetch) CUDA_TRY(cudaMemcpyAsync(out.data(), S->d_uout + skip, fetch, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  D->ctr.kernel_launches += 1;
  D->ctr.h2d_bytes += (uint64_t)a->n_cov * 36 * 8;
  D->ctr.d2h_bytes += fetch;
  const malio_pose* tc = (const malio_pose*)(out.data() + tab_bytes - skip);
  if (table) std::memcpy(table, out.data(), tab_bytes);
  if (Ln > 1 && temporal_comp) std::memcpy(temporal_comp, tc, tc_bytes);
  if (lidar_unc) std::memcpy(lidar_unc, out.data() + tab_bytes + tc_bytes, (size_t)n_unc * sizeof(malio_pose));
  if (lidar_unc_counts) for (int l = 0; l < Ln; ++l) lidar_unc_counts[l] = (uint32_t)c.n_pops[l];
  for (int l = 0; l <= Ln; ++l) S->res_table_off[l] = table_off[l];
  for (int l = 0; l + 1 < Ln; ++l) {
    std::memcpy(S->res_tcomp[l].q, tc[l].q, sizeof(tc[l].q));
    std::memcpy(S->res_tcomp[l].t, tc[l].t, sizeof(tc[l].t));
  }
  S->table_resident = true;
  return MALIO_OK;
}

}  // namespace malio_pre

// host-side spline pose (same code as the device's, compiled for the host)
extern "C" int malio_bspline_get_pose(const double* ctrl_t, const double* ctrl_T, uint32_t n_ctrl, double timestamp, double q[4], double p[3]) {
  if (!ctrl_t || !ctrl_T || !q || !p || n_ctrl < 4 || n_ctrl > MALIO_MAX_CTRL) { if (p) { p[0] = p[1] = p[2] = 0; } return 0; }
  std::vector<double> seglog((size_t)n_ctrl * 6, 0.0);
  int i0, i1, i2, i3;
  if (!find_bounding(ctrl_t, (int)n_ctrl, timestamp, i0, i1, i2, i3)) { p[0] = p[1] = p[2] = 0; return 0; }
  for (int k = i0; k <= i2; ++k) {
    double ai[16], rel[16];
    inv_se3(ctrl_T + 16 * (size_t)k, ai);
    mul4(ai, ctrl_T + 16 * (size_t)(k + 1), rel);
    log_se3(rel, seglog.data() + 6 * (size_t)k);
  }
  return spline_pose(ctrl_t, ctrl_T, seglog.data(), (int)n_ctrl, timestamp, q, p) ? 1 : 0;
}

// the scan's pose-uncertainty table (IMU_Processing.hpp:474-523, laserMapping.cpp:1028-1048)
extern "C" int malio_scan_uncertainty(malio_handle* h, const malio_scan_unc_args* a, malio_pose_entry* table, uint32_t table_cap,
                                      uint32_t* table_off, malio_pose* temporal_comp, malio_pose* lidar_unc, uint32_t* lidar_unc_counts) {
  if (!h || !a || !table || !table_off || !a->extrinsic || !a->uncertainty || (a->n_cov && !a->imu_cov)) return MALIO_ERR_INVALID_ARG;
  if (h->cfg.params.n_lidar > 1 && !temporal_comp) { h->err = "scan_uncertainty: temporal_comp required for L > 1"; return MALIO_ERR_INVALID_ARG; }
  MALIO_SETTLE(h);
  return malio_pre::scan_uncertainty(h, a, table, table_cap, table_off, temporal_comp, lidar_unc, lidar_unc_counts);
}

extern "C" int malio_scan_uncertainty_resident(malio_handle* h, const malio_scan_unc_args* a, uint32_t* table_off, malio_pose* temporal_comp) {
  if (!h || !a || !a->extrinsic || !a->uncertainty || (a->n_cov && !a->imu_cov)) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_pre::scan_uncertainty(h, a, nullptr, 0, table_off, temporal_comp, nullptr, nullptr);
}

// the front half of a scan on device memory (malio_b200.h): the wrappers check what malio_undistort / malio_voxel_grid /
// malio_upload_scan_device check on the host; the device pointers are checked inside, once the point count is known
extern "C" int malio_undistort_device(malio_handle* h, int lidar, const malio_raw_pt* d_pts, uint32_t n, const malio_undistort_args* a,
                                      float* d_cloud, int32_t* d_idx, uint8_t* d_ok, int32_t* d_pop_point, double* d_pose, uint32_t* n_pops,
                                      void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!a || !a->ctrl_t || !a->ctrl_T || (a->n_cov && !a->imu_cov_t)) return MALIO_ERR_INVALID_ARG;
  return malio_pre::undistort_device(h, lidar, d_pts, n, a, d_cloud, d_idx, d_ok, d_pop_point, d_pose, n_pops, (cudaStream_t)stream);
}
extern "C" int malio_voxel_grid_device(malio_handle* h, int lidar, const float* d_in, uint32_t n, float leaf, float* d_out, uint32_t out_cap,
                                       uint32_t* n_out, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_pre::voxel_grid_device(h, lidar, d_in, n, leaf, d_out, out_cap, n_out, (cudaStream_t)stream);
}
extern "C" int malio_upload_scan_resident(malio_handle* h, uint32_t* n_total) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_pre::upload_scan_resident(h, n_total);
}

// publish_frame_world / pcd_save (laserMapping.cpp:448-489)
extern "C" int malio_world_register(malio_handle* h, const malio_pass_state* s, int source, const float* slot_tag, float* out,
                                    uint32_t cap, uint32_t* n_out) {
  if (!h || !s || !n_out || (cap && !out)) return MALIO_ERR_INVALID_ARG;
  if (source != MALIO_WORLD_DOWNSAMPLED && source != MALIO_WORLD_DENSE) { h->err = "world register: unknown source"; return MALIO_ERR_INVALID_ARG; }
  if (source == MALIO_WORLD_DENSE && !slot_tag) { h->err = "world register: the dense cloud needs slot_tag"; return MALIO_ERR_INVALID_ARG; }
  MALIO_SETTLE(h);
  return malio_pre::world_register(h, s, source, slot_tag, out, cap, n_out);
}
extern "C" int malio_world_register_device(malio_handle* h, const malio_pass_state* s, int source, const float* slot_tag, float* d_out,
                                           uint32_t cap, uint32_t* n_out, void* stream) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  if (!s || !n_out || (cap && !d_out)) return MALIO_ERR_INVALID_ARG;
  if (source != MALIO_WORLD_DOWNSAMPLED && source != MALIO_WORLD_DENSE) { h->err = "world register: unknown source"; return MALIO_ERR_INVALID_ARG; }
  if (source == MALIO_WORLD_DENSE && !slot_tag) { h->err = "world register: the dense cloud needs slot_tag"; return MALIO_ERR_INVALID_ARG; }
  uint64_t k = 0;
  return malio_pre::world_register_to(h, s, source, slot_tag, d_out, cap, n_out, true, (cudaStream_t)stream, &k);
}
extern "C" int malio_world_accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, uint64_t* n_total) {
  if (!h || !s) return MALIO_ERR_INVALID_ARG;
  if (!slot_tag) { h->err = "world accumulate: the dense cloud needs slot_tag"; return MALIO_ERR_INVALID_ARG; }
  MALIO_SETTLE(h);
  return malio_pre::world_accumulate(h, s, slot_tag, n_total);
}
extern "C" int malio_world_save_pcd(malio_handle* h, const char* path, int clear) {
  if (!h || !path) return MALIO_ERR_INVALID_ARG;
  MALIO_SETTLE(h);
  return malio_pre::world_save_pcd(h, path, clear);
}
