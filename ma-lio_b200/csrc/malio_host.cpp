// malio_host.cpp — host C++ side of libmalio_b200.so: the C-ABI wrappers, the iterated error-state Kalman
// update on the state manifold, and the static snapshot builder.  No CUDA here; the device work is behind
// malio_dev:: (malio_knn.cu, malio_pass.cu, malio_b200.cu).  There is NO CPU fallback for the measurement: without a usable GPU
// malio_create fails with MALIO_ERR_CUDA.
//
// Reference interface mirrored (paths relative to /root/reference/MA_LIO):
//   esekf::update_iterated_dyn_share_modified   include/IKFoM_toolkit/esekfom/esekfom.hpp:495-721
//   state_ikfom manifold                        src/use-ikfom.hpp:14-27
//   MTK SO3 / S2 / vect boxplus, boxminus       include/IKFoM_toolkit/mtk/types/{SOn,S2,vect}.hpp
//   MTK::A_matrix, exp, log                     include/IKFoM_toolkit/mtk/src/mtkmath.hpp:235-289
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>
#include <numeric>
#include <vector>

#include "malio_compound.h"
#include "malio_internal.h"
#include "malio_manifold.h"

using namespace malio_manifold;

namespace {

thread_local std::string g_err = "";

// ---------------------------------------------------------------- tiny dense matrix (row-major, run-time n <= 35)
struct Mat {
  int r = 0, c = 0;
  std::vector<double> a;
  Mat() {}
  Mat(int r_, int c_) : r(r_), c(c_), a((size_t)r_ * c_, 0.0) {}
  double& operator()(int i, int j) { return a[(size_t)i * c + j]; }
  double operator()(int i, int j) const { return a[(size_t)i * c + j]; }
};

// LU with partial pivoting, in place; returns false on an exactly singular pivot
bool lu_factor(Mat& A, std::vector<int>& piv) {
  const int n = A.r;
  piv.resize(n);
  std::iota(piv.begin(), piv.end(), 0);
  for (int k = 0; k < n; ++k) {
    int p = k;
    double best = std::fabs(A(k, k));
    for (int i = k + 1; i < n; ++i)
      if (std::fabs(A(i, k)) > best) { best = std::fabs(A(i, k)); p = i; }
    if (best == 0.0) return false;
    if (p != k) {
      for (int j = 0; j < n; ++j) std::swap(A(k, j), A(p, j));
      std::swap(piv[k], piv[p]);
    }
    const double inv = 1.0 / A(k, k);
    for (int i = k + 1; i < n; ++i) {
      const double f = A(i, k) * inv;
      A(i, k) = f;
      if (f != 0.0)
        for (int j = k + 1; j < n; ++j) A(i, j) -= f * A(k, j);
    }
  }
  return true;
}
// X = A^{-1} B for B given column-block wise (B: n x m)
void lu_solve(const Mat& LU, const std::vector<int>& piv, const Mat& B, Mat& X) {
  const int n = LU.r, m = B.c;
  X = Mat(n, m);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < m; ++j) X(i, j) = B(piv[i], j);
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < i; ++k) {
      const double f = LU(i, k);
      if (f != 0.0) for (int j = 0; j < m; ++j) X(i, j) -= f * X(k, j);
    }
  for (int i = n - 1; i >= 0; --i) {
    for (int k = i + 1; k < n; ++k) {
      const double f = LU(i, k);
      if (f != 0.0) for (int j = 0; j < m; ++j) X(i, j) -= f * X(k, j);
    }
    const double inv = 1.0 / LU(i, i);
    for (int j = 0; j < m; ++j) X(i, j) *= inv;
  }
}
bool invert(const Mat& A, Mat& Ainv) {
  Mat LU = A;
  std::vector<int> piv;
  if (!lu_factor(LU, piv)) return false;
  Mat I(A.r, A.r);
  for (int i = 0; i < A.r; ++i) I(i, i) = 1.0;
  lu_solve(LU, piv, I, Ainv);
  return true;
}

// rows [idx, idx+bs) <- J * rows ; cols likewise with J^T  (block sizes 3 and 2)
template <int BS>
void left_block(Mat& M, int idx, const double J[BS][BS], int ncols) {
  for (int j = 0; j < ncols; ++j) {
    double v[BS], o[BS];
    for (int a = 0; a < BS; ++a) v[a] = M(idx + a, j);
    for (int a = 0; a < BS; ++a) { o[a] = 0; for (int b = 0; b < BS; ++b) o[a] += J[a][b] * v[b]; }
    for (int a = 0; a < BS; ++a) M(idx + a, j) = o[a];
  }
}
template <int BS>
void right_block_T(Mat& M, int idx, const double J[BS][BS]) {
  for (int i = 0; i < M.r; ++i) {
    double v[BS], o[BS];
    for (int a = 0; a < BS; ++a) v[a] = M(i, idx + a);
    for (int a = 0; a < BS; ++a) { o[a] = 0; for (int b = 0; b < BS; ++b) o[a] += v[b] * J[a][b]; }
    for (int a = 0; a < BS; ++a) M(i, idx + a) = o[a];
  }
}

}  // namespace

namespace malio_host {
// singular values of the N x 3 matrix whose Gram matrix is S (descending) = sqrt(eig(S)); closed-form
// trigonometric solution of the symmetric 3x3 characteristic polynomial, refined by one Jacobi sweep set
void sym3_singular_values(const double S[6], double sv[3]) { malio_manifold::sym3_singular_values(S, sv); }
}  // namespace malio_host

// =================================================================== C-ABI
extern "C" {

const char* malio_version(void) { return "malio_b200 0.1 (sm_90a)"; }

void malio_default_params(malio_params* p, int n_lidar) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  p->n_lidar = n_lidar;
  p->extrinsic_est_en = 1;          // config/City.yaml:23
  p->plane_th = 0.4f;               // launch/mapping_city.launch:13
  p->knn_max_sqdist = 5.0f;         // laserMapping.cpp:587
  p->cov_threshold = 0.5;           // City.yaml:50
  p->point_cov_max = 0.00125; p->point_cov_min = 0.00075;   // City.yaml:42-43
  p->plane_cov_max = 1.0; p->plane_cov_min = 0.8;           // City.yaml:44-45
  p->localize_cov_max = 2.0; p->localize_cov_min = 0.3;     // City.yaml:46-47
  p->localize_thresh_max = 0.7; p->localize_thresh_min = 0.2;   // City.yaml:48-49
  p->range_min = 0.0; p->range_max = 1.0;                   // mapping_city.launch:14-15
}

const char* malio_last_error(const malio_handle* h) { return h ? h->err.c_str() : g_err.c_str(); }

int malio_create(malio_handle** out, const malio_config* cfg) {
  if (!out || !cfg) { g_err = "null argument"; return MALIO_ERR_INVALID_ARG; }
  *out = nullptr;
  if (cfg->params.n_lidar < 1 || cfg->params.n_lidar > MALIO_MAX_LIDAR) { g_err = "n_lidar must be 1..3"; return MALIO_ERR_INVALID_ARG; }
  malio_handle* h = new malio_handle;
  h->cfg = *cfg;
  const int rc = malio_dev::create(h);
  if (rc != MALIO_OK) {
    g_err = h->err;
    malio_dev::destroy(h);
    delete h;
    return rc;
  }
  *out = h;
  return MALIO_OK;
}
void malio_destroy(malio_handle* h) {
  if (!h) return;
  malio_dev::destroy(h);
  delete h;
}
int malio_get_nccl_unique_id(uint8_t id[MALIO_NCCL_UNIQUE_ID_BYTES]) { return id ? malio_dev::get_unique_id(id) : MALIO_ERR_INVALID_ARG; }
int malio_comm_init(malio_handle* h, const uint8_t id[MALIO_NCCL_UNIQUE_ID_BYTES], int rank, int world) {
  if (!h || !id || world < 1 || rank < 0 || rank >= world) return MALIO_ERR_INVALID_ARG;
  return malio_dev::comm_init(h, id, rank, world);
}
int malio_upload_map(malio_handle* h, const malio_map_node* nodes, const float* node_cov, uint32_t n_nodes, uint32_t max_depth) {
  if (!h || (n_nodes && (!nodes || !node_cov))) return MALIO_ERR_INVALID_ARG;
  return malio_dev::upload_map(h, nodes, node_cov, n_nodes, max_depth);
}
int malio_upload_map_compact(malio_handle* h, const malio_map_point* pts, const float* node_cov, uint32_t n_nodes, uint32_t max_depth,
                             const float* root_box) {
  if (!h || (n_nodes && (!pts || !node_cov))) return MALIO_ERR_INVALID_ARG;
  return malio_dev::upload_map_compact(h, pts, node_cov, n_nodes, max_depth, root_box);
}
int malio_download_map_nodes(malio_handle* h, malio_map_node* out, uint32_t capacity) {
  if (!h || !out) return MALIO_ERR_INVALID_ARG;
  return malio_dev::download_map_nodes(h, out, capacity);
}
int malio_upload_scan(malio_handle* h, const malio_scan_pt* pts, uint32_t n_pts, const malio_pose_entry* table,
                      const uint32_t* table_off, const malio_rigid* temporal_comp) {
  if (!h || (n_pts && !pts) || !table || !table_off) return MALIO_ERR_INVALID_ARG;
  if (h->cfg.params.n_lidar > 1 && !temporal_comp) { h->err = "temporal_comp required for L > 1"; return MALIO_ERR_INVALID_ARG; }
  return malio_dev::upload_scan(h, pts, n_pts, table, table_off, temporal_comp);
}
int malio_rearm_scan(malio_handle* h) { return h ? malio_dev::rearm_scan(h) : MALIO_ERR_INVALID_ARG; }
int malio_set_timing(malio_handle* h, int enable) { return h ? malio_dev::set_timing(h, enable) : MALIO_ERR_INVALID_ARG; }
int malio_get_counters(malio_handle* h, malio_counters* out) { return (h && out) ? malio_dev::get_counters(h, out) : MALIO_ERR_INVALID_ARG; }
int malio_measure(malio_handle* h, const malio_pass_state* s, int redo_knn, double* HtRinvH, double* HtRinvh, malio_pass_stats* stats) {
  if (!h || !s || !HtRinvH || !HtRinvh) return MALIO_ERR_INVALID_ARG;
  return malio_dev::measure(h, s, redo_knn, HtRinvH, HtRinvh, stats);
}
int malio_download_rows(malio_handle* h, double* h_x, double* hvec, uint32_t cap, uint32_t* n_rows) {
  if (!h || !h_x || !hvec || !n_rows) return MALIO_ERR_INVALID_ARG;
  return malio_dev::download_rows(h, h_x, hvec, cap, n_rows);
}
int malio_download_aux(malio_handle* h, float* normal_y, uint32_t* nn_idx, float* nn_sqdist, uint8_t* selected, float* world) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  return malio_dev::download_aux(h, normal_y, nn_idx, nn_sqdist, selected, world);
}
int malio_map_incremental(malio_handle* h, const malio_pass_state* s, double filter_size_map, int ekf_inited, uint8_t* cls, float* world) {
  if (!h || !s || !cls || !(filter_size_map > 0.0)) return MALIO_ERR_INVALID_ARG;
  return malio_dev::map_incremental(h, s, filter_size_map, ekf_inited, cls, world);
}
// ---------------------------------------------------------------- N1 wrappers (malio_mapops.cu)
int malio_map_build(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n) {
  if (!h || (n && (!xyz || !normal_y))) return MALIO_ERR_INVALID_ARG;
  return malio_map::build(h, xyz, normal_y, ids, n);
}
int malio_map_add_points(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n) {
  if (!h || (n && (!xyz || !normal_y))) return MALIO_ERR_INVALID_ARG;
  return malio_map::add_points(h, xyz, normal_y, ids, n);
}
int malio_map_delete_boxes(malio_handle* h, const float* boxes, uint32_t nb, uint32_t* n_deleted) {
  if (!h || (nb && !boxes)) return MALIO_ERR_INVALID_ARG;
  return malio_map::delete_boxes(h, boxes, nb, n_deleted);
}
int malio_map_sync_voxels(malio_handle* h, const float* boxes, uint32_t nb, const float* xyz, const float* normal_y, const int32_t* ids,
                          uint32_t n_points, uint32_t* n_deleted) {
  if (!h || (nb && !boxes) || (n_points && (!xyz || !normal_y))) return MALIO_ERR_INVALID_ARG;
  return malio_map::sync_voxels(h, boxes, nb, xyz, normal_y, ids, n_points, n_deleted);
}
int malio_map_commit(malio_handle* h) { return h ? malio_map::commit(h) : MALIO_ERR_INVALID_ARG; }
int malio_map_info(malio_handle* h, uint32_t* n_live, uint32_t* n_slots) { return h ? malio_map::info(h, n_live, n_slots) : MALIO_ERR_INVALID_ARG; }
int malio_map_download(malio_handle* h, float* xyz, float* normal_y, int32_t* ids, uint32_t* slots, uint32_t cap, uint32_t* n) {
  return h ? malio_map::download(h, xyz, normal_y, ids, slots, cap, n) : MALIO_ERR_INVALID_ARG;
}

// ---------------------------------------------------------------- N2 / N3 wrappers (malio_preproc.cu)
int malio_undistort(malio_handle* h, int lidar, const malio_raw_pt* pts, uint32_t n, const malio_undistort_args* a, float* xyz,
                    int32_t* idx, uint8_t* ok, int32_t* pop_point, uint32_t* n_pops, double* pose) {
  if (!h || !a || (n && !pts) || !a->ctrl_t || !a->ctrl_T || (a->n_cov && !a->imu_cov_t)) return MALIO_ERR_INVALID_ARG;
  // the walk of IMU_Processing.hpp:476-486 assumes the cloud sorted by time (sort at :232): checked, not assumed
  for (uint32_t i = 1; i < n; ++i)
    if (pts[i].curvature < pts[i - 1].curvature) { h->err = "malio_undistort: points must be sorted by curvature (IMU_Processing.hpp:232)"; return MALIO_ERR_INVALID_ARG; }
  return malio_pre::undistort(h, lidar, pts, n, a, xyz, idx, ok, pop_point, n_pops, pose);
}
int malio_voxel_grid(malio_handle* h, int lidar, const float* in, uint32_t n, float leaf, float* out, uint32_t out_cap, uint32_t* n_out) {
  if (!h) return MALIO_ERR_INVALID_ARG;
  return malio_pre::voxel_grid(h, lidar, in, n, leaf, out, out_cap, n_out);
}
int malio_upload_scan_device(malio_handle* h, const malio_pose_entry* table, const uint32_t* table_off, const malio_rigid* temporal_comp,
                             uint32_t* n_total) {
  if (!h || !table || !table_off) return MALIO_ERR_INVALID_ARG;
  if (h->cfg.params.n_lidar > 1 && !temporal_comp) { h->err = "temporal_comp required for L > 1"; return MALIO_ERR_INVALID_ARG; }
  return malio_pre::upload_scan_device(h, table, table_off, temporal_comp, n_total);
}

// ---------------------------------------------------------------- pose-uncertainty table (malio_compound.h)
void malio_pose_initial(malio_pose* pose, const double t[3], const double q[4], const double cov[36]) {
  if (!pose || !t || !q || !cov) return;   // void like the reference's helper: a NULL argument leaves everything untouched
  malio_compound::pose_initial(pose, t, q, cov);
}
void malio_compound_pose_with_cov(const malio_pose* pose_1, const double* cov_1, const malio_pose* pose_2, const double* cov_2,
                                  malio_pose* pose_cp, double* cov_cp) {
  if (!pose_1 || !cov_1 || !pose_2 || !cov_2 || !pose_cp || !cov_cp) return;
  malio_compound::compound_pose_with_cov(pose_1, cov_1, pose_2, cov_2, pose_cp, cov_cp);
}
void malio_compound_inv_pose_with_cov(const malio_pose* pose_1, const double* cov_1, const malio_pose* pose_2, const double* cov_2,
                                      malio_pose* pose_cp, double* cov_cp) {
  if (!pose_1 || !cov_1 || !pose_2 || !cov_2 || !pose_cp || !cov_cp) return;
  malio_compound::compound_inv_pose_with_cov(pose_1, cov_1, pose_2, cov_2, pose_cp, cov_cp);
}
int malio_build_pose_unc(int n_lidar, const malio_pose* extrinsic, const malio_pose* temporal_comp,
                         const malio_pose* const* lidar_uncertainty, const uint32_t* counts, malio_pose_entry* table,
                         uint32_t* table_off) {
  if (n_lidar < 1 || n_lidar > MALIO_MAX_LIDAR || !extrinsic || !lidar_uncertainty || !counts || !table || !table_off ||
      (n_lidar > 1 && !temporal_comp))
    return -MALIO_ERR_INVALID_ARG;
  uint32_t n = 0;
  for (int num = 0; num < n_lidar; ++num) {
    table_off[num] = n;
    const int keep = (int)counts[num] - 1;                                 // laserMapping.cpp:1035, :1040
    for (int i = 0; i < keep; ++i) malio_compound::pose_unc_entry(num, extrinsic, num ? &temporal_comp[num - 1] : nullptr, &lidar_uncertainty[num][i],
                                                                  &table[n++]);
  }
  table_off[n_lidar] = n;
  return (int)n;
}

int malio_knn(malio_handle* h, const float* q, uint32_t nq, uint32_t* nn_idx, float* nn_sqdist, float* ms_device) {
  if (!h || (nq && !q)) return MALIO_ERR_INVALID_ARG;
  return malio_dev::knn(h, q, nq, nn_idx, nn_sqdist, ms_device);
}

// ---------------------------------------------------------------- IESKF (esekfom.hpp:495-721)
int malio_ieskf_update(malio_handle* h, malio_state* x, double* Pio, int max_iter, double R, malio_update_report* rep) {
  if (!h || !x || !Pio || max_iter < 0) return MALIO_ERR_INVALID_ARG;
  const StateLayout ly(h->cfg.params.n_lidar);
  const int n = ly.n, c = ly.c;
  malio_update_report rp{};
  const malio_state x_prop = *x;
  Mat P_prop(n, n);
  std::memcpy(P_prop.a.data(), Pio, sizeof(double) * n * n);
  Mat P = P_prop, Kx(n, c), G(c, c);
  std::vector<double> g(c), dx(n), dxn(n), Kh(n), step(n), KxDx(n);
  double LU[MALIO_MAX_COLS][MALIO_MAX_COLS];     // factors of Mt = (I + G P_cc)^T of the last regular pass, and its row interchanges
  int piv[MALIO_MAX_COLS];
  double Ykeep[MALIO_MAX_COLS][MALIO_MAX_DOF];   // Q[:,0:c]^T, solved for only by the pass that updates the covariance
  bool kx_lazy = false;
  bool redo = true;   // dyn_share.converge
  int t = 0, rc_last = MALIO_OK;
  double host_ms = 0.0;
  for (int it = -1; it < max_iter; ++it) {
    malio_pass_state ps;
    std::memcpy(ps.rot, x->rot, sizeof(ps.rot));
    std::memcpy(ps.pos, x->pos, sizeof(ps.pos));
    std::memcpy(ps.ext, x->ext, sizeof(ps.ext));
    malio_pass_stats st{};
    const int rc = malio_dev::measure(h, &ps, redo ? 1 : 0, G.a.data(), g.data(), &st);   // h_dyn_share, :512
    rp.passes++;
    if (redo) rp.searches++;
    rp.ms_device_total += st.ms_total;
    rc_last = rc;
    if (rc == MALIO_ERR_NO_EFFECTIVE_POINTS) continue;   // :514-517
    if (rc != MALIO_OK) { if (rep) *rep = rp; return rc; }
    const auto t0 = std::chrono::steady_clock::now();
    rp.n_eff_last = st.n_eff;
    boxminus(ly, *x, x_prop, dx.data());   // :526
    dxn = dx;
    P = P_prop;   // :530
    for (int s = 0; s <= ly.L; ++s) {      // SO3 blocks, :534-549
      const int idx = ly.so3[s];
      const M3 Jt = transpose3(A_matrix(&dx[idx]));
      double o[3];
      for (int a = 0; a < 3; ++a) o[a] = Jt.m[a][0] * dxn[idx] + Jt.m[a][1] * dxn[idx + 1] + Jt.m[a][2] * dxn[idx + 2];
      dxn[idx] = o[0]; dxn[idx + 1] = o[1]; dxn[idx + 2] = o[2];
      left_block<3>(P, idx, Jt.m, n);
      right_block_T<3>(P, idx, Jt.m);
    }
    {                                       // S2 block, :553-572
      double J2[2][2];
      S2_projection(x->grav, x_prop.grav, &dx[ly.grav], J2);
      const double d0 = dxn[ly.grav], d1 = dxn[ly.grav + 1];
      dxn[ly.grav] = J2[0][0] * d0 + J2[0][1] * d1;
      dxn[ly.grav + 1] = J2[1][0] * d0 + J2[1][1] * d1;
      left_block<2>(P, ly.grav, J2, n);
      right_block_T<2>(P, ly.grav, J2);
    }
    if (n > (int)st.n_eff) {   // degenerate branch :574-582 — needs the rows, scalar R
      const int m = (int)st.n_eff;
      std::vector<double> rows((size_t)MALIO_MAX_DOF * c), hv(MALIO_MAX_DOF);
      uint32_t nr = 0;
      const int rc2 = malio_dev::download_rows(h, rows.data(), hv.data(), (uint32_t)m, &nr);
      if (rc2 != MALIO_OK) { if (rep) *rep = rp; return rc2; }
      if ((int)nr != m) {   // a partial H would make the ranks step to different states: fail instead
        h->err = "degenerate branch: rows returned != N_eff";
        if (rep) *rep = rp;
        return MALIO_ERR_STATE;
      }
      Mat H(m, n);
      for (int r = 0; r < m; ++r) {
        for (int k = 0; k < c; ++k) H(r, k) = rows[(size_t)r * c + k] * st.loc_weight;
        hv[r] *= st.loc_weight;
      }
      Mat PHt(n, m), Sm(m, m), Si;
      for (int a = 0; a < n; ++a) for (int r = 0; r < m; ++r) { double s = 0; for (int k = 0; k < c; ++k) s += P(a, k) * H(r, k); PHt(a, r) = s; }
      for (int r = 0; r < m; ++r) for (int q = 0; q < m; ++q) { double s = 0; for (int k = 0; k < c; ++k) s += H(r, k) * PHt(k, q); Sm(r, q) = s / R + (r == q ? 1.0 : 0.0); }
      if (!invert(Sm, Si)) { h->err = "singular innovation matrix"; if (rep) *rep = rp; return MALIO_ERR_INVALID_ARG; }
      Mat K(n, m);
      for (int a = 0; a < n; ++a) for (int q = 0; q < m; ++q) { double s = 0; for (int r = 0; r < m; ++r) s += PHt(a, r) * Si(r, q); K(a, q) = s / R; }
      for (int a = 0; a < n; ++a) { double s = 0; for (int r = 0; r < m; ++r) s += K(a, r) * hv[r]; Kh[a] = s; }
      for (int a = 0; a < n; ++a) for (int b = 0; b < c; ++b) { double s = 0; for (int r = 0; r < m; ++r) s += K(a, r) * H(r, b); Kx(a, b) = s; }
      for (int a = 0; a < n; ++a) { double s = 0; for (int b = 0; b < c; ++b) s += Kx(a, b) * dxn[b]; KxDx[a] = s; }
      kx_lazy = false;
    } else {                   // :621-637
      // The reference forms Q = (P^-1 + E^T G E)^-1 with two n x n inversions (E = [I_c 0]) and uses only Q[:, 0:c].
      // By the push-through identity  Q E^T = P E^T (I_c + G P_cc)^-1 : one c x c factorisation instead.
      // I + G P_cc has eigenvalues >= 1 (product of two PSD matrices), so the solve is well conditioned.
      // Fixed-size scratch, unit-stride inner loops (this runs once per pass between two kernel sequences, with
      // the GPU idle: every microsecond here is a microsecond of scan latency).
      //   Mt = (I + G P_cc)^T  (row a, col b) = delta_ab + sum_k G(b,k) P(a,k)   [P is symmetric after the
      //   congruence projections above];  solve Mt * Yt = (P[:,0:c])^T  =>  Y = Yt^T = Q[:, 0:c]
      // Per pass only two vectors of Q[:,0:c] are needed: K_h = Q[:,0:c] g and K_x dx_new = Q[:,0:c] (G dx_new), i.e.
      //   S z = rhs  with S = I + G P_cc,   then  P[:,0:c] z.
      // So Mt = S^T is LU-factorised once (partial pivoting, factors kept), the two right-hand sides go through the
      // TRANSPOSED triangular solves (S = U^T L^T Pm), and the full n x c block Q[:,0:c] — 35 right-hand sides — is
      // only solved for in the pass that updates the covariance (below), from the same factors.
      constexpr int CM = MALIO_MAX_COLS;
      const double* Gd = G.a.data();
      const double* Pd = P.a.data();
      for (int a = 0; a < c; ++a)
        for (int b = 0; b < c; ++b) {
          const double* gr = Gd + (size_t)b * c;
          const double* pr = Pd + (size_t)a * n;
          double s = 0.0;
          for (int k = 0; k < c; ++k) s += gr[k] * pr[k];
          LU[a][b] = s + ((a == b) ? 1.0 : 0.0);
        }
      for (int k = 0; k < c; ++k) {          // Pm Mt = L U, L unit lower (multipliers stored below the diagonal)
        int p = k;
        double best = std::fabs(LU[k][k]);
        for (int i = k + 1; i < c; ++i) if (std::fabs(LU[i][k]) > best) { best = std::fabs(LU[i][k]); p = i; }
        if (best == 0.0) { h->err = "singular information matrix"; if (rep) *rep = rp; return MALIO_ERR_INVALID_ARG; }
        piv[k] = p;
        if (p != k) for (int j = 0; j < c; ++j) std::swap(LU[k][j], LU[p][j]);
        const double inv = 1.0 / LU[k][k];
        for (int i = k + 1; i < c; ++i) {
          const double f = LU[i][k] * inv;
          LU[i][k] = f;
          if (f == 0.0) continue;
          for (int j = k + 1; j < c; ++j) LU[i][j] -= f * LU[k][j];
        }
      }
      // S z = rhs:  Mt = Pm^T L U  =>  S = Mt^T = U^T L^T Pm  =>  U^T w = rhs (forward), L^T v = w (backward), z = Pm^T v
      double z1[CM], z2[CM];
      for (int k = 0; k < c; ++k) {
        z1[k] = g[k];
        const double* gr = Gd + (size_t)k * c;
        double sdx = 0.0;
        for (int b = 0; b < c; ++b) sdx += gr[b] * dxn[b];
        z2[k] = sdx;                         // G dx_new
      }
      for (int i = 0; i < c; ++i) {          // U^T w = rhs
        double s1 = z1[i], s2 = z2[i];
        for (int k = 0; k < i; ++k) { s1 -= LU[k][i] * z1[k]; s2 -= LU[k][i] * z2[k]; }
        const double inv = 1.0 / LU[i][i];
        z1[i] = s1 * inv; z2[i] = s2 * inv;
      }
      for (int i = c - 1; i >= 0; --i) {     // L^T v = w  (unit diagonal)
        double s1 = z1[i], s2 = z2[i];
        for (int k = i + 1; k < c; ++k) { s1 -= LU[k][i] * z1[k]; s2 -= LU[k][i] * z2[k]; }
        z1[i] = s1; z2[i] = s2;
      }
      for (int k = c - 1; k >= 0; --k)       // z = Pm^T v: undo the row interchanges in reverse order
        if (piv[k] != k) { std::swap(z1[k], z1[piv[k]]); std::swap(z2[k], z2[piv[k]]); }
      for (int a = 0; a < n; ++a) {          // K_h = P[:,0:c] z1 (:635), K_x dx_new = P[:,0:c] z2 (:637,:642)
        const double* pr = Pd + (size_t)a * n;
        double s = 0.0, u = 0.0;
        for (int k = 0; k < c; ++k) { s += pr[k] * z1[k]; u += pr[k] * z2[k]; }
        Kh[a] = s;
        KxDx[a] = u;
      }
      kx_lazy = true;
    }
    for (int a = 0; a < n; ++a) step[a] = Kh[a] + KxDx[a] - dxn[a];   // dx_ = K_h + (K_x - I) dx_new, :642
    std::memcpy(rp.dx_last, step.data(), sizeof(double) * n);
    boxplus(ly, *x, step.data());          // :646
    redo = true;                           // :649-657
    for (int k = 0; k < n; ++k) if (std::fabs(step[k]) > 0.001) { redo = false; break; }
    if (redo) t++;
    if (!t && it == max_iter - 2) redo = true;   // :660-663
    if (t > 1 || it == max_iter - 1) {     // final covariance, :665-718
      if (kx_lazy) {                       // Q[:,0:c]^T = Mt^-1 P[:,0:c]^T from the stored factors, then K_x = Q[:,0:c] G (:637)
        const double* Gd = G.a.data();
        const double* Pd = P.a.data();
        for (int a = 0; a < c; ++a) for (int j = 0; j < n; ++j) Ykeep[a][j] = Pd[(size_t)a * n + j];   // P(j,a) = P(a,j)
        for (int k = 0; k < c; ++k)          // Pm: all row interchanges first (the stored multipliers were swapped with their rows)
          if (piv[k] != k) for (int j = 0; j < n; ++j) std::swap(Ykeep[k][j], Ykeep[piv[k]][j]);
        for (int k = 0; k < c; ++k) {        // L^-1 (forward, unit diagonal)
          for (int i = k + 1; i < c; ++i) {
            const double f = LU[i][k];
            if (f == 0.0) continue;
            for (int j = 0; j < n; ++j) Ykeep[i][j] -= f * Ykeep[k][j];
          }
        }
        for (int i = c - 1; i >= 0; --i) {   // U^-1 (backward)
          for (int k = i + 1; k < c; ++k) {
            const double f = LU[i][k];
            if (f == 0.0) continue;
            for (int j = 0; j < n; ++j) Ykeep[i][j] -= f * Ykeep[k][j];
          }
          const double inv = 1.0 / LU[i][i];
          for (int j = 0; j < n; ++j) Ykeep[i][j] *= inv;
        }
        double* Kxd = Kx.a.data();
        for (int a = 0; a < n; ++a) {
          double* kr = Kxd + (size_t)a * c;
          for (int b = 0; b < c; ++b) kr[b] = 0.0;
          for (int k = 0; k < c; ++k) {
            const double y = Ykeep[k][a];
            const double* gr = Gd + (size_t)k * c;
            for (int b = 0; b < c; ++b) kr[b] += y * gr[b];
          }
        }
      }
      Mat Lm = P;
      for (int s = 0; s <= ly.L; ++s) {
        const int idx = ly.so3[s];
        const M3 Jt = transpose3(A_matrix(&step[idx]));
        // L rows from P rows (identical at this point for rows idx..idx+2), K_x rows, then L and P columns
        for (int j = 0; j < n; ++j) {
          double v[3] = {P(idx, j), P(idx + 1, j), P(idx + 2, j)};
          for (int a = 0; a < 3; ++a) Lm(idx + a, j) = Jt.m[a][0] * v[0] + Jt.m[a][1] * v[1] + Jt.m[a][2] * v[2];
        }
        left_block<3>(Kx, idx, Jt.m, c);
        right_block_T<3>(Lm, idx, Jt.m);
        right_block_T<3>(P, idx, Jt.m);
      }
      {
        double J2[2][2];
        S2_projection(x->grav, x_prop.grav, &step[ly.grav], J2);
        for (int j = 0; j < n; ++j) {
          const double v0 = P(ly.grav, j), v1 = P(ly.grav + 1, j);
          Lm(ly.grav, j) = J2[0][0] * v0 + J2[0][1] * v1;
          Lm(ly.grav + 1, j) = J2[1][0] * v0 + J2[1][1] * v1;
        }
        left_block<2>(Kx, ly.grav, J2, c);
        right_block_T<2>(Lm, ly.grav, J2);
        right_block_T<2>(P, ly.grav, J2);
      }
      for (int a = 0; a < n; ++a) {        // P_ = L_ - K_x[:,0:c] P_[0:c,:], :714
        double* out = Pio + (size_t)a * n;
        for (int b = 0; b < n; ++b) out[b] = Lm(a, b);
        for (int k = 0; k < c; ++k) {
          const double f = Kx(a, k);
          const double* pr = P.a.data() + (size_t)k * n;
          for (int b = 0; b < n; ++b) out[b] -= f * pr[b];
        }
      }
      host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      rp.converged_count = t;
      rp.last_status = MALIO_OK;
      rp.ms_host_solve = (float)host_ms;
      if (rep) *rep = rp;
      return MALIO_OK;
    }
    host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }
  // every remaining pass was invalid: the reference leaves P_ at its last projected value
  std::memcpy(Pio, P.a.data(), sizeof(double) * n * n);
  rp.converged_count = t;
  rp.last_status = rc_last;
  rp.ms_host_solve = (float)host_ms;
  if (rep) *rep = rp;
  return rc_last == MALIO_OK ? MALIO_OK : MALIO_ERR_NO_EFFECTIVE_POINTS;
}

// ---------------------------------------------------------------- static snapshot builder
namespace {
struct BuildCtx {
  const float* xyz;
  malio_map_node* out;
  uint32_t* order;     // work array of point indices, permuted in place
  uint32_t* order_out;
  uint32_t max_depth;
};
// builds the subtree over order[l..r] rooted at slot `slot`; returns its AABB in box[6]
void build_rec(BuildCtx& C, int64_t l, int64_t r, uint32_t slot, uint32_t depth, float box[6], uint32_t& max_depth) {
  if (depth > max_depth) max_depth = depth;
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t i = l; i <= r; ++i) {
    const float* p = C.xyz + 3 * (size_t)C.order[i];
    for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], p[k]); mx[k] = std::max(mx[k], p[k]); }
  }
  int axis = 0;   // longest extent (ikd_Tree.cpp:712-716)
  for (int k = 1; k < 3; ++k) if (mx[k] - mn[k] > mx[axis] - mn[axis]) axis = k;
  const int64_t mid = (l + r) >> 1;
  std::nth_element(C.order + l, C.order + mid, C.order + r + 1, [&](uint32_t a, uint32_t b) {
    return C.xyz[3 * (size_t)a + axis] < C.xyz[3 * (size_t)b + axis];
  });
  malio_map_node& o = C.out[slot];
  const float* p = C.xyz + 3 * (size_t)C.order[mid];
  o.x = p[0]; o.y = p[1]; o.z = p[2];
  C.order_out[slot] = C.order[mid];
  uint32_t link = 0;
  for (int k = 0; k < 6; ++k) { o.lbox[k] = 0.f; o.rbox[k] = 0.f; }
  const int64_t nl = mid - l, nr = r - mid;
  if (nl > 0) { link |= MALIO_LINK_HAS_LEFT; }
  if (nr > 0) { link |= MALIO_LINK_HAS_RIGHT | (uint32_t)(slot + 1 + nl); }
  o.link = link;
  for (int k = 0; k < 3; ++k) { box[2 * k] = mn[k]; box[2 * k + 1] = mx[k]; }
  float lb[6], rb[6];
  uint32_t dl = depth, dr = depth;
  const bool spawn = (r - l) > 65536;
  if (nl > 0 && nr > 0 && spawn) {
#pragma omp task shared(C, lb, dl) firstprivate(l, mid, slot, depth)
    build_rec(C, l, mid - 1, slot + 1, depth + 1, lb, dl);
#pragma omp task shared(C, rb, dr) firstprivate(r, mid, slot, depth, nl)
    build_rec(C, mid + 1, r, (uint32_t)(slot + 1 + nl), depth + 1, rb, dr);
#pragma omp taskwait
  } else {
    if (nl > 0) build_rec(C, l, mid - 1, slot + 1, depth + 1, lb, dl);
    if (nr > 0) build_rec(C, mid + 1, r, (uint32_t)(slot + 1 + nl), depth + 1, rb, dr);
  }
  if (nl > 0) std::memcpy(o.lbox, lb, sizeof(lb));
  if (nr > 0) std::memcpy(o.rbox, rb, sizeof(rb));
  max_depth = std::max(max_depth, std::max(dl, dr));
}
}  // namespace

int malio_build_static_snapshot(const float* xyz, uint32_t n, malio_map_node* nodes_out, uint32_t* order_out, uint32_t* max_depth_out) {
  if (n == 0) { if (max_depth_out) *max_depth_out = 0; return MALIO_OK; }
  if (!xyz || !nodes_out || !order_out || n > MALIO_LINK_INDEX_MASK) return MALIO_ERR_INVALID_ARG;
  std::vector<uint32_t> order(n);
  std::iota(order.begin(), order.end(), 0u);
  BuildCtx C{xyz, nodes_out, order.data(), order_out, 0};
  float box[6];
  uint32_t md = 0;
#pragma omp parallel
#pragma omp single
  build_rec(C, 0, (int64_t)n - 1, 0, 1, box, md);
  if (max_depth_out) *max_depth_out = md;
  return MALIO_OK;
}

}  // extern "C"
