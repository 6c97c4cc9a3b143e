/*
 * malio_b200.h — C-ABI of the H100-native (sm_90a) MA-LIO measurement hot path.
 *
 * Drop-in boundary (SURVEY.md §8b).  The reference's plug-in point is the IKFoM
 * measurement-model callback
 *     typedef void measurementModel_dyn_share(state&, dyn_share_datastruct<double>&)
 *         MA_LIO/include/IKFoM_toolkit/esekfom/esekfom.hpp:130   (installed :152-168, invoked :512)
 * implemented by
 *     void h_share_model(state_ikfom&, esekfom::dyn_share_datastruct<double>&)
 *         MA_LIO/src/laserMapping.cpp:552-760
 * which in turn calls
 *     KD_TREE::Nearest_Search(PointType, int k, PointVector&, vector<float>&, float)
 *         MA_LIO/include/ikd-Tree/ikd_Tree.h:328 / ikd_Tree.cpp:426-461  (call site laserMapping.cpp:586)
 * and whose N_eff x 24 output is reduced by
 *     esekf::update_iterated_dyn_share_modified        esekfom.hpp:495-721  (O(N) part :621-637).
 *
 * Because the device path fuses the H^T R^-1 H / H^T R^-1 h reduction, this ABI sits one
 * level above the callback: malio_measure() replaces h_share_model *and* esekfom.hpp:622-635
 * and returns the reduced c x c system.  malio_ieskf_update() is the host-side iterated
 * update (replaces esekfom.hpp:495-721 as a whole).
 *
 * Conventions: plain C types only; caller owns every host buffer (pinned memory recommended);
 * the handle owns device memory, streams, events and the NCCL communicator.  Every call returns
 * a malio_status; calls on one handle must come from one thread at a time; all calls are
 * synchronous at return unless stated otherwise.
 */
#ifndef MALIO_B200_H_
#define MALIO_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MALIO_MAX_LIDAR 3   /* use-ikfom.hpp:14-27 builds the manifold for 3 LiDARs; L is run-time here (1..3) */
#define MALIO_K 5           /* NUM_MATCH_POINTS, common_lib.h:22 */
#define MALIO_MAX_COLS (6 * (MALIO_MAX_LIDAR + 1))            /* c = 6(L+1), laserMapping.cpp:642 */
#define MALIO_MAX_DOF (17 + 6 * MALIO_MAX_LIDAR)              /* n = 17+6L, esekfom.hpp:158 */
#define MALIO_MAX_TREE_DEPTH 96                              /* traversal stack bound; deeper snapshots are rejected */
#define MALIO_NCCL_UNIQUE_ID_BYTES 128

typedef enum malio_status {
  MALIO_OK = 0,
  MALIO_ERR_INVALID_ARG = 1,
  MALIO_ERR_CUDA = 2,          /* CUDA runtime / driver failure (no GPU, OOM, launch error) */
  MALIO_ERR_NCCL = 3,
  MALIO_ERR_NO_EFFECTIVE_POINTS = 4, /* N_eff == 0: reference sets valid=false (laserMapping.cpp:635-639) */
  MALIO_ERR_STATE = 5,         /* call order violated (e.g. measure before upload) */
  MALIO_ERR_TREE_TOO_DEEP = 6,
  MALIO_ERR_CAPACITY = 7
} malio_status;

/* ---- map snapshot: one record per live ikd-Tree node, DFS pre-order ---------------------------
 * Mirrors what KD_TREE::Search reads per visit (ikd_Tree.cpp:1073-1255): the node's point, its
 * point_deleted flag, and both children's node_range_* boxes (KD_TREE_NODE, ikd_Tree.h:59-82),
 * after Push_Down (ikd_Tree.cpp:1371-1466).  tree_deleted subtrees are not exported (Search
 * returns immediately on them, :1075).  The left child of node i, when present, is node i+1. */
typedef struct malio_map_node {
  float x, y, z;
  uint32_t link;      /* bits 0..27 index of the right child; bit 31 has_left; bit 30 has_right;
                         bit 29 point_deleted */
  float lbox[6];      /* left child's {x_min,x_max,y_min,y_max,z_min,z_max}; undefined if !has_left */
  float rbox[6];      /* right child's */
} malio_map_node;     /* 64 bytes */

#define MALIO_LINK_HAS_LEFT  0x80000000u
#define MALIO_LINK_HAS_RIGHT 0x40000000u
#define MALIO_LINK_POINT_DELETED 0x20000000u
#define MALIO_LINK_INDEX_MASK 0x0FFFFFFFu

/* Compact snapshot record = the first 16 bytes of malio_map_node.  With malio_upload_map_compact() the host ships only
 * these (plus the map-side weights): 20 bytes per node instead of 68, and the device rebuilds both children's boxes
 * of every node bottom-up as the tight bounding box of the live (not point_deleted) points below — which is what
 * KD_TREE::Update maintains in node_range_* (ikd_Tree.cpp:1469-1635). */
typedef struct malio_map_point {
  float x, y, z;
  uint32_t link;      /* as in malio_map_node */
} malio_map_point;    /* 16 bytes */

/* ---- scan point: feats_down_body entry as h_share_model reads it (laserMapping.cpp:565-570,694) */
typedef struct malio_scan_pt {
  float x, y, z;        /* point in its own LiDAR frame */
  uint16_t lidar;       /* PointType::intensity after laserMapping.cpp:975 */
  uint16_t table_idx;   /* int(PointType::normal_x), laserMapping.cpp:694,737 */
} malio_scan_pt;        /* 16 bytes */

/* ---- one entry of pose_unc[l][j] (struct Pose, common_lib.h:57-63): only T_ and cov_ are read by
 * evalPointUncertainty (associate_uct.hpp:153-175) */
typedef struct malio_pose_entry {
  double T[16];        /* row-major 4x4 */
  double cov[36];      /* row-major 6x6 */
} malio_pose_entry;

typedef struct malio_rigid {
  double q[4];         /* w, x, y, z */
  double t[3];
} malio_rigid;

/* ---- pose part of state_ikfom read by h_share_model (use-ikfom.hpp:14-27; extrinsic_update,
 * laserMapping.cpp:291-308) */
typedef struct malio_pass_state {
  double rot[4];       /* s.rot, (w,x,y,z) */
  double pos[3];       /* s.pos */
  malio_rigid ext[MALIO_MAX_LIDAR];   /* offset_R_l / offset_T_l */
} malio_pass_state;

/* ---- run-time parameters (parameters.cpp:17-66; launch/mapping_city.launch:9-15; City.yaml:41-50) */
typedef struct malio_params {
  int32_t n_lidar;            /* L, 1..3 */
  int32_t extrinsic_est_en;   /* laserMapping.cpp:681 */
  float plane_th;             /* esti_plane threshold, common_lib.h:184 */
  float knn_max_sqdist;       /* 5.0f, laserMapping.cpp:587 */
  double cov_threshold;
  double point_cov_max, point_cov_min;
  double plane_cov_max, plane_cov_min;
  double localize_cov_max, localize_cov_min;
  double localize_thresh_max, localize_thresh_min;
  double range_min, range_max;
} malio_params;

typedef struct malio_config {
  malio_params params;
  int32_t device;             /* CUDA device ordinal */
  int32_t sort_queries;       /* 1: Morton-order the scan on the device (internal; outputs stay in caller order) */
  uint32_t max_points;        /* capacity hints; buffers grow on demand when 0 */
  uint32_t max_map_nodes;
  float knn_cell_size;        /* k-NN fast path: edge of the cell-list index built over the snapshot at upload
                                 (metres).  0 = automatic (starts at 1 m = 2 x filter_size_map), < 0 = index off:
                                 every query walks the flattened ikd-Tree.  Results are identical either way. */
} malio_config;

typedef struct malio_pass_stats {
  uint32_t n_points;          /* N of this rank's shard */
  uint32_t n_eff;             /* effct_feat_num, summed over ranks */
  int32_t valid;              /* dyn_share.valid */
  int32_t searched;           /* 1 if this pass ran the k-NN */
  double u_min, u_max;        /* min/max_unit_cov, laserMapping.cpp:615-628 */
  double tau_min, tau_max;    /* min/max_cov, laserMapping.cpp:646-703 */
  double sigma[3];            /* singular values of h_x[:,0:3] before the localization weight */
  double loc_weight;          /* weight, laserMapping.cpp:749-756 */
  float ms_sort;              /* Morton keys + sort of the scan (first pass of a scan only, else 0) */
  float ms_knn, ms_plane, ms_reduce, ms_total;   /* device time of this pass (CUDA events); ms_knn = the k-NN kernel alone */
} malio_pass_stats;

typedef struct malio_handle malio_handle;

/* fill p with the reference defaults for L LiDARs (City.yaml / mapping_city.launch values) */
void malio_default_params(malio_params* p, int n_lidar);

int malio_create(malio_handle** out, const malio_config* cfg);
void malio_destroy(malio_handle* h);
const char* malio_last_error(const malio_handle* h);   /* static storage when h == NULL */
const char* malio_version(void);

/* multi-GPU: one process per GPU.  Rank 0 calls malio_get_nccl_unique_id and ships the bytes to the
 * other ranks (torch.distributed / MPI / a socket — plumbing); every rank then calls malio_comm_init.
 * With a communicator attached, malio_measure all-reduces {min,max} and the reduced system over the
 * ranks; each rank uploads only its own block of scan points. */
int malio_get_nccl_unique_id(uint8_t id[MALIO_NCCL_UNIQUE_ID_BYTES]);
int malio_comm_init(malio_handle* h, const uint8_t id[MALIO_NCCL_UNIQUE_ID_BYTES], int rank, int world);

/* once per scan: flattened ikd-Tree snapshot (include/malio_flatten.hpp produces it) and the map-side
 * weight normal_y of every node (quirk: an input field, SURVEY.md §8a-1).  root is node 0. */
int malio_upload_map(malio_handle* h, const malio_map_node* nodes, const float* node_cov,
                     uint32_t n_nodes, uint32_t max_depth);

/* Same snapshot in compact form (see malio_map_point): 3.4x less host->device traffic per scan.
 * root_box (optional, may be NULL): {x_min,x_max,y_min,y_max,z_min,z_max} bounding every live point — the ikd-Tree
 * root's node_range_* — saves the read-back of the rebuilt root record. */
int malio_upload_map_compact(malio_handle* h, const malio_map_point* pts, const float* node_cov,
                             uint32_t n_nodes, uint32_t max_depth, const float* root_box);
/* test / debug: read back the device-resident 64-byte node records (boxes included). */
int malio_download_map_nodes(malio_handle* h, malio_map_node* out, uint32_t capacity);

/* once per scan: this rank's block of the down-sampled merged scan + the pose tables.
 * table holds pose_unc[0], pose_unc[1], ... back to back; pose_unc[l] = table[table_off[l] .. table_off[l+1]).
 * temporal_comp[l-1] is kf.temporal_comp[l-1] (IMU_Processing.hpp:517-519), l = 1..L-1. */
int malio_upload_scan(malio_handle* h, const malio_scan_pt* pts, uint32_t n_pts,
                      const malio_pose_entry* table, const uint32_t* table_off /* L+1 */,
                      const malio_rigid* temporal_comp /* L-1, may be NULL when L==1 */);

/* re-arm the scan that is already resident on the device (same points / tables as the last malio_upload_scan):
 * resets the per-scan state (Nearest_Points, point_selected_surf, internal ordering) without any host copy.
 * Lets a caller time the device path with inputs resident in HBM. */
int malio_rearm_scan(malio_handle* h);

/* one pass of h_share_model + esekfom.hpp:622-635.
 *   HtRinvH : c x c row-major, = h_x^T diag(1/R) h_x   (HTH, esekfom.hpp:629)
 *   HtRinvh : c,              = h_x^T diag(1/R) h     (HT * dyn_share.h, esekfom.hpp:635)
 * redo_knn = dyn_share.converge on entry (laserMapping.cpp:583).
 * Returns MALIO_ERR_NO_EFFECTIVE_POINTS (stats->valid = 0) when N_eff == 0. */
int malio_measure(malio_handle* h, const malio_pass_state* s, int redo_knn,
                  double* HtRinvH, double* HtRinvh, malio_pass_stats* stats);

/* rows of the last pass for the degenerate branch n > N_eff (esekfom.hpp:574-582): up to cap rows of
 * h_x (row-major, c columns) and h, in the library's internal (cell-sorted) point order — with a communicator attached the
 * rows of all ranks, concatenated in rank order — scaled by the plane weight (laserMapping.cpp:714-715) but NOT yet by
 * the localization weight: multiply by stats->loc_weight (laserMapping.cpp:758-759), as malio_ieskf_update does. */
int malio_download_rows(malio_handle* h, double* h_x, double* hvec, uint32_t cap, uint32_t* n_rows);

/* side outputs of the last pass, caller order; any pointer may be NULL.
 *   normal_y : trace of the point covariance for all N points (laserMapping.cpp:699,730,741)
 *   nn_idx   : N x 5 snapshot node indices, ascending by (distance, x) as Nearest_Search returns them;
 *              0xFFFFFFFF where fewer than 5 were found
 *   nn_sqdist: N x 5
 *   selected : point_selected_surf after the pass
 *   world    : N x 3 feats_down_world (laserMapping.cpp:576-578) */
int malio_download_aux(malio_handle* h, float* normal_y, uint32_t* nn_idx, float* nn_sqdist,
                       uint8_t* selected, float* world);

/* ---- next to the path (SURVEY.md §8f N1): map_incremental's per-point decision ------------------------
 * laserMapping.cpp:398-446, evaluated on the device from what the last pass left there (Nearest_Points of the last
 * search, normal_y) and the state AFTER the update (pointBodyToWorld, laserMapping.cpp:134-147).  Caller order.
 *   cls[i] = MALIO_MAP_SKIP   normal_y > cov_threshold (:406)
 *            MALIO_MAP_ADD    goes to PointToAdd            -> ikdtree.Add_Points(.., true)   (:434, :437, :440)
 *            MALIO_MAP_ADD_NO_DOWNSAMPLE  PointNoNeedDownsample -> ikdtree.Add_Points(.., false)  (:421-425)
 *            MALIO_MAP_DROP   a neighbour is closer to the voxel centre (:428-433)
 *   world : N x 3 feats_down_world for the points that were not skipped (zeros for skipped ones); may be NULL
 * filter_size_map = filter_size_map_min, ekf_inited = flg_EKF_inited (laserMapping.cpp:989). */
#define MALIO_MAP_SKIP 0
#define MALIO_MAP_ADD 1
#define MALIO_MAP_ADD_NO_DOWNSAMPLE 2
#define MALIO_MAP_DROP 3
int malio_map_incremental(malio_handle* h, const malio_pass_state* s, double filter_size_map, int ekf_inited,
                          uint8_t* cls, float* world);

/* ---- next to the path (SURVEY.md §8f N3): the pose-uncertainty table that feeds malio_upload_scan -------------
 * struct Pose (common_lib.h:57-63) and Barfoot's 4th-order SE(3) covariance compounding
 * (associate_uct.hpp:29-142), host C++.  Output arguments MAY alias the second input pose exactly as the reference's
 * call sites do (laserMapping.cpp:1042-1044): the functions touch the fields in the reference's order, so the
 * aliasing behaviour (adjointMatrix sees the already overwritten T_, associate_uct.hpp:99) is reproduced. */
typedef struct malio_pose {
  double q[4];        /* q_, (w,x,y,z) */
  double t[3];        /* t_ */
  double T[16];       /* T_, row-major 4x4 */
  double cov[36];     /* cov_, row-major 6x6 */
} malio_pose;

/* PoseInitial (common_lib.h:129-142) */
void malio_pose_initial(malio_pose* pose, const double t[3], const double q[4], const double cov[36]);
/* compoundPoseWithCov, method 2 (associate_uct.hpp:88-142); also sets pose_cp->cov (:134) */
void malio_compound_pose_with_cov(const malio_pose* pose_1, const double cov_1[36], const malio_pose* pose_2,
                                  const double cov_2[36], malio_pose* pose_cp, double cov_cp[36]);
/* compoundInvPoseWithCov, method 2 (associate_uct.hpp:29-86); does NOT touch pose_cp->cov unless cov_cp points to it */
void malio_compound_inv_pose_with_cov(const malio_pose* pose_1, const double cov_1[36], const malio_pose* pose_2,
                                      const double cov_2[36], malio_pose* pose_cp, double cov_cp[36]);
/* pose_unc of one scan (laserMapping.cpp:1028-1048) in the layout malio_upload_scan takes.
 *   extrinsic[l]            struct Pose of LiDAR l's extrinsic, l < n_lidar
 *   temporal_comp[l-1]      kf.temporal_comp[l-1], l = 1..n_lidar-1 (may be NULL when n_lidar == 1)
 *   lidar_uncertainty[l]    kf.lidar_uncertainty[l][0 .. counts[l]); the LAST entry of each list is dropped (:1035,:1040)
 * table must hold sum(counts[l] - 1) entries; table_off gets n_lidar + 1 offsets.  Returns the number of entries,
 * or a negative malio_status. */
int malio_build_pose_unc(int n_lidar, const malio_pose* extrinsic, const malio_pose* temporal_comp,
                         const malio_pose* const* lidar_uncertainty, const uint32_t* counts,
                         malio_pose_entry* table, uint32_t* table_off);

/* ---- next to the path (SURVEY.md §8f N2): per-raw-point B-spline undistortion ------------------------------------
 * ImuProcess::UndistortPcl's point loop (IMU_Processing.hpp:468-508) for ONE LiDAR: per raw point the spline pose
 * BsplineSE3::get_pose (BsplineSE3.cpp:84-118: 3 x exp_se3(b * log_se3(.)), quat_ops.h:190-243), the motion compensation
 * into the LiDAR's scan-end frame (:492) and the walk of the IMU-covariance list that yields the point's uncertainty-table
 * index (:476-486, written to `intensity` :496).  On the device the log_se3 of every control-point pair is taken once,
 * each point evaluates three exp_se3, and the sequential one-pop-per-point walk is computed as a min-plus prefix scan.
 * Points arrive in buffer order (ascending time); like the reference the loop runs from the last point down to the
 * SECOND one — point 0 is never touched.  Where get_pose fails the point keeps its coordinates and `intensity`. */
typedef struct malio_raw_pt {
  float x, y, z;
  float curvature;      /* time offset from the scan start in ms (preprocess.cpp:91,139,200) */
} malio_raw_pt;

typedef struct malio_undistort_args {
  double beg_time;            /* meas.lidar_beg_time[lid_num - num - 1] (:474) */
  malio_rigid extrinsic;      /* extrinsic_quat[num], extrinsic_trans[num] */
  malio_rigid lt_imu_frame;   /* lt_imu_frame_quat[num], lt_imu_frame_trans[num]: IMU pose at this LiDAR's scan end */
  const double* ctrl_t;       /* spline control points: timestamps ascending (BsplineSE3::control_points keys) */
  const double* ctrl_T;       /* ... and their 4x4 poses, row-major, n_ctrl x 16 */
  uint32_t n_ctrl;            /* <= MALIO_MAX_CTRL */
  const double* imu_cov_t;    /* imu_cov[k].first.first, ascending */
  uint32_t n_cov;             /* <= MALIO_MAX_COV */
  int32_t cov_pointer;        /* its value when the point loop starts (:455-466) */
} malio_undistort_args;
#define MALIO_MAX_CTRL 512
#define MALIO_MAX_COV 512
#define MALIO_IDX_UNTOUCHED INT32_MIN

/* lidar = slot (0..L-1) whose device-resident result malio_voxel_grid(.., NULL input) picks up.  Host outputs (any may be
 * NULL): xyz n x 3 float; idx n (the value the reference writes to `intensity`, MALIO_IDX_UNTOUCHED where it writes nothing);
 * ok n (spline_flag); pop_point[k] = index of the point at which the k-th table entry is pushed (:487-494), n_pops their
 * number (malio_scan_uncertainty builds the table entries from them on the device); pose n x 7 (q wxyz, p).  The handle keeps
 * the slot's pop points, spline poses, cov_pointer, lt_imu_frame and n_cov for malio_scan_uncertainty. */
int malio_undistort(malio_handle* h, int lidar, const malio_raw_pt* pts, uint32_t n, const malio_undistort_args* a,
                    float* xyz, int32_t* idx, uint8_t* ok, int32_t* pop_point, uint32_t* n_pops, double* pose);

/* BsplineSE3::get_pose on the host (lt_imu_frame poses, the <= n_cov table-entry poses).  q = (w,x,y,z).  1 on success. */
int malio_bspline_get_pose(const double* ctrl_t, const double* ctrl_T, uint32_t n_ctrl, double timestamp, double q[4], double p[3]);

/* ---- next to the path (SURVEY.md §8f N3, second half): pcl::VoxelGrid down-sampling (laserMapping.cpp:968-983) --------
 * PCL's filter with setLeafSize(leaf, leaf, leaf) and default settings restated on the device: voxel index
 * floor(x / leaf) relative to the cloud's minimum, one output point per occupied voxel in ascending voxel index, every
 * field the centroid of the voxel's points (float sums taken in ascending input index).  What the hot path reads of the
 * result is x, y, z and the averaged `intensity` (the table index, moved to normal_x at :975).
 * in == NULL: take the device-resident output of the last malio_undistort*(h, lidar, ...) (x, y, z, intensity = idx,
 * curvature; points the undistortion left untouched keep intensity 0); MALIO_ERR_STATE when that call did not complete (an
 * unordered cloud given to malio_undistort_device).  in != NULL: n x 5 floats
 * {x, y, z, intensity, curvature} from the host.  Outputs (may be NULL): out n_out x 5 floats, same layout, at most out_cap
 * of them; *n_out = the full count.  Non-finite points are skipped; a cloud without a finite point gives n_out = 0.
 * MALIO_ERR_CAPACITY (nothing computed) when the grid has more than 2^28 voxels, more than 2^24 voxels along one axis, or
 * a voxel index floor(x / leaf) outside int.  PCL accepts up to 2^31 voxels, but its per-axis index is a float
 * subtraction that can round up to the axis' size above 2^24 voxels; such leaf sizes are refused here instead.
 * The down-sampled cloud also stays on the device as LiDAR `lidar`'s part of the next scan (malio_upload_scan_device). */
int malio_voxel_grid(malio_handle* h, int lidar, const float* in, uint32_t n, float leaf, float* out, uint32_t out_cap,
                     uint32_t* n_out);

/* Merge the device-resident down-sampled clouds of LiDARs 0..L-1 (feats_down_body = sum of feats_down_vec[num],
 * laserMapping.cpp:983; lidar id -> `intensity`, int(averaged intensity) -> table_idx) into the scan of the handle without
 * a host bounce; then as malio_upload_scan.  n_total (optional) receives the merged size. */
int malio_upload_scan_device(malio_handle* h, const malio_pose_entry* table, const uint32_t* table_off,
                             const malio_rigid* temporal_comp, uint32_t* n_total);

/* ---- next to the path (SURVEY.md §8f N2, second half): the scan's pose-uncertainty table from its undistortion ----------
 * The rest of UndistortPcl (IMU_Processing.hpp:474-523) and the pose_unc loop of laserMapping.cpp:1028-1048, on the device,
 * after malio_undistort has run on every slot 0..L-1 of the scan.  For the k-th pop point of slot num (pop_point[k]):
 *   uncertainty[num][k] = inv(extrinsic[num]) * inv(lt_lidar_frame[num]) * (PoseInitial(spline pose, imu_cov[c0 - k]) * extrinsic[num])
 * with the reference's three compoundings (:487-492) and the spline pose undistort_kernel compensated that point with, bit for
 * bit; c0 = that slot's cov_pointer, lt_lidar_frame[0] = PoseInitial(lt_imu_frame[0], getUncertainty()) (:450) and
 * lt_lidar_frame[num] = PoseInitial(lt_imu_frame[num], imu_cov[c0]) (:471).  temporal_comp[num-1] = lt_lidar_frame[0]^-1
 * lt_lidar_frame[num] (:518).  pose_unc[num] = all but the last entry of uncertainty[num] (:1035, :1040), LiDARs >= 1 moved into
 * LiDAR 0's frame by the compoundings of :1042-1044 (outputs aliasing the second input).  A slot with 0 or 1 pops gets no entry.
 * A pop point the spline cannot reach: the reference reads an uninitialised quaternion there (get_pose, BsplineSE3.cpp:91-96,
 * sets the translation to zero and a local rotation matrix to the identity, but never the quaternion); this library uses the
 * identity rotation with zero translation (DESIGN.md, quirk 8c of §8(a)).
 * extrinsic is the same struct Pose for both sources: the state's extrinsic and getExtrinsicUncertainty(num) are unchanged by
 * the prediction between laserMapping.cpp:952 and IMU_Processing.hpp:448.
 * Matrices are row-major.  Eigen's M6D (Matrix<double,6,6>) is column-major: pass kf.getUncertainty() and every imu_cov[k]
 * through Eigen::Map<Eigen::Matrix<double,6,6,Eigen::RowMajor>> (or transpose), and build malio_pose.cov the same way. */
typedef struct malio_scan_unc_args {
  const double* imu_cov;        /* n_cov x 36: imu_cov[k].first.second, the list (same order) whose times malio_undistort got */
  uint32_t n_cov;               /* must equal the n_cov of every malio_undistort call of the scan */
  const malio_pose* extrinsic;  /* L: PoseInitial(extrinsic[num], t, q, kf.getExtrinsicUncertainty(num)) (:444-448) */
  const double* uncertainty;    /* 36: kf.getUncertainty() (:450) */
} malio_scan_unc_args;
/* Outputs, copied from the device in one transfer: table / table_off (L + 1) as malio_upload_scan and malio_upload_scan_device
 * take them; temporal_comp L - 1 poses (may be NULL when L == 1; malio_rigid = its q and t); lidar_unc (may be NULL) the lists
 * kf.lidar_uncertainty back to back in slot order, sum of the slots' n_pops entries; lidar_unc_counts (may be NULL) their L sizes.
 * MALIO_ERR_STATE when a slot 0..L-1 has not been undistorted; MALIO_ERR_INVALID_ARG for a NULL argument, an n_cov other than
 * the undistort calls saw, or a slot >= 1 whose cov_pointer is -1; MALIO_ERR_CAPACITY when the table needs more than table_cap
 * entries (the needed number is in table_off[L]).  No kernel runs on any error. */
int malio_scan_uncertainty(malio_handle* h, const malio_scan_unc_args* a, malio_pose_entry* table, uint32_t table_cap,
                           uint32_t* table_off, malio_pose* temporal_comp, malio_pose* lidar_unc, uint32_t* lidar_unc_counts);

/* ---- after the update (SURVEY.md §3.1): publish_frame_world and the saved map (laserMapping.cpp:448-489, :1076-1077) --------
 * RGBpointBodyToWorld (:149-163) per point, on the device, with the state AFTER the update (pass a malio_pass_state built from
 * the updated malio_state, as for malio_map_incremental; extrinsics from the state, extrinsic_update :291-308) and the temporal
 * compensation of the last malio_upload_scan* (identity before the first):
 *   lid = int(intensity); p_w = rot (q_E[0] p + t_E[0]) + pos                                   (lid == 0)
 *                         p_w = rot (q_C[lid-1] (q_E[lid] p + t_E[lid]) + t_C[lid-1]) + pos     (otherwise)
 * in double, stored as float, and intensity_out = the input point's normal_y.  The xyz are bit-identical to
 * malio_map_incremental's world output (pointBodyToWorld, :134-147, is the same expression).  The output cloud is n x 4 floats
 * {x, y, z, intensity}; as PointXYZINormal its normal_x/y/z and curvature are 0.  The two clouds of :452:
 *   MALIO_WORLD_DOWNSAMPLED  feats_down_body: the handle's scan in caller order (lid = its `lidar` field), intensity = normal_y of
 *                            the last pass (what malio_download_aux returns).  MALIO_ERR_STATE before a malio_measure /
 *                            malio_ieskf_update on the current scan.
 *   MALIO_WORLD_DENSE        feats_undistort (:977-981): the device-resident results of the last malio_undistort of slots
 *                            0..L-1, concatenated in slot order, each in its own buffer order, point 0 and the points the
 *                            spline could not reach included as they are (lid = slot).  intensity = the raw points' normal_y,
 *                            which sync_packages sets to the cloud's position in lidar_buffer (:321-322) — not the slot in
 *                            general (feats_undistort_vec[num] = lidar_multi[lid_num-num-1], IMU_Processing.hpp:231) — given
 *                            per slot in slot_tag[L].  MALIO_ERR_STATE until malio_undistort has run on every slot 0..L-1
 *                            (0 points is a valid, empty slot).
 * With a communicator attached every rank registers what it holds (its block of the scan, its own slots); nothing is gathered.
 * Neither call changes what any other entry point returns. */
#define MALIO_WORLD_DOWNSAMPLED 0
#define MALIO_WORLD_DENSE 1
/* publish_frame_world's cloud (scan_pub_en, dense_pub_en selects the source): at most cap points to out (n x 4 floats; out may
 * be NULL when cap == 0, to ask the size), *n_out = the full count.  slot_tag: L floats, dense only (may be NULL otherwise). */
int malio_world_register(malio_handle* h, const malio_pass_state* s, int source, const float* slot_tag, float* out, uint32_t cap,
                         uint32_t* n_out);
/* pcd_save_en: pcl_wait_save += the registered DENSE cloud (:468-475), kept on the device (16 B per point, no copy to the host).
 * The buffer starts at 65536 points and at least doubles whenever it grows (device-side copy); a failed allocation returns
 * MALIO_ERR_CUDA and leaves the accumulated cloud intact.  n_total (may be NULL) = points accumulated since the last clear. */
int malio_world_accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, uint64_t* n_total);
/* pcd_writer.writeBinary(path, *pcl_wait_save) (:484, :1090), copied out in chunks through a pinned buffer and written by the
 * same code as malio_write_pcd_binary; clear != 0 then empties the cloud (pcl_wait_save->clear(), :485).  MALIO_ERR_STATE on an
 * empty cloud, MALIO_ERR_INVALID_ARG when the file cannot be opened or written; no file is left behind on any error.  The
 * scan_wait_num / pcd_save_interval bookkeeping and the file names (scans_<k>.pcd, result.pcd) stay with the caller. */
int malio_world_save_pcd(malio_handle* h, const char* path, int clear);
/* The saved map as a voxel map (opt-in, beside the dense cloud above; a deliberate extension beyond the reference's dense file):
 * memory grows with the occupied voxels, work per call with the scan.  The map holds exactly the points malio_world_accumulate
 * would append, in its order (slots 0..L-1, point order, scan after scan; the xyz are world_kernel's bits), folded per voxel
 * into a centroid {x, y, z, intensity} with intensity = slot_tag averaged like every other field.  It is defined as
 * malio_voxel_grid (pcl::VoxelGrid) applied to the concatenation of those dense clouds, with absolute voxel indices:
 *   voxel of a point   (int)floorf(x * il) per axis, il = 1.0f / leaf in float (PCL's relative index gives the same voxel
 *                      wherever |floorf(x * il)| < 2^24); points with a non-finite coordinate are skipped
 *   centroid           float sums from 0.f continued point by point in that order across all scans, a u32 count, sum / count
 *   order              ascending voxel index (k, j, i) as signed ints: z, then y, then x
 * malio_world_voxel_accumulate folds the current dense cloud in: the preconditions and errors of malio_world_accumulate
 * (MALIO_ERR_STATE until malio_undistort* has run on every slot 0..L-1, slot_tag required), and MALIO_ERR_INVALID_ARG for a leaf
 * that is not finite and > 0 or that differs from the map's (fixed by the first call after creation or a clearing save).  A
 * point whose voxel index falls outside int returns MALIO_ERR_CAPACITY with the map unchanged.  The call waits once, at its
 * end, for the voxel count and that verdict; growing the table first drains the handle's stream.  n_voxels may be NULL.
 * malio_world_voxel_download_device: the centroids in order as n x 4 floats into device memory, with the size protocol of
 * malio_world_register_device (d_out == NULL and cap == 0 asks the size, *n_out = the full count, at most cap written) and its
 * device-memory contract (pointer checks before anything is enqueued, 16-byte alignment, ordered on `stream`, returns after
 * enqueueing).
 * malio_world_voxel_save_pcd: the centroids in order through malio_world_save_pcd's writer; MALIO_ERR_STATE on an empty map;
 * clear != 0 then empties the map and releases its leaf.
 * Device memory: 32 B per entry (key, sums, count; the entries at least double when they grow) and a hash of 4 B per slot at
 * most half full, plus scratch for the scan (48 B per point).  The sort by key of a download or a save needs 32 B per voxel more;
 * a download keeps that area until the next save, a save releases it (and writes through it, with no further copy).
 * malio_world_voxel_info: voxels in use, entry capacity, and the device bytes the voxel map holds now, scratch included (any may
 * be NULL). */
int malio_world_voxel_accumulate(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf, uint64_t* n_voxels);
int malio_world_voxel_download_device(malio_handle* h, float* d_out, uint64_t cap, uint64_t* n_out, void* stream);
int malio_world_voxel_save_pcd(malio_handle* h, const char* path, int clear);
int malio_world_voxel_info(malio_handle* h, uint64_t* n_voxels, uint64_t* capacity, uint64_t* device_bytes);
/* Clearing moving objects out of the voxel map: free-space evidence per voxel, counted while the scans are accumulated, and a
 * save without the voxels that later rays passed straight through (a car's trail along its lane).  tests/carve_ref.py restates
 * every step in numpy.
 * malio_world_voxel_accumulate_carve does to the centroids exactly what malio_world_voxel_accumulate does (same bits, same
 * preconditions and errors), then counts this scan, one scan per call, into two u32 counters per voxel:
 *   hit(v)  += 1 when at least one finite point of this scan has its key in v
 *   miss(v) += 1 when v is in the map after this scan's fold, no point of this scan has its key in v, and at least one ray of
 *           this scan passes v
 * Both are set semantics over the scan: thread order cannot change them.  Entries created by malio_world_voxel_accumulate
 * start at hit = miss = 0, and those calls change no counter.
 * A ray belongs to each finite dense point p of slot l (the points the fold takes, their world bits w):
 *   origin o = body_to_world(s, l, (0, 0, 0)), the float bits malio_world_register gives for a point at the slot's origin
 *   u = o * il, e = w * il per axis (float products, il = 1.0f / leaf as for the key); start cell floor(u), end cell floor(e)
 *   len = sqrt(dx*dx + dy*dy + dz*dz) with d = (double)w - (double)o, sums left to right; lim = fmin(max_range, len - end_margin)
 *   inv_a = 1.0 / ((double)e_a - (double)u_a); next face of axis a from cell c: ((double)c + (step_a > 0 ? 1.0 : 0.0) -
 *   (double)u_a) * inv_a, step_a = +-1 towards the end cell.  All in double, no FP contraction.
 *   The walk takes exactly |di| + |dj| + |dk| steps (ending on floor(e), whatever the rounding); each step moves one cell
 *   along the axis with steps left whose next face is smallest, ties to x, then y, then z.  A cell's entry parameter t is 0
 *   for the start cell, else the face value of the step that entered it.
 *   A visited cell is passed when it is not floor(e) and t * len < lim (strict).
 * malio_world_voxel_evidence_device: the (hit, miss) pairs (n x 2 u32) in the centroid order of malio_world_voxel_download_device,
 * with its size protocol and device-memory contract (8-byte alignment).  Zeros for a map that was never carved.
 * Keep rule: a voxel is dropped when miss >= min_miss and (double)miss > (double)max_miss_per_hit * (double)hit; every other
 * voxel is kept.  malio_world_voxel_download_kept_device gives the kept centroids in the same order, the bits the unfiltered
 * download gives for them, with the same size protocol (*n_out = the kept count) and device-memory contract, except that it
 * waits for the kept count before it enqueues the copy-out.  malio_world_voxel_save_pcd_kept writes them through
 * malio_world_voxel_save_pcd's writer; MALIO_ERR_STATE (nothing written) on an empty map or when the rule keeps no voxel;
 * clear != 0 empties the map as that call does and resets the counters (either save's clear resets them).
 * Refusals, each before anything changes (centroids, counters and entry count stay as they were):
 *   MALIO_ERR_INVALID_ARG  NULL h, s, slot_tag, a or k; max_range not finite and > 0; end_margin not finite and >= 0;
 *                          max_miss_per_hit not finite and >= 0; the leaf errors of malio_world_voxel_accumulate
 *   MALIO_ERR_CAPACITY     (double)max_range * il above MALIO_CARVE_MAX_RANGE_CELLS (a ray visits at most about three times that
 *                          many cells before it stops being passed); an end or an origin (of a slot with points) whose voxel
 *                          index falls outside int
 * With a communicator attached every rank carves what it holds, as malio_world_voxel_accumulate folds it.
 * Device memory: 12 B per entry (hit, miss and the last scan that counted the entry), allocated by the first carve call, grown
 * with the entries; 0 for a map that is never carved.  malio_world_voxel_info's device_bytes includes it.  The kept download
 * and save use the sort area of a download (32 B per voxel) and no more. */
#define MALIO_CARVE_MAX_RANGE_CELLS 65536.0
typedef struct malio_carve_args {
  float max_range;   /* m, finite, > 0: a ray is followed at most this far from its origin */
  float end_margin;  /* m, finite, >= 0: voxels entered within this distance of the ray's end are not passed */
} malio_carve_args;
typedef struct malio_carve_keep {
  uint32_t min_miss;       /* a voxel is dropped only when miss >= min_miss ... */
  float max_miss_per_hit;  /* ... and (double)miss > max_miss_per_hit * (double)hit */
} malio_carve_keep;
int malio_world_voxel_accumulate_carve(malio_handle* h, const malio_pass_state* s, const float* slot_tag, float leaf,
                                       const malio_carve_args* a, uint64_t* n_voxels);
int malio_world_voxel_evidence_device(malio_handle* h, uint32_t* d_hit_miss, uint64_t cap, uint64_t* n_out, void* stream);
int malio_world_voxel_download_kept_device(malio_handle* h, const malio_carve_keep* k, float* d_out, uint64_t cap,
                                           uint64_t* n_out, void* stream);
int malio_world_voxel_save_pcd_kept(malio_handle* h, const char* path, const malio_carve_keep* k, int clear);
/* Keeping a saved map current: seed the voxel map from the saved file (session n's kept map is session n+1's prior), carve it
 * while localizing, and report what changed.  tests/world_seed_ref.py restates every step in numpy.
 * malio_world_voxel_seed folds n > 0 points xyzi (n x 4 floats {x, y, z, intensity}: what malio_read_pcd returns) into an empty
 * map (just created, or after a clearing save: no accumulate since).  The result is exactly the map one
 * malio_world_voxel_accumulate would hold if its dense cloud were these n points in input order, with world bits = the input
 * xyz and intensity = xyzi[4p + 3]: same keys, same float sums point by point, same skipping of non-finite points; the call
 * fixes the leaf.  The seeded voxels are the entries this call creates: entries are numbered in creation order and never
 * renumbered, so the seeded set is the entry range [0, n_seeded), one integer per map, reset by a clearing save.  Each
 * seeded voxel starts at hit = seed_hits, miss = 0 (and no carve scan has counted it); seed_hits > 0 allocates the carve
 * counters of the first carve call here, and that call then leaves them as they are.  Entries a later accumulate creates
 * start at hit = miss = 0, as before.
 * The points are folded in chunks of at most MALIO_SEED_CHUNK, in input order, each through the accumulate pipeline (a stable
 * sort keeps input order inside a chunk), so every voxel's sums still see its points one by one in order and the result does
 * not depend on the chunking; the scan-sized scratch (48 B per point) is bounded by the chunk, not by n.  The entry table is
 * sized for n voxels before the first chunk (at most one per point); the call waits once, at its end, for the voxel count
 * and the verdict.  malio_world_voxel_seed stages the points through a pinned buffer into a chunk-sized device buffer, freed
 * before it returns.  malio_world_voxel_seed_device reads d_xyzi in place with the device-memory contract of the other
 * _device calls (pointer check, 16-byte alignment, ordered on `stream`); it returns after its one wait.  n_voxels may be NULL.
 * Refusals, each before anything changes:
 *   MALIO_ERR_INVALID_ARG  NULL h or xyzi, n == 0, a leaf that is not finite and > 0, device-memory contract (_device)
 *   MALIO_ERR_STATE        the map is not empty (it holds voxels, or an accumulate since creation or the last clearing save
 *                          fixed its leaf)
 *   MALIO_ERR_CAPACITY     a finite point whose voxel index falls outside int, or more than 2^31 - 1 points: the map is empty
 *                          again with its leaf unset, even when earlier chunks had been folded
 * The seed is per handle: with a communicator attached each rank seeds its own map from the points it is given, and nothing
 * is split or exchanged between ranks.
 * malio_world_voxel_changes_device: removed = the seeded voxels the keep rule k drops, added = the voxels not seeded that k
 * keeps, each as centroids in ascending (z, y, x) order with the bits the unfiltered download gives for them (kept = (seeded
 * minus removed) plus added, the two disjoint).  A map that was never seeded gives removed = {} and added = kept; a map that
 * was never carved keeps everything.  The size protocol and contract of malio_world_voxel_download_kept_device per output
 * (NULL / 0 asks the count, *n_removed / *n_added = the full counts, at most cap written, 16-byte alignment), waiting for both
 * counts before it enqueues the copies.  malio_world_voxel_save_changes_pcd writes each set through malio_world_voxel_save_pcd's
 * writer; a NULL path skips its set, an empty set writes no file (not an error); the counts are reported either way (each
 * may be NULL).  The map is not cleared.  MALIO_ERR_STATE on an empty map.  Both use the sort area of a download (32 B per
 * voxel) and no more. */
#define MALIO_SEED_CHUNK (1u << 22)
int malio_world_voxel_seed(malio_handle* h, const float* xyzi, uint64_t n, float leaf, uint32_t seed_hits, uint64_t* n_voxels);
int malio_world_voxel_seed_device(malio_handle* h, const float* d_xyzi, uint64_t n, float leaf, uint32_t seed_hits,
                                  uint64_t* n_voxels, void* stream);
int malio_world_voxel_changes_device(malio_handle* h, const malio_carve_keep* k,
                                     float* d_removed, uint64_t cap_removed, uint64_t* n_removed,
                                     float* d_added, uint64_t cap_added, uint64_t* n_added, void* stream);
int malio_world_voxel_save_changes_pcd(malio_handle* h, const malio_carve_keep* k, const char* removed_path,
                                       const char* added_path, uint64_t* n_removed, uint64_t* n_added);
/* Rebuilding the voxel map from a corrected trajectory: keep the session's dense scans on the device, then fold them again under
 * other states (a pose graph's, a GNSS/INS fusion's, ground truth), another leaf or other carve settings.
 * tests/scan_store_ref.py restates the rebuild as a loop over the accumulate restatements.
 * The scan store (per handle, independent of the voxel map: a clearing save does not touch it) holds per stored scan
 *   points   the dense rows malio_world_accumulate registers: slots 0..L-1 in slot order, each in its buffer order (point 0 and
 *            the untouched points included), as x, y, z in the LiDAR frame with their bits unchanged, 12 B per point.  The points
 *            live in device blocks of MALIO_STORE_BLOCK_POINTS points; a scan never crosses a block, a larger scan gets a block
 *            of its own.  Growing allocates a new block and copies nothing: a failed allocation returns MALIO_ERR_CUDA with the
 *            store unchanged.
 *   record   malio_stored_scan on the host: the caller's time stamp as given, the state, the temporal compensation of the last
 *            malio_upload_scan* (identity before the first), slot_tag and the point count per slot (0 beyond L).
 * malio_scan_store_add stores the current dense cloud with state s: the preconditions and errors of malio_world_accumulate
 * (MALIO_ERR_STATE until malio_undistort* has run on every slot 0..L-1, slot_tag required), MALIO_ERR_CAPACITY above 2^31 - 1
 * points.  The rows are copied device to device on the handle's stream; the call returns after enqueueing (it waits only
 * when it allocates a block) and changes nothing any other call returns.  n_scans (may be NULL) = the stored scans.
 * malio_scan_store_put appends a record and its n x 3 host points (n = the sum of rec->n_points): how a store is loaded back
 * from a file.  MALIO_ERR_INVALID_ARG when n_points is not 0 beyond L or n is above 2^31 - 1.
 * malio_scan_store_get: record k (rec may be NULL) and, with xyz != NULL, its points into xyz (cap points); *n_out = its
 * point count; cap below it returns MALIO_ERR_CAPACITY with nothing read.  MALIO_ERR_INVALID_ARG for k beyond the store.
 * malio_scan_store_register_device: stored scan k registered with s (NULL: its stored state) and its stored temporal
 * compensation, as n x 4 floats {x, y, z, slot_tag}: the bits malio_world_register(.., MALIO_WORLD_DENSE, ..) gave for that
 * scan (rot = identity, pos = 0 gives the scan in the body frame).  The size protocol and device-memory contract of
 * malio_world_register_device (d_out == NULL and cap == 0 asks the size, 16-byte alignment, ordered on `stream`, returns after
 * enqueueing).
 * malio_scan_store_info: stored scans, stored points and the device bytes of the blocks (any may be NULL).
 * malio_scan_store_clear releases every block and record.
 * With a communicator attached each rank stores what it holds, as malio_world_voxel_accumulate folds it.
 *
 * malio_world_voxel_rebuild is the sequence malio_world_voxel_accumulate(_carve)(states[k - first] or, with states == NULL, the
 * stored state; the stored slot_tag; leaf; carve) for k = first .. first + count - 1 in index order, each scan with its stored
 * points and stored temporal compensation.  After it the centroids, the evidence, n_voxels, the leaf and the carve scan count
 * are exactly what that sequence leaves; the entry capacity and device_bytes may differ (the table grows per chunk, not per
 * scan).  It works on any map those calls accept: a cleared map gives a fresh one, a seeded map carved by the corrected
 * session is malio_world_voxel_seed followed by a carved rebuild.  n_seeded is not touched; count == 0 changes nothing.
 * Plain: the rows of whole scans of one block are folded in chunks of at most MALIO_SEED_CHUNK rows (a larger scan alone),
 * one fold per chunk; the stable sort keeps (scan, slot, point) order, so each voxel's sums continue point by point as the
 * per-scan calls continue them.  Carved: one scan at a time (hit and miss are per-scan sets), enqueued back to back.  Either
 * way the call waits once, at its end; growing the table drains the handle's stream first.
 * Refusals, each before anything changes (centroids, counters, entry count and leaf stay as they were):
 *   MALIO_ERR_INVALID_ARG  NULL h; first + count beyond the store; the leaf errors of malio_world_voxel_accumulate; the argument
 *                          errors of malio_world_voxel_accumulate_carve
 *   MALIO_ERR_CAPACITY     the max_range cap; any row's voxel index outside int under its scan's state, or with carve any
 *                          origin of a slot with points.  The one difference from the sequence, which would have folded the
 *                          scans before the faulty one: every row of the range is checked in a key-only pass first.
 * Device memory: the rebuild's scratch is that of one chunk (48 B per row) plus about 1 KB per scan of the range, released
 * before the call returns; a carved rebuild adds 20 B per row of its largest scan. */
#define MALIO_STORE_BLOCK_POINTS (1u << 24)
typedef struct malio_stored_scan {
  double time;                                      /* the caller's stamp, as given */
  malio_pass_state state;                           /* the state it was stored with */
  malio_rigid temporal_comp[MALIO_MAX_LIDAR - 1];   /* LiDAR l >= 1 at l - 1 */
  float slot_tag[MALIO_MAX_LIDAR];
  uint32_t n_points[MALIO_MAX_LIDAR];               /* 0 beyond L */
} malio_stored_scan;
int malio_scan_store_add(malio_handle* h, const malio_pass_state* s, const float* slot_tag, double time, uint64_t* n_scans);
int malio_scan_store_put(malio_handle* h, const malio_stored_scan* rec, const float* xyz, uint64_t* n_scans);
int malio_scan_store_get(malio_handle* h, uint64_t k, malio_stored_scan* rec, float* xyz, uint64_t cap, uint64_t* n_out);
int malio_scan_store_register_device(malio_handle* h, uint64_t k, const malio_pass_state* s, float* d_out, uint64_t cap,
                                     uint64_t* n_out, void* stream);
int malio_scan_store_info(malio_handle* h, uint64_t* n_scans, uint64_t* n_points, uint64_t* device_bytes);
int malio_scan_store_clear(malio_handle* h);
int malio_world_voxel_rebuild(malio_handle* h, uint64_t first, uint64_t count, const malio_pass_state* states, float leaf,
                              const malio_carve_args* carve, uint64_t* n_voxels);
/* Closing loops over the scan store: register a stored scan against a submap of stored scans on the device
 * (malio_scan_store_match), then optimize the odometry chain with the loop edges on the host (malio_pose_graph_optimize); the
 * corrected states go to malio_world_voxel_rebuild.  tests/loop_ref.py restates the match bit for bit.
 * malio_scan_store_match, the contract (every device expression uses only +, -, *, / and sqrt on doubles, plus floor, each sum
 * in the order given; the transcendental functions run on the host):
 *   target rows  for each stored scan k in [target_first, target_first + target_count), in (scan, slot, point) order, the float4
 *                rows malio_scan_store_register_device(k, NULL) gives; a row with a non-finite coordinate is left out.
 *   source rows  stored scan `source` registered with its stored extrinsics and temporal compensation under rot = identity,
 *                pos = 0 (the body frame), as floats b; non-finite rows are left out, n_points counts the others.
 *   model        per level l, leaf = (double)leaf[l]: a target row's key is floor((double)x / leaf) per axis; a key outside
 *                [-2^20, 2^20) refuses the call (MALIO_ERR_CAPACITY).  Per voxel, in row order: n, the sums (one addition at a
 *                time from 0.0), mu = sum / n, then C_ij = sum of d_i * d_j (d = x - mu) in row order, / n.  Cyclic Jacobi with
 *                MALIO_MATCH_JACOBI_SWEEPS sweeps over the pairs (0,1), (0,2), (1,2): a pair with A_pq == 0 is skipped, else
 *                theta = (A_qq - A_pp) / (2 A_pq), t = 1 / (|theta| + sqrt(theta^2 + 1)) negated for theta < 0,
 *                c = 1 / sqrt(t^2 + 1), s = t c; columns p, q of A and V become (c a_p - s a_q, s a_p + c a_q), then rows p, q of
 *                A the same.  The eigenvalues are A's diagonal ordered by (value, index); the normal n is V's column of the
 *                smallest.  The voxel has a plane when n >= min_points and lambda0 <= planarity * lambda1.
 *   pose         (q, p), starting at the guess's rot / pos (NULL: the source's stored state); R = q_to_R(q) on the host.
 *   correspond   w_i = ((R_i0 b0 + R_i1 b1) + R_i2 b2) + p_i; base key floor(w_i / leaf); among the plane voxels of the base
 *                voxel and its 26 neighbours (offsets in (dz, dy, dx) ascending order, keys outside the range skipped) the one
 *                with the smallest e = (d0 d0 + d1 d1) + d2 d2, d = w - mu, the first on ties.  Inlier when e <= leaf * leaf and
 *                |r| <= gate[l], r = (n0 d0 + n1 d1) + n2 d2.
 *   step         per inlier m_i = (R_0i n0 + R_1i n1) + R_2i n2 (R^T n), J = [b x m, m]; the 29 doubles J_i J_j (i <= j,
 *                row-major), J_i r, r r and 1, zero for the other rows, are summed as a perfect binary tree (pairs of adjacent
 *                entries, level by level) over the source index padded with zeros to the smallest power of two >= the source
 *                rows.  The host solves (J^T J) delta = -J^T r by LL^T Cholesky (in index order; a pivot <= 0, or fewer than 6
 *                inliers, ends the level as failed), then q <- normalize(q (x) quat_from_R(R(exp_se3(delta)))),
 *                p <- p + q_rot(q_old, t(exp_se3(delta))).  A level ends after the step whose every |delta_i| is below eps_rot
 *                (i < 3) / eps_pos (i >= 3), after max_iter steps, or on a failure; iterations[l] counts the steps taken.
 *   report       at the final pose, one more evaluation at the finest level: info = J^T J / sigma^2 (symmetric 6 x 6),
 *                rms = sqrt(sum r^2 / inliers) (0 without inliers), fitness = inliers / n_points, eig_min the smallest
 *                eigenvalue of info (host Jacobi, to a tolerance).  rot / pos: the estimate T_est; rel = T_anchor^-1 T_est as
 *                rel_rot = conj(q_anchor) * q_est, rel_pos = q_rot_conj(q_anchor, p_est - p_anchor) with the anchor's stored
 *                state: the loop edge (anchor, source) of malio_pose_graph_optimize, its info the edge's.  converged: the finest
 *                level ended on eps (the coarser levels only bring the pose into its basin and may end on max_iter).
 *                target_voxels[l]: the voxels of level l with a plane.
 * Errors, each leaving the handle as it was:
 *   MALIO_ERR_INVALID_ARG  NULL h, a or rep; source or anchor beyond the store; an empty range or one beyond the store; the
 *                          anchor outside the range; n_levels 0 or above MALIO_MATCH_MAX_LEVELS; a leaf, gate, sigma or
 *                          planarity that is not finite and > 0; max_iter 0; a guess rot / pos that is not finite
 *   MALIO_ERR_STATE        a communicator is attached (each rank stores only its block of a scan)
 *   MALIO_ERR_CAPACITY     a key outside [-2^20, 2^20); 2^31 or more target rows; scratch above MALIO_MATCH_MAX_BYTES
 * The call changes no store record or block, voxel map, device map or prior; of the counters only launches and copies grow.
 * It is synchronous.  Device memory: about 105 B per target row plus 16 B per source row, local to the call and released
 * before it returns; device_bytes reports it. */
#define MALIO_MATCH_MAX_LEVELS 4
#define MALIO_MATCH_JACOBI_SWEEPS 8
#define MALIO_MATCH_KEY_RANGE (1 << 20)
#define MALIO_MATCH_MAX_BYTES (16ull << 30)
typedef struct malio_match_args {
  uint64_t target_first, target_count;   /* the submap: stored scans [first, first + count) under their stored states */
  uint32_t n_levels;                     /* coarse to fine */
  float leaf[MALIO_MATCH_MAX_LEVELS];    /* voxel edge of the plane model per level, metres */
  float gate[MALIO_MATCH_MAX_LEVELS];    /* inlier gate on |residual| per level, metres */
  uint32_t max_iter;                     /* Gauss-Newton steps per level */
  double eps_rot, eps_pos;               /* a level ends when every |dtheta_i| < eps_rot and every |dt_i| < eps_pos */
  uint32_t min_points;                   /* a voxel with fewer target points has no plane */
  double planarity;                      /* plane when lambda0 <= planarity * lambda1 */
  double sigma;                          /* residual standard deviation for the information matrix, metres */
} malio_match_args;
typedef struct malio_match_report {
  double rot[4], pos[3];                 /* the source scan's state in the submap's frame */
  double rel_rot[4], rel_pos[3];         /* the loop edge: T_anchor^-1 * T_source, with T_anchor = the anchor's stored state */
  double info[36];                       /* 6 x 6 information of the edge, order [dtheta, dt] (log_se3's order) */
  double rms, fitness, eig_min;          /* over the inliers; inliers / finite source points; smallest eigenvalue of info */
  uint32_t n_points, n_inliers, iterations[MALIO_MATCH_MAX_LEVELS];
  int32_t converged;                     /* the finest level ended on eps, not on max_iter or a failed step */
  uint64_t target_points, target_voxels[MALIO_MATCH_MAX_LEVELS], device_bytes;
} malio_match_report;
int malio_scan_store_match(malio_handle* h, uint64_t source, uint64_t anchor, const malio_pass_state* guess,
                           const malio_match_args* a, malio_match_report* rep);
/* malio_pose_graph_optimize (host, no handle): node k is (rot, pos) of odo[k], node 0 fixed.  Edges: odometry k -> k + 1 with
 * Z = odo[k]^-1 odo[k + 1] and Omega = diag(sigma_rot^-2 x 3, sigma_pos^-2 x 3); loops[i] with Z = (rot, pos) and Omega = info.
 * Residual e = log_se3(Z^-1 T_a^-1 T_b), the nodes perturbed on the right as malio_scan_store_match's pose
 * (T <- T exp_se3(delta)), Jacobians J_b = I and J_a = -Ad(T_b^-1 T_a) (first order in e).  Gauss-Newton: the exact solve of
 * the normal equations (block-tridiagonal Cholesky of the chain, the loop edges through Woodbury with Omega = S S^T from its
 * eigen-decomposition: the capacitance I + V^T T^-1 V is SPD for a rank-deficient Omega too); the step is halved (at most 20
 * times) while the total chi^2 grows.  The solve ends with converged = 1 when every |delta| is below eps_rot / eps_pos, or when
 * no halving of a later step lowers chi^2 (the Jacobians are first order, so at the minimum their step may point past it).  It
 * ends with converged = 0 after max_iter steps, when a factor is not positive definite, or when no halving of the first step
 * lowers chi^2 (out is then odo's states).  out[k] is odo[k] with rot and pos replaced (the extrinsics copied);
 * with no loop edge out is odo byte for byte.  loop_chi2 (may be NULL): each loop edge's final e^T Omega e.
 *   MALIO_ERR_INVALID_ARG  NULL odo, a, out or rep, n == 0, NULL loops with n_loops > 0, n_loops above the cap; a loop index
 *                          >= n or a == b; a loop info that is not finite or not symmetric; a sigma or eps that is not > 0
 *                          (or not finite); max_iter 0 */
#define MALIO_POSE_GRAPH_MAX_LOOPS 256
typedef struct malio_pose_edge { uint64_t a, b; double rot[4], pos[3]; double info[36]; } malio_pose_edge;
typedef struct malio_pose_graph_args { double sigma_rot, sigma_pos; uint32_t max_iter; double eps_rot, eps_pos; } malio_pose_graph_args;
typedef struct malio_pose_graph_report {
  uint32_t iterations; int32_t converged; double chi2_odo, chi2_loop, chi2_loop_before; double ms;
} malio_pose_graph_report;
int malio_pose_graph_optimize(const malio_pass_state* odo, uint64_t n, const malio_pose_edge* loops, uint32_t n_loops,
                              const malio_pose_graph_args* a, malio_pass_state* out, double* loop_chi2,
                              malio_pose_graph_report* rep);
/* Host: the same PCD file from n > 0 host points (n x 4 floats {x, y, z, intensity}): the header of PCDWriter::writeBinary for
 * PointXYZINormal (FIELDS x y z intensity normal_x normal_y normal_z curvature, WIDTH = POINTS = n, HEIGHT 1, DATA binary) and
 * n packed 32-byte records with normal_x/y/z = curvature = 0.  MALIO_ERR_INVALID_ARG for n == 0, a NULL argument or a file
 * that cannot be opened or written (no file is left behind). */
int malio_write_pcd_binary(const char* path, const float* xyzi, uint64_t n);

/* ---- next to the path (SURVEY.md §8f N4): City dataset .bin scans without ROS -------------------------------------
 * One file = one scan of packed records as the reference's file player reads them (file_player/src/ROSThread.cpp:776-795
 * Livox, :952-967 Ouster), followed by the per-sensor conversion of MA_LIO/src/preprocess.cpp to the time-stamped raw
 * cloud (x, y, z, curvature = time offset in ms) that UndistortPcl / malio_undistort consume.  Host code. */
typedef struct malio_livox_pt {   /* livox_ros_driver::CustomPoint fields the player fills */
  float x, y, z;
  uint8_t reflectivity, tag, line, pad;
  uint32_t offset_time;           /* only 2 bytes per record are stored in the file (ROSThread.cpp:789) */
} malio_livox_pt;
typedef struct malio_ouster_pt {  /* OusterPointXYZIRT */
  float x, y, z, intensity;
  uint16_t ring, pad;
  uint32_t t;
} malio_ouster_pt;
/* out may be NULL to count.  eof_quirk != 0 appends the zero record the player's `while(!file.eof())` loop produces. */
int malio_read_livox_bin(const char* path, malio_livox_pt* out, uint32_t cap, uint32_t* n_out, int eof_quirk);
int malio_read_ouster_bin(const char* path, malio_ouster_pt* out, uint32_t cap, uint32_t* n_out, int eof_quirk);
/* Preprocess::avia_handler (preprocess.cpp:59-110): n_scans = N_SCANS[lidar], point_filter_num, blind as in the YAML */
int malio_preprocess_livox(const malio_livox_pt* pts, uint32_t n, int n_scans, int point_filter_num, double blind, malio_raw_pt* out,
                           float* intensity, uint32_t cap, uint32_t* n_out);
/* Preprocess::oust64_handler (preprocess.cpp:112-152) */
int malio_preprocess_ouster(const malio_ouster_pt* pts, uint32_t n, int point_filter_num, double blind, float time_unit_scale,
                            malio_raw_pt* out, float* intensity, uint32_t cap, uint32_t* n_out);

/* ---- next to the path (SURVEY.md §8f N1): the map as a device-resident point set, kept in step by deltas -------------
 * Instead of flattening the live ikd-Tree and re-uploading ~20 B per node every scan, the device keeps the map's live
 * points in slots {x, y, z, normal_y, id} and receives what the reference's map-maintenance calls change
 * (include/malio_mapsync.hpp has the host side and the reasoning):
 *   malio_map_build          <- KD_TREE::Build(points)                         ikd_Tree.cpp:370-424  (laserMapping.cpp:1007)
 *   malio_map_delete_boxes   <- KD_TREE::Delete_Point_Boxes(boxes)             :648-676              (laserMapping.cpp:223)
 *   malio_map_add_points     <- KD_TREE::Add_Points(points, false)             :478-584              (laserMapping.cpp:444)
 *   malio_map_sync_voxels    <- KD_TREE::Add_Points(points, true) followed by malio::collect_voxel_sync on the tree: the
 *                               content of every touched voxel box replaces the device's                (laserMapping.cpp:443)
 * Boxes are half-open, min <= p < max per axis, exactly Search_by_range's / Delete_by_range's test (:1270,:807).
 * The cell-list index is rebuilt on the device (~70 us at 1M points) by the next malio_measure / malio_knn / malio_map_commit;
 * dead slots are compacted away when they exceed half of the slots.  In this mode the search never walks a tree: every
 * neighbour list and every distance is the reference's, except for exact distance ties, which the reference breaks by
 * traversal order — those queries are counted (malio_counters.knn_tie_queries) and broken by slot index.
 * nn_idx of malio_download_aux / malio_knn are SLOT indices in this mode; malio_map_download gives slot -> id.
 * A map without a live point (built empty, or everything deleted) answers like a snapshot of 0 nodes: every index
 * 0xFFFFFFFF, every distance +inf, nothing selected (MALIO_ERR_NO_EFFECTIVE_POINTS from malio_measure), whatever its history.
 * A later malio_upload_map* call switches the handle back to snapshot mode: malio_map_add_points / _delete_boxes /
 * _sync_voxels / _info / _download then return MALIO_ERR_STATE until the next malio_map_build (malio_map_commit is a no-op).
 * ids == NULL: malio_map_build numbers the points 0..n-1; malio_map_add_points and malio_map_sync_voxels give each point the
 * slot index it is appended at (the number of slots at that moment; a compaction renumbers the slots, not the ids).
 * Pinned by tests/test_gpu_mapops_edges.py against a numpy mirror and a brute-force k-NN (tests/test_mapops_edges_cpu.py).
 * Host arrays are consumed when a call returns.  Per-scan-sized batches (<= 65536 points, <= 16384 boxes) pass through a pinned
 * bounce buffer and the call returns WITHOUT waiting for the device; n_deleted (may be NULL) costs a device round trip when asked. */
int malio_map_build(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids /* may be NULL: 0..n-1 */, uint32_t n);
int malio_map_add_points(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids /* may be NULL */, uint32_t n);
int malio_map_delete_boxes(malio_handle* h, const float* boxes /* nb x {min3, max3} */, uint32_t nb, uint32_t* n_deleted);
int malio_map_sync_voxels(malio_handle* h, const float* boxes, uint32_t nb, const float* xyz, const float* normal_y,
                          const int32_t* ids, uint32_t n_points, uint32_t* n_deleted);
int malio_map_commit(malio_handle* h);
int malio_map_info(malio_handle* h, uint32_t* n_live, uint32_t* n_slots);
/* live points in slot order (test / debug): any of xyz (n x 3), normal_y, ids, slots may be NULL */
int malio_map_download(malio_handle* h, float* xyz, float* normal_y, int32_t* ids, uint32_t* slots, uint32_t cap, uint32_t* n);

/* ---- localization in a saved map: a prior map of any extent on the device and the local-map window over it ------------------
 * The reference reads map_file_path and never uses it (parameters.cpp:24).  These calls give it a use: load the saved map once,
 * then per scan slide the cube lasermap_fov_segment (laserMapping.cpp:171-224) keeps around the sensor over it, and localize
 * against the window without growing the map.  The window IS the device-resident map above (slots + cell-list index): malio_measure,
 * malio_ieskf_update, malio_knn*, malio_map_incremental and the device-memory calls work on it unchanged (slot indices, ties).
 * Without inserts the map is a fixed point set and the live set a pure function of it and the cube, so the device owns it alone.
 *
 * malio_prior_map_load / _load_device: the prior (n x 3 xyz, n normal_y, ids NULL = 0..n-1), sorted by tile on the device (20 B
 * per point, 12 B per occupied tile); it replaces the handle's previous prior and ends the window.  A non-finite point
 * (MALIO_ERR_INVALID_ARG) or a tile index outside +-2^20 tiles (MALIO_ERR_CAPACITY) refuses the load and keeps the previous prior
 * and its window.  n == 0 loads an empty prior.  _load_device follows the stream-order and pointer-check contract of the
 * device-memory entry points (block above malio_knn_device): xyz / normal_y / ids are device memory of the handle's device
 * (NULL where required, misaligned, host, pinned, managed or other-device -> MALIO_ERR_INVALID_ARG before anything is enqueued);
 * the handle's stream waits on an event recorded on `stream` on entry, `stream` waits on an event recorded after the last access
 * to the caller's arrays; n == 0 reads no pointer and enqueues nothing on `stream`.  Like malio_map_build_device the call waits
 * for the device (the key check, the tile count) before it returns.
 *
 * malio_prior_map_window(pos_lid, cube_len, det_range): pos_lid = state.pos + state.rot * ext_t[0] in double (:1056).
 *   First call after a load, or after malio_map_build* / malio_upload_map* ended the window: the cube is
 *     vertex_min = (float)(pos - cube_len / 2.0), vertex_max = (float)(pos + cube_len / 2.0)      (:177-185, BoxPointType floats)
 *   and the device map is rebuilt to hold exactly prior ∩ cube, replacing what it held, as malio_map_build would.
 *   Later calls: the move test, mov_dist and the new cube are :187-219 with the reference's types (dist_to_map_edge float,
 *   MOV_THRESHOLD = 1.5f, mov_dist a float of a double max, float vertices).  On a move, old ∖ new dies through the reference's
 *   cub_needrm slabs (malio_map_delete_boxes, half-open), then prior ∩ (new ∖ old) is appended in slot order and the index is
 *   committed.  Without a move nothing is enqueued and no device work is done.
 *   Invariant: in a run that makes no other map calls, the live set after every call is exactly prior ∩ cube, min <= p < max per
 *   axis.  It holds exactly, not up to rounding: a slab's face and the new cube's face are the same float operation
 *   (new.max = old.max - mov_dist and the slab's min = old.max - mov_dist; likewise on the other side), and old.min - mov_dist
 *   rounds to at most old.min, so what the slabs spare of the old cube lies in the new one.  Points added with
 *   malio_map_add_points* stay live until a slab covers them, as in the reference.
 *   Slot order is deterministic: prior points enter in tile-key order ((z, y, x) tiles), input order within a tile; two runs give
 *   the same slots and so the same tie breaks (knn_tie_queries).
 *   MALIO_ERR_STATE before a load; MALIO_ERR_INVALID_ARG for a non-finite pos_lid, cube_len not finite and > 0 or det_range not
 *   finite and >= 0; MALIO_ERR_CAPACITY when the cell-list index cannot cover the window's live points (as malio_map_build); after
 *   an error the next call builds the window afresh.
 *   rep: initialized / moved on this call, the cube after it, the slabs of this call (half-open), the points they killed, the
 *   points that entered, and the live points after the window's last commit (on a call without a move: as the previous call left
 *   them, points added since included once committed).
 * malio_prior_map_info: points and occupied tiles of the prior, and the device bytes the prior and the window's scratch hold (the
 * device map's slots are the device-resident map's; any output may be NULL).
 * malio_prior_map_clear: releases the prior; the device map keeps its points, malio_prior_map_window returns MALIO_ERR_STATE until
 * the next load. */
typedef struct malio_window_report {
  int32_t initialized, moved;      /* first call on this prior / the cube moved on this call */
  float cube[6];                   /* LocalMap_Points after the call: {min3, max3} */
  uint32_t n_boxes;
  float boxes[3 * 6];              /* cub_needrm of this call, {min3, max3} each */
  uint32_t n_killed, n_entered, n_live;
} malio_window_report;
int malio_prior_map_load(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n);
int malio_prior_map_load_device(malio_handle* h, const float* d_xyz, const float* d_normal_y, const int32_t* d_ids, uint32_t n,
                                void* stream);
int malio_prior_map_window(malio_handle* h, const double pos_lid[3], double cube_len, float det_range, malio_window_report* rep);
int malio_prior_map_info(malio_handle* h, uint64_t* n_points, uint32_t* n_tiles, uint64_t* device_bytes);
int malio_prior_map_clear(malio_handle* h);

/* ---- localization past the prior's edge: the session layer ------------------------------------------------------------------
 * Where the prior has no data a localizing drive would find no planes and lose track.  malio_prior_map_extend takes the place of
 * map_incremental (laserMapping.cpp:398-446) in localization: run it after the IESKF update of a scan, with the state after the
 * update and before any other map call, and it adds the scan's points where the window holds nothing.  What it adds is the
 * session: an append-only store on the device, owned by the prior, that survives window slides.
 *   1. Decision: the classes and world points of malio_map_incremental(s, filter_size_map, ekf_inited = 1), on the device.
 *   2. Admission: each candidate (MALIO_MAP_ADD or MALIO_MAP_ADD_NO_DOWNSAMPLE) has Add_Points(.., true)'s voxel box
 *      (ikd_Tree.cpp:491-497): per axis lo = floor(x / ds) * ds, hi = lo + ds in float, ds = (float)filter_size_map, half-open.
 *      It is admitted when that box holds no live point of the window at the call's start (prior, session or caller-added
 *      points alike; every admission of one call sees the same live set) and the point lies in its own box and in neither
 *      neighbour's along any axis (at sizes that are not powers of two the faces round; such a point could meet another box's
 *      fold).  The prior is never changed: where it has data it is the authority.
 *   3. Fold: the admitted MALIO_MAP_ADD candidates of one box, in caller order, by Add_Points' down-sample rule
 *      (ikd_Tree.cpp:498-534: downsample_size/8, strict <, same_point).  The box was empty and no other box's point lies in it,
 *      so this is Add_Points(admitted ADD, true) on the real tree, exactly.
 *   4. The admitted MALIO_MAP_ADD_NO_DOWNSAMPLE points are added unfolded, as Add_Points(.., false) (laserMapping.cpp:444).
 *   5. Inserted points carry normal_y = 0.001 (feats_down_world's) and id -1 - k, k their session index.  Session order: the
 *      fold winners by ascending caller index, then the admitted no-downsample points by caller index.
 *   6. Every inserted point enters the session; those inside the current cube (min <= p < max) are also appended to the window,
 *      which is then committed.
 * The window's invariant becomes (prior ∪ session) ∩ cube, exactly, after every window and extend call of a run that makes no
 * other map calls.  A window call that builds the window enqueues prior ∩ cube as before, then session ∩ cube in session order;
 * a move appends prior ∩ (new ∖ old), then session ∩ (new ∖ old) in session order.  With an empty session the window does
 * exactly what it did before.  malio_prior_map_load* starts an empty session (a refused load keeps the previous prior and its
 * session), malio_prior_map_clear releases it; malio_map_build* and malio_upload_map* end the window, not the session.
 * Memory: 16 B per session point ({x, y, z, normal_y}; the ids are implied), up to 20 B with the store's growth slack, plus the
 * window's slots of the ones inside the cube.  A slide tests every session point but sizes its scratch by the points that enter.
 * Errors: MALIO_ERR_INVALID_ARG for NULL h or s, filter_size_map not finite and > 0; MALIO_ERR_STATE without a current window
 * (before malio_prior_map_window, or after a map build or upload ended it) or before a pass; MALIO_ERR_CAPACITY when a
 * candidate's voxel index lies outside +-2^20 per axis or is not finite (nothing is added), or past 2^31 - 1 session points.
 * The call always waits for the device once for its counts (and again in the commit when points entered the window); rep may
 * be NULL.  rep: candidates, admitted candidates, inserted points, session points after the call.
 * malio_prior_map_session_download: the session's points, n x {x, y, z, normal_y} in session order (xyzi NULL: only the count);
 * MALIO_ERR_CAPACITY when cap < n, MALIO_ERR_STATE before a load.  Writing prior ∪ session as the next session's prior: load
 * the concatenation of the two (the session ids are -1 - k). */
typedef struct malio_extend_report {
  uint32_t n_candidates;   /* points map_incremental classed MALIO_MAP_ADD or MALIO_MAP_ADD_NO_DOWNSAMPLE */
  uint32_t n_admitted;     /* candidates whose voxel box held no live point at the call's start */
  uint32_t n_inserted;     /* points appended to the session (fold winners + admitted no-downsample points) */
  uint64_t n_session;      /* session points after the call */
} malio_extend_report;
int malio_prior_map_extend(malio_handle* h, const malio_pass_state* s, double filter_size_map, malio_extend_report* rep);
int malio_prior_map_session_download(malio_handle* h, float* xyzi, uint64_t cap, uint64_t* n_out);

/* ---- relocalization in a loaded prior map: the first pose of a drive, from a guess good to tens of metres and no heading ------
 * A caller that starts in a saved map knows roll and pitch (gravity), a rough position (GNSS, the last stop) and nothing of the
 * heading; the IESKF's basin is a few degrees and a few metres.  malio_relocalize closes that gap with an exact search over
 * n_yaw candidate yaws and a lattice of positions around the guess s, keeping its tilt, on the resident scan and the loaded prior.
 *
 * Definitions (tests/reloc_ref.py restates each step):
 *   1. Candidate rotation k = 0 .. n_yaw-1: theta_k = yaw_lo + (double)k * yaw_step, c = cos(theta_k / 2), s_ = sin(theta_k / 2)
 *      (the C library's, double, host), q_k = q_yaw(theta_k) (x) s.rot computed as
 *        w = c*w0 - s_*z0;  x = c*x0 - s_*y0;  y = c*y0 + s_*x0;  z = c*z0 + s_*w0      (host code, no FP contraction)
 *      a yaw about the prior's z axis applied after the guess's rotation.
 *   2. Registered points: every point of the resident scan (caller order, its lidar field, the extrinsics of s, the temporal
 *      compensation of the last upload) as w = body_to_world(s with rot = q_k): the float bits malio_world_register gives for that
 *      state.  A point with a non-finite w is skipped (in neither score nor n_points).
 *   3. Voxels: a point's base voxel is floor((double)w_i / res) per axis; a prior point's voxel floor((double)x_i / res)
 *      (normal_y ignored); a voxel is occupied when any prior point falls in it.
 *   4. score(k, a, b, c) = the finite points whose base voxel shifted by the integer offset (a, b, c) is occupied, a and b in
 *      [-half_xy, half_xy], c in [-half_z, half_z].  The shift is an index shift (a translation by res * (a, b, c) in real
 *      arithmetic) so that no lattice step re-rounds a point.
 *   5. Result: the maximum score over the n_yaw x (2 half_xy + 1)^2 x (2 half_z + 1) candidates; ties go to the smallest k, then
 *      c, then b, then a (signed, ascending).  When no candidate scores above 0 the result is the first candidate
 *      (0, -half_z, -half_xy, -half_xy) with score 0.  rep: rot = q_k, pos[i] = s.pos[i] + (double)offset[i] * res, offset = (a, b, c),
 *      n_points = the finite points under yaw k.
 * Search: exact branch-and-bound (malio_reloc.cu).  Level d of an occupancy pyramid holds G_d[v] = OR of the occupancy over
 * v + [0, 2^d) per axis still split at d; a node (k, d, corner u) is bounded by the sum over the points of G_d[base_k + u], which
 * no leaf under it exceeds, and is pruned when that bound is below max(best, 1) (strict: optimal leaves and ties survive, so
 * the tie-break above is exact).  Search memory is O(levels x chunk) nodes whatever the scene; a scene where every candidate
 * ties (a ground-only prior) takes the exhaustive time in that memory.  rep counts n_candidates, nodes_bounded (nodes whose
 * bound was computed, leaves included) and leaves_scored; both are deterministic.  device_bytes = the call's scratch (per-yaw
 * voxel indices, the pyramid, the node lists), all released before it returns.
 * Errors, each leaving everything as it was:
 *   MALIO_ERR_INVALID_ARG  NULL h, s, a or rep; n_yaw == 0; res not finite and > 0; a non-finite yaw_lo, yaw_step, s.pos or s.rot
 *   MALIO_ERR_STATE        before a malio_prior_map_load*; before a scan upload (or after a call that took the scan's buffers,
 *                          as malio_measure would refuse); with a communicator attached (each rank holds only its block of the scan)
 *   MALIO_ERR_CAPACITY     more than 2^32 candidates; n_yaw x (12 B x scan points + 36 B) above MALIO_RELOC_MAX_INDEX_BYTES; a
 *                          registered point's voxel index with |index| >= 2^30; a pyramid box of 2^31 or more voxels along an axis
 *                          or above MALIO_RELOC_MAX_PYRAMID_BYTES (levels x one bit per voxel of the box the lookups reach: the
 *                          scan's voxel extent + the lattice + the top window, per axis; a +-100 m box at 0.5 m with a 100 m
 *                          scan needs about 0.2 GB)
 * It changes nothing else: the prior, the window and the device map's slots, the resident scan (still measurable) and
 * malio_prior_map_info stay as they were; of malio_counters only kernel_launches, h2d_bytes and d2h_bytes grow.  Synchronous. */
#define MALIO_RELOC_MAX_PYRAMID_BYTES (2ull << 30)
#define MALIO_RELOC_MAX_INDEX_BYTES (4ull << 30)
typedef struct malio_reloc_args {
  double yaw_lo, yaw_step;  /* candidate yaws theta_k = yaw_lo + k * yaw_step (double), k = 0 .. n_yaw-1 */
  uint32_t n_yaw;
  double res;               /* lattice step = voxel edge, metres */
  uint32_t half_xy, half_z; /* offsets a, b in [-half_xy, half_xy], c in [-half_z, half_z] (lattice steps) */
} malio_reloc_args;
typedef struct malio_reloc_report {
  double rot[4], pos[3];    /* the best candidate's state rotation (w,x,y,z) and position */
  int32_t yaw_index, offset[3];
  uint32_t score, n_points; /* scan points in occupied voxels / scan points with finite registered coordinates */
  uint64_t n_candidates, nodes_bounded, leaves_scored;
  uint64_t device_bytes;    /* peak scratch of the call, all released before it returns */
} malio_reloc_report;
int malio_relocalize(malio_handle* h, const malio_pass_state* s, const malio_reloc_args* a, malio_reloc_report* rep);

/* ---- relocalization without a position guess: place descriptors of the prior, each candidate checked by malio_relocalize -------
 * malio_relocalize needs a position good to tens of metres.  Without one (no GNSS fix, a lost track), malio_place_db_build
 * describes every place of the loaded prior once, and malio_relocalize_global ranks them against the resident scan in
 * milliseconds and hands the best few, each in a small box, to malio_relocalize.  Every stage is integer once the heights are
 * binned, so tests/place_ref.py restates each step bit for bit.  All arithmetic below is IEEE double, no FP contraction.
 *
 * 1. Binning table (host, once per build).  Stencil: every integer column offset (ox, oy) != (0, 0) with
 *    x^2 + y^2 < r_max^2, x = ox * cell, y = oy * cell; the sensor's own column is not in it.  Ring: the number of k in
 *    1 .. n_ring-1 with x^2 + y^2 >= rk^2, rk = r_max * k / n_ring (so an offset on a ring boundary goes to the outer ring).
 *    Sector (n_sector % 4 == 0, Q = n_sector / 4): quadrant q = 0 for x > 0, y >= 0; 1 for x <= 0, y > 0; 2 for x < 0, y <= 0;
 *    3 for x >= 0, y < 0.  (u, v) = (x, y), (y, -x), (-x, -y), (-y, x) for q = 0 .. 3 turns the offset into quadrant 0; the sector
 *    is q * Q + the number of j in 1 .. Q-1 with bx_j * v - by_j * u >= 0, where (bx_j, by_j) = (cos phi_j, sin phi_j),
 *    phi_j = 2 pi j / n_sector (the C library's, host), and bx_j = by_j = sqrt(0.5) when 8 j == n_sector.  So an offset on a
 *    sector boundary goes to the counter-clockwise sector, and a quarter-turned offset (-oy, ox) lands exactly Q sectors on.
 *    Bin = ring * n_sector + sector.
 * 2. Level of a column height z_rel (metres above the sensor): 0 (empty) when z_rel < z_lo, else
 *    1 + clamp(floor((z_rel - z_lo) / dz), 0, 14).  A bin's value is the maximum level of its columns, capped per ring at
 *    cap_r = the level of rho_r * tan(fov_up) (rho_r = r_max * ring / n_ring, the ring's inner radius; host tan), never below 1;
 *    no cap when fov_up >= pi/2.  The cap keeps near tall walls comparable between a map and a scan whose beams stop at fov_up.
 *    Occlusion (block_level > 0): in every sector, the bins of the rings beyond the first ring whose value is >= block_level
 *    are set to 0, so that a map, which holds what lies behind a wall and the roof over a building's footprint, compares with a
 *    scan, which does not.  Ring key: per ring, the sum of its bin values after that (rotation-invariant exactly).
 * 3. Database (malio_place_db_build): column (i, j) = (floor((double)x / cell), floor((double)y / cell)) of every prior point;
 *    colmax / colmin = the largest / smallest z (float) of a column's points.  Positions: every occupied column whose i and j are
 *    multiples of m = step / cell, ordered by (j, i) ascending; its sensor sits at ((i + 0.5) cell, (j + 0.5) cell, z_s) with
 *    z_s = (double)colmin + sensor_height (the slot-0 origin's height above ground, from calibration).  Its descriptor takes, for
 *    every stencil offset whose column (i + ox, j + oy) is occupied, z_rel = (double)colmax - z_s.
 * 4. Query (malio_relocalize_global, step 1): every finite point of the resident scan registered as body_to_world with s.pos = 0
 *    (the bits malio_world_register gives), o = the slot-0 origin registered the same way (body point 0 of LiDAR 0);
 *    rel = (double)w - (double)o per axis; column offset floor(rel / cell + 0.5) in x and y (the sensor on a column centre, as a
 *    database position); a column's height is the largest rel z of its points; then the table, levels and caps of the database.
 * 5. Stage 1: d1(p) = sum over rings of |key_q[r] - key_p[r]|; keep the k1 smallest (d1, p).  Stage 2: for those,
 *    d2(p) = min over shifts s of sum_r sum_c |Q[r][c] - D_p[r][(c + s) mod n_sector]|, ties to the smallest s; keep the k2 smallest
 *    (d2, p).  Stage 3: for each kept p in that order, malio_relocalize from the state s with rot = q_yaw(theta) (x) s.rot
 *    (theta = shift * 2 pi / n_sector, malio_relocalize's product and cos / sin) and pos = (x_p, y_p, z_s) - rot * ext_t[0]
 *    (q_rot of step 4, so that the slot-0 origin sits at the position), the yaws of +-1.5 sectors:
 *    n_yaw = 2 * ceil(1.5 * (2 pi / n_sector) / yaw_step) + 1, yaw_lo = -(double)(n_yaw / 2) * yaw_step, and the lattice res,
 *    half_xy, half_z.  The result is the highest verified score, ties to the lower rank; rep holds its pose, score and n_points as
 *    malio_reloc_report does.  With no position (an empty prior) the result is s itself with score 0 and n_candidates 0.
 *
 * malio_place_db_build: replaces any database of the handle (a failed build leaves none).  Device memory: two 4 B column grids
 * over the prior's column bounding box during the build (MALIO_PLACE_MAX_GRID_BYTES), then per position 16 B + n_ring x n_sector
 * / 2 B of nibbles + 2 B per ring key (MALIO_PLACE_MAX_DB_BYTES).  Any later malio_prior_map_load* (refused or not) or
 * malio_prior_map_clear releases the database; malio_prior_map_info does not count it.  Errors: MALIO_ERR_INVALID_ARG (NULL h, a
 * or rep; cell / step / r_max / dz not finite and > 0; step not a positive integer multiple of cell; n_ring == 0; n_sector not a
 * positive multiple of 4; n_ring x n_sector > MALIO_PLACE_MAX_BINS; r_max / cell > MALIO_PLACE_MAX_RADIUS_CELLS; sensor_height or
 * z_lo not finite; fov_up NaN; block_level > 15), MALIO_ERR_STATE (before a prior load), MALIO_ERR_CAPACITY (a column index outside +-2^30, or
 * either byte limit).
 * malio_place_db_download (test / debug): positions in order, any output may be NULL: cols n x 2 (i, j), z_s n, nibbles n x
 * bytes_per_position (bin b in byte b / 2, low nibble for even b), ring_keys n x n_ring.  *n = the count; at most cap written.
 * malio_relocalize_global: MALIO_ERR_INVALID_ARG (NULL h, s, a or rep; k1 == 0 or > MALIO_PLACE_MAX_K1; k2 == 0, > k1 or >
 * MALIO_PLACE_MAX_K2; yaw_step not finite and > 0; a non-finite s.rot; malio_relocalize's argument errors), MALIO_ERR_STATE
 * (before a prior load, before a database build, before a scan upload, a communicator attached), MALIO_ERR_CAPACITY (from
 * malio_relocalize).  It changes nothing else (prior, window, device map, resident scan, database); of malio_counters only
 * kernel_launches, h2d_bytes and d2h_bytes grow.  Synchronous. */
#define MALIO_PLACE_MAX_BINS 4096
#define MALIO_PLACE_MAX_RADIUS_CELLS 256
#define MALIO_PLACE_MAX_K1 1024
#define MALIO_PLACE_MAX_K2 32
#define MALIO_PLACE_MAX_GRID_BYTES (4ull << 30)
#define MALIO_PLACE_MAX_DB_BYTES (8ull << 30)
typedef struct malio_place_args {
  double cell, step, r_max;           /* column edge, lattice step (a multiple of cell), stencil radius: metres (1, 1, 60) */
  uint32_t n_ring, n_sector;          /* 20, 72 */
  double sensor_height;               /* the slot-0 origin's height above the ground, metres */
  double z_lo, dz;                    /* level 1 starts at z_lo (-sensor_height + 0.5: the ground is empty), dz per level (1 m) */
  double fov_up;                      /* the LiDARs' upward field of view, radians; >= pi/2 turns the cap off */
  uint32_t block_level;               /* occlusion: a bin of at least this level hides the rings behind it (2); 0 = off */
} malio_place_args;
typedef struct malio_place_db_report {
  uint64_t n_positions;
  uint32_t grid_nx, grid_ny;          /* column grid over the prior's bounding box */
  uint32_t n_stencil, bytes_per_position;
  uint64_t device_bytes;              /* the database as it stays on the device */
  uint64_t scratch_bytes;             /* peak scratch of the build (grids, flags, scan), released before it returns */
} malio_place_db_report;
typedef struct malio_global_args {
  uint32_t k1, k2;                    /* stage-1 and stage-2 survivors (256, 8) */
  double yaw_step;                    /* verification yaw step, radians (1 degree) */
  double res;                         /* verification lattice step, metres (0.5) */
  uint32_t half_xy, half_z;           /* verification box (ceil(step / (2 res)) + 2, 2) */
} malio_global_args;
typedef struct malio_global_candidate {
  uint32_t position, shift;           /* database index, sector shift */
  uint32_t d1, d2;                    /* ring-key and bin distances */
  int32_t col[2];                     /* the position's column (i, j) */
  double z_s;
  double guess_rot[4], guess_pos[3];  /* the state handed to malio_relocalize */
  double rot[4], pos[3];              /* its result */
  uint32_t score, n_points;
} malio_global_candidate;
typedef struct malio_global_report {
  double rot[4], pos[3];              /* the best verified pose (rot w,x,y,z) */
  uint32_t score, n_points, best_rank;
  uint32_t n_candidates;              /* candidates verified: min(k2, positions) */
  uint32_t n_stage1;                  /* min(k1, positions) */
  malio_reloc_args verify;            /* the malio_relocalize arguments of every candidate */
  malio_global_candidate cand[MALIO_PLACE_MAX_K2];
  uint32_t stage1[MALIO_PLACE_MAX_K1], stage1_d1[MALIO_PLACE_MAX_K1];   /* the stage-1 list in rank order */
  uint8_t query[MALIO_PLACE_MAX_BINS];                                  /* the query's bin values */
  double ms_rank, ms_verify;          /* host clock: query descriptor + stages 1-2; stage 3 */
  uint64_t device_bytes;              /* peak scratch of the call (malio_relocalize's included), released before it returns */
} malio_global_report;
int malio_place_db_build(malio_handle* h, const malio_place_args* a, malio_place_db_report* rep);
int malio_place_db_info(malio_handle* h, uint64_t* n_positions, uint64_t* device_bytes);
int malio_place_db_download(malio_handle* h, int32_t* cols, double* z_s, uint8_t* nibbles, uint16_t* ring_keys, uint64_t cap, uint64_t* n);
int malio_relocalize_global(malio_handle* h, const malio_pass_state* s, const malio_global_args* a, malio_global_report* rep);

/* ---- a 2-D occupancy grid for navigation: ground, obstacle band and free floor per cell ------------------------------------------
 * malio_grid_build_device turns a point set into the raster a navigation stack loads (nav_msgs/OccupancyGrid values as u8;
 * malio_write_grid_pgm writes it in the map_server PGM + YAML format).  The grid is a pure function of the points and the
 * arguments: no ray casting, no session state.  Every step is a min, a count or a flag per cell, so thread order cannot change
 * the result; tests/grid_ref.py restates each step.
 *   1. Points: rows of 4 floats {x, y, z, w}, w ignored.  A row with a non-finite x, y or z is skipped (n_nonfinite).
 *   2. Column of a point: fi = floorf(x * ir), fj = floorf(y * ir), ir = 1.0f / res in float (the voxel map's key rule in 2-D);
 *      the comparisons below are made on these floats.
 *   3. Region: cells i0 <= i < i0 + nx, j0 <= j < j0 + ny, and the ground half-width w (cells).  Only points whose column lies in
 *      the padded region [i0 - w, i0 + nx + w) x [j0 - w, j0 + ny + w) take part (n_used; the others count in n_outside).
 *   4. zmin(c): the smallest z of column c's points, in the order of the order-preserving u32 key of the float (-0.0 < +0.0).
 *   5. ground(c): the minimum of zmin over the (2w+1)^2 columns around c (the same key order); NaN (0x7FC00000) when none of them
 *      holds a point.
 *   6. A point in region cell c with d = z - ground(c) (float32) is a band point when h_lo <= d <= h_hi, a floor point when
 *      d < h_lo, and overhead (ignored: canopies, balconies) when d > h_hi.
 *   7. Cell class: MALIO_GRID_OCCUPIED when the cell holds at least min_obstacle_points band points, else MALIO_GRID_FREE when it
 *      holds a floor point, else MALIO_GRID_UNKNOWN (empty cells, and cells seen only from above).
 * Outputs: d_cls, u8 ny x nx row-major, row r at cell row j0 + r; d_ground (may be NULL), float in the same layout: ground(c)
 * per region cell, an elevation raster.  rep (may be NULL): points used, skipped as non-finite, outside the padded region, cells
 * per class, and device_bytes, the call's peak scratch.
 * Tiling: the pad is exactly w, so the grid of a region equals the same cells cut from the grid of any larger region.  A map
 * too large for one raster is exported in tiles that stitch without seams.
 * Sources (one body):
 *   MALIO_GRID_POINTS     n rows at d_xyzi, device memory of the handle's device, 16-byte aligned (read as float4).
 *   MALIO_GRID_VOXEL_MAP  the handle's voxel map in place: exactly the grid of what malio_world_voxel_download_kept_device(k)
 *                         returns, or with k NULL of what malio_world_voxel_download_device returns (the same centroid bits and
 *                         keep rule; no sort area is used).  d_xyzi and n are ignored.
 *   MALIO_GRID_PRIOR      the loaded prior's points followed by its session layer (malio_prior_map_session_download).
 * malio_grid_build: MALIO_GRID_POINTS with host arrays: xyzi (n x 4), cls and ground (may be NULL) in host memory; the points are
 * staged through a pinned chunk and a device buffer of at most MALIO_GRID_CHUNK rows (read twice), counted in device_bytes with
 * the device copies of the outputs.
 * malio_grid_extent_device: ext = {imin, jmin, imax, jmax}, the column indices of the source's finite points (step 2, with res);
 * {0, 0, -1, -1} when it has none.  The region i0 = imin, nx = imax - imin + 1 (likewise j) is "the whole map".
 * Memory: scratch of 4 (nx + 2w)(ny + 2w) + 4 nx (ny + 2w) + 4 nx ny + 64 bytes (at most 12 B per padded cell: the column minima,
 * the filter's half-way raster, the band count and floor bit per region cell, the report's counters); the caller's outputs are
 * extra.  All scratch is allocated by the call and released before it returns: nothing stays on the handle, and
 * malio_world_voxel_info / malio_prior_map_info report the same bytes before and after.  With a communicator attached each
 * rank grids what its own handle holds; nothing is exchanged.
 * Stream order (the _device calls): the device-memory contract of the other _device calls (block above malio_knn_device); the
 * handle's stream waits on `stream` on entry and `stream` on the handle's after the last access to the caller's arrays; the call
 * waits once, at its end, before its scratch goes back.
 * Errors, each before anything is written:
 *   MALIO_ERR_INVALID_ARG  NULL h, args or d_cls (cls), d_xyzi with n > 0 for MALIO_GRID_POINTS; an unknown source; res not
 *                          finite and > 0; nx or ny == 0; h_lo, h_hi not finite or 0 < h_lo <= h_hi not holding;
 *                          min_obstacle_points == 0; any of i0 - w, i0 + nx + w, j0 - w, j0 + ny + w beyond +-2^24 (exact as a
 *                          float); the device-memory contract (host, managed, other-device or misaligned pointers)
 *   MALIO_ERR_STATE        MALIO_GRID_VOXEL_MAP with an empty voxel map; MALIO_GRID_PRIOR before a malio_prior_map_load*
 *   MALIO_ERR_CAPACITY     scratch above MALIO_GRID_MAX_BYTES (err names the bytes needed); 2^31 or more source rows;
 *                          (extent) a finite point's column index beyond +-2^24
 * malio_write_grid_pgm (host, no handle): cls (ny x nx, as above) as a binary P5 PGM, top row at the largest y, occupied -> 0,
 * free -> 254, unknown -> 205 (map_saver's trinary values), and a YAML beside it: image (the PGM's base name), mode trinary,
 * resolution res, origin [i0 * res, j0 * res, 0.0] (double products, printed to round-trip; the nominal corner of cell (i0, j0):
 * cells are floorf(x * ir), so a point within a rounding of a cell face may lie in the neighbour), negate 0,
 * occupied_thresh 0.65, free_thresh 0.196 (205 decodes as unknown under p = (255 - v) / 255, the ROS 1 and nav2 loaders' rule).
 * MALIO_ERR_INVALID_ARG for a NULL argument, nx or ny == 0, res not finite and > 0, a class value other than 0 / 100 / 255, or a
 * file that cannot be written; neither file is left behind on an error. */
#define MALIO_GRID_POINTS 0
#define MALIO_GRID_VOXEL_MAP 1
#define MALIO_GRID_PRIOR 2
#define MALIO_GRID_FREE 0
#define MALIO_GRID_OCCUPIED 100
#define MALIO_GRID_UNKNOWN 255
#define MALIO_GRID_MAX_BYTES (16ull << 30)
#define MALIO_GRID_MAX_BOUND 16777216
#define MALIO_GRID_CHUNK (1u << 22)
typedef struct malio_grid_args {
  float res;                      /* cell edge, metres */
  int32_t i0, j0;                 /* the region's first cell */
  uint32_t nx, ny;                /* the region's cells along x and y */
  uint32_t ground_halfwidth;      /* w, cells */
  float h_lo, h_hi;               /* the obstacle band above the ground, metres */
  uint32_t min_obstacle_points;   /* band points that make a cell occupied */
} malio_grid_args;
typedef struct malio_grid_report {
  uint64_t n_used, n_nonfinite, n_outside;
  uint64_t n_occupied, n_free, n_unknown;
  uint64_t device_bytes;          /* peak scratch of the call, released before it returns */
} malio_grid_report;
int malio_grid_build_device(malio_handle* h, int source, const float* d_xyzi, uint64_t n, const malio_carve_keep* k,
                            const malio_grid_args* args, uint8_t* d_cls, float* d_ground, void* stream, malio_grid_report* rep);
int malio_grid_build(malio_handle* h, const float* xyzi, uint64_t n, const malio_grid_args* args, uint8_t* cls, float* ground,
                     malio_grid_report* rep);
int malio_grid_extent_device(malio_handle* h, int source, const float* d_xyzi, uint64_t n, const malio_carve_keep* k, float res,
                             int32_t* ext, void* stream);
int malio_write_grid_pgm(const char* pgm_path, const char* yaml_path, const uint8_t* cls, uint32_t nx, uint32_t ny, float res,
                         int32_t i0, int32_t j0);

/* Host: read a binary PCD file as this library (and pcl::PCDWriter::writeBinary) writes it into n x 4 floats {x, y, z, intensity}.
 * x y z must be fields of TYPE F, SIZE 4, COUNT 1; intensity (F 4) is optional (0 without it); every other field of fixed size
 * is skipped.  POINTS must equal WIDTH x HEIGHT and the file must hold POINTS records.  xyzi may be NULL with cap == 0 to ask the
 * size; *n_out = POINTS, and MALIO_ERR_CAPACITY (nothing read) when cap is smaller.  DATA ascii / binary_compressed, a malformed
 * or truncated file, or a file that cannot be opened -> MALIO_ERR_INVALID_ARG. */
int malio_read_pcd(const char* path, float* xyzi, uint64_t cap, uint64_t* n_out);

/* cumulative counters since malio_create: kernels launched by this library, k-NN kernel launches, queries they
 * processed and their summed device time (CUDA events) — what bench.py's roofline is computed from. */
typedef struct malio_counters {
  uint64_t kernel_launches;
  uint64_t knn_launches;
  uint64_t knn_queries;
  double knn_ms;
  uint64_t h2d_bytes, d2h_bytes;
  uint64_t knn_fallback_queries;  /* queries the cell-list fast path handed to the exact ikd-Tree-order traversal */
  uint64_t knn_ring2_queries;     /* queries that needed the 5x5x5 cell block */
  uint64_t knn_candidates;        /* map points the 3x3x3 scans looked at (summed only while timing is enabled) */
  uint64_t pass_launches;         /* measurement passes timed (fused pass kernel, or gate+reduce+fold on the NCCL path) */
  uint64_t pass_points;           /* scan points those passes processed */
  uint64_t pass_fit_launches;     /* ... of which ran the plane fit (search passes) */
  double pass_ms;                 /* their summed device time (CUDA events; only while timing is enabled) */
  uint64_t knn_tie_queries;       /* device-resident map mode: queries with two of the six best distances within PointType_CMP's
                                     1e-10 window, broken by slot index instead of the reference's traversal order (exempted ties) */
  uint64_t map_slots, map_live;   /* device-resident map: slots in use / live points after the last commit */
  uint64_t map_compactions;
  /* multi-GPU, in-kernel exchange: device time (globaltimer) block 0 spent pushing its min/max keys to the peers and waiting for
   * all of theirs (this includes waiting for the slowest rank to LAUNCH its pass), the same for the system sum, and the number
   * of passes that exchanged */
  double exchange_min_wait_ms, exchange_sum_wait_ms;
  uint64_t exchange_passes;
} malio_counters;
int malio_get_counters(malio_handle* h, malio_counters* out);

/* per-pass CUDA-event timing (the ms_* fields of malio_pass_stats and knn_ms of the counters); on by default,
 * costs ~7 event records per pass on the host when enabled. */
int malio_set_timing(malio_handle* h, int enable);

/* stand-alone k-NN (BASELINE config C5, the microbench): queries are world-frame points. */
int malio_knn(malio_handle* h, const float* queries_xyz, uint32_t n_queries,
              uint32_t* nn_idx, float* nn_sqdist, float* ms_device);

/* ---- device-memory entry points: inputs and outputs stay in device memory, the work is ordered on the caller's stream ----------
 * queries / nn_idx / nn_sqdist / xyz / normal_y / ids are device memory of the handle's device (cudaMalloc, cudaMallocAsync or a
 * memory pool, e.g. torch's CUDA tensors).  stream is a cudaStream_t of that device (NULL = the legacy default stream).
 * Results are bit-identical to the host-pointer call on the same inputs: malio_knn_device gives malio_knn's lists (caller order,
 * ascending by (distance, x), 0xFFFFFFFF / +inf where fewer than 5 were found; slot indices in device-resident map mode), with
 * and without sort_queries; malio_map_build_device / _add_points_device give malio_map_build / _add_points' slots, ids (ids ==
 * NULL numbers them as there), commit and compaction.
 * Stream order, no host wait for the call's own work:
 *   - on entry the handle's stream waits on an event recorded on `stream`: everything enqueued there before the call is seen;
 *   - on exit `stream` waits on an event recorded after the last access to the caller's buffers: work enqueued on `stream` after
 *     the call sees the results, and the caller's input buffers may be reused (or freed) once `stream` has passed the call;
 *   - malio_knn_device returns after enqueueing (no cudaStreamSynchronize).  malio_map_build_device still waits, as
 *     malio_map_build does, for the bounding box its commit reads back; malio_map_add_points_device returns after enqueueing.
 *   - a call that must grow the handle's buffers first waits for the handle's earlier work (not for `stream`'s).
 * Arguments checked on the host before anything is enqueued: a NULL, misaligned (not 4-byte), host (pageable or pinned),
 * managed or other-device pointer returns MALIO_ERR_INVALID_ARG.  Managed memory is refused: these calls exist for data already
 * resident in HBM, and a page migration in the middle of a search would make its cost depend on where the pages happen to be;
 * prefetch into plain device memory, or use the host-pointer calls.  n == 0: no pointer is read and nothing is enqueued on
 * `stream` (malio_map_build_device with n == 0 builds an empty map exactly as malio_map_build does).  malio_knn_device before a
 * map exists returns MALIO_ERR_STATE, malio_map_add_points_device before malio_map_build* too.
 * Deferred device-side results — the one behaviour that differs from malio_knn: the traversal fault bit (the stack guard of the
 * exact ikd-Tree-order search, see MALIO_ERR_TREE_TOO_DEEP) and the fallback / ring-2 / tie counters of a malio_knn_device call
 * are only known once the device has run it.  They are copied behind the search and folded in by the NEXT call on the handle,
 * whatever its entry point (malio_get_counters included), which first waits for that copy.  A fault is returned by that next
 * call as MALIO_ERR_TREE_TOO_DEEP instead of running it; the fault stays with its handle as for malio_knn (later searches on the
 * same map report it again, the next malio_upload_map* clears it) and other handles are not affected.  A CUDA error of the
 * enqueued work surfaces the same way, as MALIO_ERR_CUDA of the next call.
 * Shared buffers: like malio_knn, malio_knn_device uses the per-point buffers of the scan path: a malio_measure after it needs a
 * new malio_upload_scan* (MALIO_ERR_STATE otherwise).
 * Counters: knn_launches, knn_queries and kernel_launches grow as for malio_knn; knn_ms is not (reading it would need a host
 * wait) and h2d_bytes / d2h_bytes do not grow. */
int malio_knn_device(malio_handle* h, const float* d_queries, uint32_t n_queries, uint32_t* d_nn_idx, float* d_nn_sqdist,
                     void* stream);
int malio_map_build_device(malio_handle* h, const float* d_xyz, const float* d_normal_y, const int32_t* d_ids, uint32_t n,
                           void* stream);
int malio_map_add_points_device(malio_handle* h, const float* d_xyz, const float* d_normal_y, const int32_t* d_ids, uint32_t n,
                                void* stream);

/* ---- the measurement path on device memory: the scan in, the per-point outputs out, ordered on the caller's stream ----------
 * The same contract as the block above, for malio_upload_scan, malio_download_aux, malio_map_incremental and
 * malio_world_register.  d_* pointers are device memory of the handle's device; table, table_off, temporal_comp, s, slot_tag and
 * n_out stay host memory exactly as in the host calls (the tables are small and built on the host, table_off is read there).
 * Results are bit-identical to the host call on the same inputs (the same kernels write the caller's arrays instead of the
 * library's staging buffers), with and without sort_queries, in snapshot and in device-resident map mode.
 * Stream order as above: the handle's stream waits on an event recorded on `stream` on entry, and `stream` waits on an event
 * recorded after the last access to the caller's buffers on exit.  A call that must grow the handle's buffers first waits for
 * the handle's earlier work (not for `stream`'s); so does a later host call that grows them (malio_upload_scan, malio_undistort,
 * malio_world_register, malio_upload_map*).
 * Checks, in this order: the wrapper's argument checks of the host call (NULL s / n_out / table / table_off, temporal_comp for
 * L > 1, filter_size_map <= 0, source, slot_tag) -> MALIO_ERR_INVALID_ARG; the host call's state errors (MALIO_ERR_STATE before a
 * malio_measure on the current scan, before malio_undistort of every slot for MALIO_WORLD_DENSE); then, when there is a point
 * to read or write, every d_* pointer given: NULL (where the host call needs it), not 4-byte aligned (d_out: not 16-byte
 * aligned, world_kernel stores float4), host (pageable or pinned), managed or other-device memory -> MALIO_ERR_INVALID_ARG.
 * Nothing is enqueued on any error.  n == 0 (no scan point, an empty cloud, cap == 0): no d_* pointer is read and nothing is
 * enqueued on `stream`.
 *
 * malio_upload_scan_from_device: n_pts malio_scan_pt records (16 B: x, y, z, lidar | table_idx << 16) in device memory, 4-byte
 * aligned.  They are copied device-to-device into the handle (about 1 us per 100k points), since the passes of several
 * malio_measure calls read them and the caller may reuse its buffer as soon as `stream` has passed the call.  Like
 * malio_upload_scan it rejects a record with lidar >= n_lidar before it changes anything: a small kernel checks the records
 * where they are and the call WAITS for its verdict, so it returns only after `stream` has reached it (as
 * malio_map_build_device waits for its bounding box).  On such a record it returns MALIO_ERR_INVALID_ARG and the previous scan
 * is still resident and measurable.  Counters: kernel_launches + 1 (the check), h2d_bytes + the table only.
 * malio_download_aux_device: malio_download_aux's outputs in caller order: d_normal_y N floats, d_nn_idx / d_nn_sqdist N x 5,
 * d_selected N bytes, d_world N x 3 floats; any of them may be NULL (skipped).  Returns after enqueueing.
 * malio_map_incremental_device: d_cls N bytes (required), d_world N x 3 floats (may be NULL).  Returns after enqueueing.
 * malio_world_register_device: malio_world_register's protocol: d_out == NULL with cap == 0 asks for the size, *n_out = the
 * full count, at most cap points {x, y, z, intensity} are written to d_out.  With cap >= the count the points are registered
 * straight into d_out, otherwise into the handle's staging buffer followed by a device-to-device copy of the first cap points.
 * Returns after enqueueing.
 * The three output calls add their kernel launches to kernel_launches; d2h_bytes does not grow. */
int malio_upload_scan_from_device(malio_handle* h, const malio_scan_pt* d_pts, uint32_t n_pts, const malio_pose_entry* table,
                                  const uint32_t* table_off, const malio_rigid* temporal_comp, void* stream);
int malio_download_aux_device(malio_handle* h, float* d_normal_y, uint32_t* d_nn_idx, float* d_nn_sqdist, uint8_t* d_selected,
                              float* d_world, void* stream);
int malio_map_incremental_device(malio_handle* h, const malio_pass_state* s, double filter_size_map, int ekf_inited,
                                 uint8_t* d_cls, float* d_world, void* stream);
int malio_world_register_device(malio_handle* h, const malio_pass_state* s, int source, const float* slot_tag, float* d_out,
                                uint32_t cap, uint32_t* n_out, void* stream);

/* ---- the front half of a scan on device memory: raw clouds in, the pose table kept on the device ------------------------------
 * The same contract as the two blocks above, for malio_undistort, malio_voxel_grid, malio_scan_uncertainty and
 * malio_upload_scan_device: with these a scan goes from raw clouds in device memory to the updated state and every per-point
 * output without a point or a table entry crossing the bus.  d_* pointers are plain device memory of the handle's device
 * (a NULL where one is required, a misaligned (not 4-byte), host (pageable or pinned), managed or other-device pointer ->
 * MALIO_ERR_INVALID_ARG before anything is enqueued or the slot is touched); `stream` is the caller's cudaStream_t; the handle's
 * stream waits on an event recorded on `stream` on entry, `stream` waits on an event recorded after the last access to the
 * caller's buffers; with no point to read (n == 0, an empty slot) no d_* pointer is read and nothing is enqueued on `stream`;
 * growing the handle's buffers first waits for the handle's earlier work.  The small host-side inputs (malio_undistort_args with
 * its control points and IMU times, malio_scan_unc_args, leaf) and the scalar outputs (n_pops, n_out, table_off, temporal_comp,
 * n_total) are host memory as in the host calls.  Every kernel is the host call's: results are bit-identical to the host calls
 * on the same inputs.
 *
 * malio_undistort_device: malio_undistort of n raw points (16 B: x, y, z, curvature) read where they are; they are not copied
 * and nothing reads them once `stream` has passed the call.  Outputs (any may be NULL) are device-to-device copies of what the
 * slot holds: d_cloud n x 5 floats {x, y, z, intensity (= idx as float, 0 where untouched), curvature}, the rows
 * malio_voxel_grid* takes as input (there is no separate xyz output); d_idx n; d_ok n bytes; d_pop_point n_cov entries (the first
 * *n_pops are pop points, the rest -1); d_pose n x 7 doubles.  The argument errors are malio_undistort's, in its order, before
 * anything is enqueued.  The time-order check runs on the device (a point whose time is below its predecessor's; a NaN time is
 * accepted exactly where malio_undistort accepts it) and its verdict comes back with the pop count in the call's ONE host wait, at
 * its end, behind the undistortion itself.  So, unlike malio_undistort, which refuses an unordered cloud before it touches the
 * slot, malio_undistort_device returns MALIO_ERR_INVALID_ARG (malio_undistort's message) with the slot left WITHOUT a valid
 * result: malio_voxel_grid*(.., NULL input), malio_scan_uncertainty*, the dense world registration and malio_upload_scan_resident
 * return MALIO_ERR_STATE until the slot is undistorted again, and the outputs given hold unspecified values.  Counters:
 * kernel_launches + malio_undistort's + 1 (the check), h2d_bytes + the control points and IMU times only, d2h_bytes unchanged.
 *
 * malio_voxel_grid_device: malio_voxel_grid with d_in (n x 5 floats; NULL = the slot's undistorted cloud) read where it is and
 * min(*n_out, out_cap) rows copied device-to-device to d_out (may be NULL).  *n_out is the full count.  The call waits, as
 * malio_voxel_grid does, for the grid geometry and for the output count (they size allocations) and returns with the last kernel
 * and the copy enqueued.  The result also stays in the slot for malio_upload_scan_device / _resident.  MALIO_ERR_CAPACITY cases,
 * non-finite points, a cloud without a finite point, n == 0: as malio_voxel_grid, nothing written.
 *
 * malio_scan_uncertainty_resident: malio_scan_uncertainty without the table transfer: the same checks, error codes and kernel,
 * but only the L - 1 temporal compensations come back (table_off L + 1 and temporal_comp L - 1 may be NULL); the table stays on
 * the device and the handle remembers its offsets and the compensations.  malio_scan_uncertainty leaves its table resident too.
 * Counters: h2d_bytes + imu_cov, d2h_bytes + (L - 1) * sizeof(malio_pose).
 * malio_upload_scan_resident: malio_upload_scan_device with the table (copied device-to-device into the scan's own buffer, so
 * the next scan's malio_scan_uncertainty* may run while this scan is measured), offsets and compensations of the last
 * malio_scan_uncertainty*.  MALIO_ERR_STATE when there is none, when a slot was undistorted again since it was built, or when a
 * slot has no down-sampled cloud; MALIO_ERR_INVALID_ARG when a LiDAR's table has fewer than two entries.  h2d_bytes does not
 * grow. */
int malio_undistort_device(malio_handle* h, int lidar, const malio_raw_pt* d_pts, uint32_t n, const malio_undistort_args* a,
                           float* d_cloud, int32_t* d_idx, uint8_t* d_ok, int32_t* d_pop_point, double* d_pose, uint32_t* n_pops,
                           void* stream);
int malio_voxel_grid_device(malio_handle* h, int lidar, const float* d_in, uint32_t n, float leaf, float* d_out, uint32_t out_cap,
                            uint32_t* n_out, void* stream);
int malio_scan_uncertainty_resident(malio_handle* h, const malio_scan_unc_args* a, uint32_t* table_off, malio_pose* temporal_comp);
int malio_upload_scan_resident(malio_handle* h, uint32_t* n_total);

/* ---- host IESKF -----------------------------------------------------------------------------
 * state_ikfom for L LiDARs (use-ikfom.hpp:14-27): DOF n = 17+6L laid out as
 *   pos 0-2 | rot 3-5 | offset_R_l 6+3l | offset_T_l 6+3L+3l | vel | bg | ba | grav (S2, 2 DOF). */
typedef struct malio_state {
  double pos[3];
  double rot[4];                       /* w,x,y,z */
  malio_rigid ext[MALIO_MAX_LIDAR];    /* offset_R_l, offset_T_l */
  double vel[3], bg[3], ba[3];
  double grav[3];                      /* S2, |grav| = 9.809 */
} malio_state;

typedef struct malio_update_report {
  int32_t passes;               /* passes run (<= max_iter+1) */
  int32_t searches;             /* passes that ran the k-NN */
  int32_t converged_count;      /* t in esekfom.hpp:658 */
  int32_t last_status;
  uint32_t n_eff_last;
  float ms_device_total;        /* sum of device time over the passes */
  float ms_host_solve;          /* host 35x35 algebra */
  double dx_last[MALIO_MAX_DOF];  /* last state increment dx_ (esekfom.hpp:642) */
} malio_update_report;

/* esekf::update_iterated_dyn_share_modified (esekfom.hpp:495-721): iterates malio_measure and the host
 * algebra; x and P (n x n row-major) are updated in place.  R is LASER_POINT_COV (laserMapping.cpp:38),
 * only used by the degenerate branch. */
int malio_ieskf_update(malio_handle* h, malio_state* x, double* P, int max_iter, double R,
                       malio_update_report* report);

/* ---- host utility: static snapshot builder --------------------------------------------------
 * Builds a balanced k-d tree over points (median split on the longest axis, as KD_TREE::BuildTree,
 * ikd_Tree.cpp:696-735) directly in snapshot form, for callers without a live ikd-Tree (benchmarks,
 * the k-NN microbench).  order_out[i] = index into xyz of the point stored in node i. */
int malio_build_static_snapshot(const float* xyz, uint32_t n, malio_map_node* nodes_out,
                                uint32_t* order_out, uint32_t* max_depth_out);

#ifdef __cplusplus
}
#endif
#endif /* MALIO_B200_H_ */
