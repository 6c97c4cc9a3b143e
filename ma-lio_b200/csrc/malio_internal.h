// malio_internal.h — shared between the CUDA translation unit and the host C++ of libmalio_b200.so.
#ifndef MALIO_INTERNAL_H_
#define MALIO_INTERNAL_H_

#include <cstdint>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "malio_b200.h"

// Reduced system as the device produces it: fixed, L=3-shaped and padded so that one kernel serves L=1..3.
//   rows  : 24  (Jacobian columns, always at their L=3 positions: 0-5 | 6+3l | 15+3l)
//   cols  : 28  = 24 Jacobian columns | 1 residual column (-> H^T R^-1 h) | 3 "rho*h_0..2" columns
//           (-> the un-weighted 3x3 normal scatter that JacobiSVD's singular values come from)
// Only the 27 upper-triangular 4x4 blocks (row group i <= col group j) are computed and stored.
#define MALIO_RED_ROWS 24
#define MALIO_RED_COLS 28
#define MALIO_RED_BLOCKS 27
#define MALIO_RED_DOUBLES (MALIO_RED_BLOCKS * 16 + 2)   // + n_eff + spare

// The states of a handle, each defined by the CUDA unit named beside it
namespace malio_devstate { struct DeviceState; }   // malio_device.cuh
namespace malio_pre { struct PreState; }           // malio_preproc.cu
namespace malio_map { struct MapOps; }             // malio_mapops.cu
namespace malio_vox { struct VoxState; }           // malio_voxmap.cu
namespace malio_prior { struct PriorState; }       // malio_prior.cu
namespace malio_place { struct PlaceDb; }          // malio_place.cu
namespace malio_store { struct StoreState; }       // malio_store.cu

// The owner of one state of a handle.  malio_host.cpp deletes the handle without seeing the state types, so the owner keeps
// the deleter of the unit that created the state.  Feature states are created by malio_buf::acquire and freed by
// malio_buf::release (malio_buffer.h).
template <class S>
struct malio_owner : std::unique_ptr<S, void (*)(S*)> {
  malio_owner() : std::unique_ptr<S, void (*)(S*)>(nullptr, nullptr) {}
  explicit malio_owner(S* s) : std::unique_ptr<S, void (*)(S*)>(s, [](S* p) { delete p; }) {}
};

struct malio_handle {
  malio_config cfg{};
  std::string err;
  malio_owner<malio_devstate::DeviceState> dev;
  malio_owner<malio_pre::PreState> pre;      // undistortion, voxel grid, world registration
  malio_owner<malio_map::MapOps> mapst;      // the device-resident map
  malio_owner<malio_vox::VoxState> voxmap;   // the saved map as a voxel map
  malio_owner<malio_prior::PriorState> prior;   // localization in a prior map
  malio_owner<malio_place::PlaceDb> place;   // place descriptors of the prior
  malio_owner<malio_store::StoreState> store;   // the session's dense scans, kept for a rebuild of the voxel map
  // counts malio_map::build_from / leave calls: a prior-map window is the device map only while no other call rebuilt or left it
  uint64_t map_epoch = 0;
  // set while a call that returned after enqueueing (malio_knn_device) still has device-side results to hand over: its
  // traversal fault bit and search statistics.  The next entry point on the handle runs it first (MALIO_SETTLE).
  int (*deferred)(malio_handle* h) = nullptr;
};

// first thing every C-ABI entry point that takes a handle does: wait for and fold in what an earlier enqueued call left on
// the device; a fault found there is that call's status, returned instead of running this one
#define MALIO_SETTLE(h)                                              \
  do {                                                               \
    if ((h)->deferred) {                                             \
      if (int settle_rc_ = (h)->deferred(h)) return settle_rc_;      \
    }                                                                \
  } while (0)

// CUDA TU entry points used by the C-ABI wrappers
namespace malio_dev {
int create(malio_handle* h);
void destroy(malio_handle* h);
int upload_map(malio_handle* h, const malio_map_node* nodes, const float* cov, uint32_t n, uint32_t depth);
int upload_map_compact(malio_handle* h, const malio_map_point* pts, const float* cov, uint32_t n, uint32_t depth,
                       const float* root_box);
int download_map_nodes(malio_handle* h, malio_map_node* out, uint32_t cap);
int upload_scan(malio_handle* h, const malio_scan_pt* pts, uint32_t n, const malio_pose_entry* table,
                const uint32_t* table_off, const malio_rigid* tcomp);
int measure(malio_handle* h, const malio_pass_state* s, int redo_knn, double* HtRinvH, double* HtRinvh,
            malio_pass_stats* st);
int download_rows(malio_handle* h, double* h_x, double* hvec, uint32_t cap, uint32_t* n_rows);
int download_aux(malio_handle* h, float* normal_y, uint32_t* nn_idx, float* nn_d2, uint8_t* sel, float* world);
int knn(malio_handle* h, const float* q, uint32_t nq, uint32_t* idx, float* d2, float* ms);
// device-memory queries and lists, ordered on the caller's stream (a cudaStream_t); malio_b200.cu
int knn_device(malio_handle* h, const float* q, uint32_t nq, uint32_t* idx, float* d2, struct CUstream_st* caller);
int map_incremental(malio_handle* h, const malio_pass_state* s, double fs, int ekf_inited, uint8_t* cls, float* world);
int rearm_scan(malio_handle* h);
int grow_slots(malio_handle* h, uint32_t n, uint32_t keep);
int index_from_slots(malio_handle* h, uint32_t n_slots, const float box[6]);
int get_counters(malio_handle* h, malio_counters* out);
int set_timing(malio_handle* h, int enable);
int comm_init(malio_handle* h, const uint8_t* id, int rank, int world);
int get_unique_id(uint8_t* id);
}  // namespace malio_dev

// malio_mapops.cu — the device-resident map (SURVEY.md §8f N1)
namespace malio_map {
int commit(malio_handle* h);   // pending deltas -> compaction (when worth it) + cell-list index; no-op when clean
void leave(malio_handle* h);   // a snapshot upload took the handle: back to snapshot mode, the map_* calls refuse until the next build
int build(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n);
int add_points(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n);
// the same with device arrays read in place, ordered on the caller's stream; pointers checked first (MALIO_ERR_INVALID_ARG)
int build_device(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n, struct CUstream_st* caller);
int add_points_device(malio_handle* h, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t n, struct CUstream_st* caller);
int delete_boxes(malio_handle* h, const float* boxes, uint32_t nb, uint32_t* n_deleted);
int sync_voxels(malio_handle* h, const float* boxes, uint32_t nb, const float* xyz, const float* normal_y, const int32_t* ids, uint32_t m,
                uint32_t* n_deleted);
// the live points of each of nb half-open boxes (device memory, nb x {min3, max3}) into d_counts, enqueued on the handle's
// stream; the index must be committed (MALIO_ERR_STATE otherwise).  Changes nothing.
int count_boxes(malio_handle* h, const float* d_boxes, uint32_t nb, uint32_t* d_counts);
int info(malio_handle* h, uint32_t* n_live, uint32_t* n_slots);
int download(malio_handle* h, float* xyz, float* normal_y, int32_t* ids, uint32_t* slots, uint32_t cap, uint32_t* n);
}  // namespace malio_map

// malio_preproc.cu
namespace malio_pre {
int undistort(malio_handle* h, int lidar, const malio_raw_pt* pts, uint32_t n, const malio_undistort_args* a, float* xyz,
              int32_t* idx, uint8_t* ok, int32_t* pop_point, uint32_t* n_pops, double* pose);
int voxel_grid(malio_handle* h, int lidar, const float* in, uint32_t n, float leaf, float* out, uint32_t out_cap, uint32_t* n_out);
int upload_scan_device(malio_handle* h, const malio_pose_entry* table, const uint32_t* table_off, const malio_rigid* tcomp,
                       uint32_t* n_total);
// the device-resident undistorted clouds of slots 0..L-1 (n x 5 floats each) for malio_voxmap.cu; MALIO_ERR_STATE until every
// slot has been undistorted, as for the dense world registration
int world_dense_source(malio_handle* h, const float* ud[MALIO_MAX_LIDAR], uint32_t n[MALIO_MAX_LIDAR]);
}  // namespace malio_pre

// malio_prior.cu — localization in a prior map
namespace malio_prior {
// the loaded prior's n points as float4 {x, y, z, normal_y} in tile order, device memory of the handle's device, valid until the
// next load or clear (malio_reloc.cu reads them); MALIO_ERR_STATE before a load
int points(const malio_handle* h, const float** xyzw, uint32_t* n);
// the session layer's n points as float4 {x, y, z, normal_y} in session order, valid until the next extend, load or clear
// (malio_grid.cu reads them); MALIO_ERR_STATE before a load
int session(const malio_handle* h, const float** xyzw, uint32_t* n);
}  // namespace malio_prior

// malio_voxmap.cu — the voxel map's entries for malio_grid.cu, in entry order (not key order): n entries of float4 sums and u32
// counts, and their (hit, miss) pairs as uint2, NULL for a map that was never carved.  Device memory of the handle's device,
// valid until the next call that changes the map.  MALIO_ERR_STATE for an empty map.
namespace malio_vox {
struct Entries { const float* sum; const uint32_t* cnt; const uint32_t* hit_miss; uint64_t n; };
int entries(const malio_handle* h, Entries* e);
}  // namespace malio_vox

// malio_store.cu — the stored scans for malio_voxmap.cu's rebuild: scan k's record and its n_points[0] + .. rows of {x, y, z}
// floats in device memory (NULL when it has no point), valid until the next put, add or clear; `block` numbers the device
// block that holds them.  count() is 0 for a handle that never stored a scan.
namespace malio_store {
struct View { const malio_stored_scan* rec; const float* xyz; uint64_t rows; uint32_t block; };
uint64_t count(const malio_handle* h);
View view(const malio_handle* h, uint64_t k);
// the first n rows of stored scan k registered with s (NULL: its stored state) as malio_scan_store_register_device registers
// them, n x 4 floats {x, y, z, slot_tag} into out (16-byte aligned device memory of the handle's device), enqueued on the
// handle's stream
int enqueue_register(malio_handle* h, uint64_t k, const malio_pass_state* s, uint64_t n, float* out);
}  // namespace malio_store

// malio_reloc.cu — relocalization in a loaded prior (malio_relocalize after its NULL checks; malio_place.cu verifies with it)
namespace malio_reloc {
int relocalize(malio_handle* h, const malio_pass_state* s, const malio_reloc_args* a, malio_reloc_report* rep);
}  // namespace malio_reloc

// malio_pcd.cpp — pcl::PCDWriter::writeBinary for PointXYZINormal (host)
namespace malio_pcd {
constexpr uint32_t CHUNK = 1u << 18;   // points per fetch
// fetch(first, count, &xyzi) points *xyzi at count x {x, y, z, intensity} floats of points [first, first + count)
using Fetch = std::function<int(uint64_t first, uint64_t count, const float** xyzi)>;
std::string header(uint64_t n);
// n > 0 points; on any failure the file is removed and a malio_status returned (err says why)
int write_binary(const char* path, uint64_t n, const Fetch& fetch, std::string& err);
}  // namespace malio_pcd

// host math shared by measure() (localization weight) and the IESKF
namespace malio_host {
void sym3_singular_values(const double S[6] /* xx,xy,xz,yy,yz,zz */, double sv[3]);
}

#endif
