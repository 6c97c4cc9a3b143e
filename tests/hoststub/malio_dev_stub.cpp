// TEST INFRASTRUCTURE ONLY — a stand-in for the CUDA translation units (ma-lio_b200/csrc/malio_*.cu) so that the
// product's HOST code (malio_host.cpp: malio_ieskf_update, the degenerate branch, manifold operators, C-ABI argument
// checks) can be driven on a machine without a GPU: malio_dev::measure / download_rows call back into the test, which
// supplies the reduced system (from the oracle).  Linked only into tests/hoststub/libmalio_hoststub.so, never shipped.
#include <cstring>

#include "malio_internal.h"

extern "C" {
typedef int (*stub_measure_fn)(const malio_pass_state* s, int redo_knn, double* HtRinvH, double* HtRinvh, malio_pass_stats* st);
typedef int (*stub_rows_fn)(double* h_x, double* hvec, uint32_t cap, uint32_t* n_rows);
static stub_measure_fn g_measure = nullptr;
static stub_rows_fn g_rows = nullptr;
void malio_stub_set_callbacks(stub_measure_fn m, stub_rows_fn r) { g_measure = m; g_rows = r; }
}

namespace malio_dev {
int create(malio_handle*) { return MALIO_OK; }
void destroy(malio_handle*) {}
int upload_map(malio_handle*, const malio_map_node*, const float*, uint32_t, uint32_t) { return MALIO_OK; }
int upload_map_compact(malio_handle*, const malio_map_point*, const float*, uint32_t, uint32_t, const float*) { return MALIO_OK; }
int download_map_nodes(malio_handle*, malio_map_node*, uint32_t) { return MALIO_ERR_STATE; }
int upload_scan(malio_handle*, const malio_scan_pt*, uint32_t, const malio_pose_entry*, const uint32_t*, const malio_rigid*) { return MALIO_OK; }
int measure(malio_handle* h, const malio_pass_state* s, int redo_knn, double* HtRinvH, double* HtRinvh, malio_pass_stats* st) {
  if (!g_measure) { h->err = "stub: no measure callback"; return MALIO_ERR_STATE; }
  return g_measure(s, redo_knn, HtRinvH, HtRinvh, st);
}
int download_rows(malio_handle* h, double* h_x, double* hvec, uint32_t cap, uint32_t* n_rows) {
  if (!g_rows) { h->err = "stub: no rows callback"; return MALIO_ERR_STATE; }
  return g_rows(h_x, hvec, cap, n_rows);
}
int download_aux(malio_handle*, float*, uint32_t*, float*, uint8_t*, float*) { return MALIO_ERR_STATE; }
int knn(malio_handle*, const float*, uint32_t, uint32_t*, float*, float*) { return MALIO_ERR_STATE; }
int map_incremental(malio_handle*, const malio_pass_state*, double, int, uint8_t*, float*) { return MALIO_ERR_STATE; }
int rearm_scan(malio_handle*) { return MALIO_OK; }
int get_counters(malio_handle*, malio_counters* out) { std::memset(out, 0, sizeof(*out)); return MALIO_OK; }
int set_timing(malio_handle*, int) { return MALIO_OK; }
int comm_init(malio_handle*, const uint8_t*, int, int) { return MALIO_ERR_NCCL; }
int get_unique_id(uint8_t*) { return MALIO_ERR_NCCL; }
}  // namespace malio_dev

namespace malio_map {
int commit(malio_handle*) { return MALIO_OK; }
int build(malio_handle*, const float*, const float*, const int32_t*, uint32_t) { return MALIO_ERR_STATE; }
int add_points(malio_handle*, const float*, const float*, const int32_t*, uint32_t) { return MALIO_ERR_STATE; }
int delete_boxes(malio_handle*, const float*, uint32_t, uint32_t*) { return MALIO_ERR_STATE; }
int sync_voxels(malio_handle*, const float*, uint32_t, const float*, const float*, const int32_t*, uint32_t, uint32_t*) { return MALIO_ERR_STATE; }
int info(malio_handle*, uint32_t*, uint32_t*) { return MALIO_ERR_STATE; }
int download(malio_handle*, float*, float*, int32_t*, uint32_t*, uint32_t, uint32_t*) { return MALIO_ERR_STATE; }
}  // namespace malio_map

namespace malio_pre {
int undistort(malio_handle*, int, const malio_raw_pt*, uint32_t, const malio_undistort_args*, float*, int32_t*, uint8_t*, int32_t*, uint32_t*, double*) { return MALIO_ERR_STATE; }
int voxel_grid(malio_handle*, int, const float*, uint32_t, float, float*, uint32_t, uint32_t*) { return MALIO_ERR_STATE; }
int upload_scan_device(malio_handle*, const malio_pose_entry*, const uint32_t*, const malio_rigid*, uint32_t*) { return MALIO_ERR_STATE; }
}  // namespace malio_pre

namespace malio_host {
// sym3_singular_values lives in malio_host.cpp (declared in malio_internal.h); nothing to add here
}
