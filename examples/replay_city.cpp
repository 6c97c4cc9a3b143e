// examples/replay_city.cpp — the MA-LIO measurement side driven from C++ through the C-ABI, without ROS.
//
// What a maintainer wires into laserMapping.cpp (INTEGRATION.md §2, §2b, §2c), as one stand-alone program that compiles against
// the REAL reference tree type (KD_TREE<pcl::PointXYZINormal>, MA_LIO/include/ikd-Tree/ikd_Tree.h):
//
//   per scan:  .bin files  -> malio_read_*_bin + malio_preprocess_*          (file_player/src/ROSThread.cpp, src/preprocess.cpp)
//              raw clouds  -> malio_undistort  -> malio_voxel_grid            (IMU_Processing.hpp:468-508, laserMapping.cpp:968-983)
//              pose tables -> malio_build_pose_unc                            (laserMapping.cpp:1028-1048)
//              merged scan -> malio_upload_scan_device                        (laserMapping.cpp:972-983)
//              filter step -> malio_ieskf_update                              (esekfom.hpp:495-721, laserMapping.cpp:1052)
//              map upkeep  -> ikdtree.Add_Points + malio::collect_voxel_sync + malio_map_sync_voxels / malio_map_add_points
//                                                                             (laserMapping.cpp:398-446)
//
// There is no IMU stream in this example: the spline's control points are a constant pose (no motion inside the scan) and the
// uncertainty lists hold two entries of a small constant covariance, so the numbers it prints are those of a static sensor.
// The point is the call sequence and that it compiles and links against the header, the library and the reference's tree.
// Tests: tests/test_examples_cpu.py runs its --host-only part, tests/test_gpu_more.py the whole program on the GPU.
//
// Build (build() does this through oracle/Makefile when the reference checkout is present; running it needs an H100):
//   g++ -O2 -std=c++14 -fopenmp -pthread -w -Ioracle/pcl_shim -I<reference>/MA_LIO/include/ikd-Tree -Iinclude \
//       examples/replay_city.cpp -Lma-lio_b200/malio_b200 -lmalio_b200 -o oracle/_ref/replay_city
//   ./replay_city ouster.bin avia.bin tele.bin      (no arguments: one synthetic scan per LiDAR)
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "ikd_Tree.cpp"        // the reference's tree, from where it lies (resolved through -I; nothing is copied)
#include "malio_b200.h"
#include "malio_mapsync.hpp"

using PointType = pcl::PointXYZINormal;
using PointVector = KD_TREE<PointType>::PointVector;

#define CHECK(call)                                                                                    \
  do {                                                                                                 \
    const int rc_ = (call);                                                                            \
    if (rc_ != MALIO_OK) { std::fprintf(stderr, "%s -> %d: %s\n", #call, rc_, malio_last_error(g_h)); std::exit(1); } \
  } while (0)

static malio_handle* g_h = nullptr;

// one LiDAR's raw cloud: from a City .bin file, or synthetic (a ground plane and a wall seen from the origin)
static std::vector<malio_raw_pt> load_raw(const char* path, bool ouster, unsigned seed) {
  std::vector<malio_raw_pt> raw;
  if (path) {
    uint32_t n = 0, m = 0;
    if (ouster) {
      CHECK(malio_read_ouster_bin(path, nullptr, 0, &n, 1));
      std::vector<malio_ouster_pt> rec(n);
      CHECK(malio_read_ouster_bin(path, rec.data(), n, &n, 1));
      raw.resize(n);
      std::vector<float> inten(n);
      CHECK(malio_preprocess_ouster(rec.data(), n, /*point_filter_num=*/1, /*blind=*/0.5, /*time_unit_scale=*/1.0e-3f, raw.data(), inten.data(), n, &m));
    } else {
      CHECK(malio_read_livox_bin(path, nullptr, 0, &n, 1));
      std::vector<malio_livox_pt> rec(n);
      CHECK(malio_read_livox_bin(path, rec.data(), n, &n, 1));
      raw.resize(n);
      std::vector<float> inten(n);
      CHECK(malio_preprocess_livox(rec.data(), n, /*n_scans=*/6, 1, 0.5, raw.data(), inten.data(), n, &m));
    }
    raw.resize(m);
    return raw;
  }
  std::mt19937 gen(seed);
  std::uniform_real_distribution<float> u(-1.f, 1.f);
  const int n = ouster ? 60000 : 20000;
  raw.resize(n);
  for (int i = 0; i < n; ++i) {
    const bool wall = (i % 3) == 0;
    raw[i].x = wall ? 12.f + 0.02f * u(gen) : 30.f * u(gen);
    raw[i].y = 30.f * u(gen);
    raw[i].z = wall ? 5.f * (u(gen) + 1.f) : -1.5f + 0.02f * u(gen);
    raw[i].curvature = 100.f * (float)i / (float)n;      // ms from the scan start, ascending as UndistortPcl expects
  }
  return raw;
}

// --host-only: the host-side pieces alone (pose table, spline pose, the reference tree + the delta read-back), no device:
// what tests/test_examples_cpu.py runs without a GPU
static int host_only() {
  const double q_id[4] = {1, 0, 0, 0}, t0[3] = {0, 0, 0}, t1[3] = {0.3, 0.1, -0.05};
  double cov6[36];
  std::memset(cov6, 0, sizeof(cov6));
  for (int k = 0; k < 6; ++k) cov6[7 * k] = 1e-7;
  malio_pose ext[2], tc[1], unc[2][3];
  const malio_pose* up[2] = {unc[0], unc[1]};
  const uint32_t counts[2] = {3, 3};
  malio_pose_initial(&ext[0], t0, q_id, cov6); malio_pose_initial(&ext[1], t1, q_id, cov6); malio_pose_initial(&tc[0], t0, q_id, cov6);
  for (int l = 0; l < 2; ++l) for (int j = 0; j < 3; ++j) malio_pose_initial(&unc[l][j], t0, q_id, cov6);
  malio_pose_entry table[4];
  uint32_t off[3];
  const int n_tab = malio_build_pose_unc(2, ext, tc, up, counts, table, off);
  std::vector<double> ct, cT;
  for (int k = 0; k < 8; ++k) { ct.push_back(0.01 * k); const double I4[16] = {1, 0, 0, 0.1 * k, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; cT.insert(cT.end(), I4, I4 + 16); }
  double q[4], p[3];
  const int ok = malio_bspline_get_pose(ct.data(), cT.data(), 8, 0.035, q, p);
  KD_TREE<PointType>& tree = *new KD_TREE<PointType>(0.5f, 0.6f, 0.5f);
  PointVector pts, add;
  std::mt19937 gen(3);
  std::uniform_real_distribution<float> u(-10.f, 10.f);
  for (int i = 0; i < 20000; ++i) { PointType a; a.x = u(gen); a.y = u(gen); a.z = 0.2f * u(gen); a.normal_y = 0.001f; pts.push_back(a); }
  for (int i = 0; i < 500; ++i) { PointType a; a.x = u(gen); a.y = u(gen); a.z = 0.2f * u(gen); a.normal_y = 0.001f; add.push_back(a); }
  tree.Build(pts);
  tree.Add_Points(add, true);
  malio::VoxelSync sync;
  malio::collect_voxel_sync<KD_TREE<PointType>, BoxPointType>(tree, add, 0.5f, sync, [](const PointType&) { return 0; }, 4);
  std::printf("host-only: table entries %d (offsets %u %u %u), spline ok %d p.x %.6f, tree valid %d, touched voxels %zu, points read back %zu, outside %u\n",
              n_tab, off[0], off[1], off[2], ok, p[0], tree.validnum(), sync.counts.size(), sync.normal_y.size(), sync.outside_own_box);
  return (n_tab == 4 && ok == 1 && sync.counts.size() > 0 && sync.outside_own_box == 0) ? 0 : 3;
}

int main(int argc, char** argv) {
  if (argc > 1 && std::strcmp(argv[1], "--host-only") == 0) return host_only();
  const int L = 3;
  malio_config cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  malio_default_params(&cfg.params, L);
  cfg.device = 0;
  cfg.sort_queries = 1;
  if (malio_create(&g_h, &cfg) != MALIO_OK) { std::fprintf(stderr, "malio_create: %s\n", malio_last_error(nullptr)); return 1; }
  std::printf("%s\n", malio_version());

  // ---- a constant-pose spline over the scan: control points every 10 ms (BsplineSE3.cpp:34) with margin on both sides
  const double t_beg = 1000.0, scan_s = 0.1;
  std::vector<double> ctrl_t, ctrl_T;
  for (int k = -3; k < 14; ++k) {
    ctrl_t.push_back(t_beg + 0.01 * k);
    const double I4[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    ctrl_T.insert(ctrl_T.end(), I4, I4 + 16);
  }
  const double cov_t[2] = {t_beg - 0.004, t_beg + scan_s + 0.01};   // imu_cov time stamps: one before, one after the scan

  // ---- extrinsics (Extrinsic.txt would provide them) and the two-entry uncertainty lists of every LiDAR
  const double q_id[4] = {1, 0, 0, 0};
  const double t_ext[3][3] = {{0, 0, 0}, {0.3, 0.1, -0.05}, {0.3, -0.1, -0.05}};
  double cov6[36];
  std::memset(cov6, 0, sizeof(cov6));
  for (int k = 0; k < 6; ++k) cov6[7 * k] = 1e-7;
  malio_pose extrinsic[3], temporal_comp[2], unc[3][3];
  const malio_pose* unc_ptr[3];
  uint32_t counts[3];
  const double t0[3] = {0, 0, 0};
  for (int l = 0; l < L; ++l) {
    malio_pose_initial(&extrinsic[l], t_ext[l], q_id, cov6);
    for (int j = 0; j < 3; ++j) malio_pose_initial(&unc[l][j], t0, q_id, cov6);
    unc_ptr[l] = unc[l];
    counts[l] = 3;                                      // the last entry of each list is dropped (laserMapping.cpp:1035)
    if (l > 0) malio_pose_initial(&temporal_comp[l - 1], t0, q_id, cov6);
  }
  std::vector<malio_pose_entry> table(6);
  uint32_t table_off[4];
  if (malio_build_pose_unc(L, extrinsic, temporal_comp, unc_ptr, counts, table.data(), table_off) < 0) return 1;
  malio_rigid tcomp[2];
  for (int l = 1; l < L; ++l) { std::memcpy(tcomp[l - 1].q, q_id, sizeof(q_id)); std::memcpy(tcomp[l - 1].t, t0, sizeof(t0)); }

  // ---- N2 + N3 per LiDAR, the clouds stay on the device
  for (int l = 0; l < L; ++l) {
    const std::vector<malio_raw_pt> raw = load_raw(argc > l + 1 ? argv[l + 1] : nullptr, l == 0, 7u + (unsigned)l);
    malio_undistort_args ua;
    std::memset(&ua, 0, sizeof(ua));
    ua.beg_time = t_beg;
    std::memcpy(ua.extrinsic.q, q_id, sizeof(q_id)); std::memcpy(ua.extrinsic.t, t_ext[l], sizeof(t_ext[l]));
    double q_end[4], p_end[3];
    if (!malio_bspline_get_pose(ctrl_t.data(), ctrl_T.data(), (uint32_t)ctrl_t.size(), t_beg + scan_s, q_end, p_end)) return 1;
    std::memcpy(ua.lt_imu_frame.q, q_end, sizeof(q_end)); std::memcpy(ua.lt_imu_frame.t, p_end, sizeof(p_end));
    ua.ctrl_t = ctrl_t.data(); ua.ctrl_T = ctrl_T.data(); ua.n_ctrl = (uint32_t)ctrl_t.size();
    ua.imu_cov_t = cov_t; ua.n_cov = 2; ua.cov_pointer = 1;
    std::vector<int32_t> pops(2);
    uint32_t n_pops = 0, n_down = 0;
    CHECK(malio_undistort(g_h, l, raw.data(), (uint32_t)raw.size(), &ua, nullptr, nullptr, nullptr, pops.data(), &n_pops, nullptr));
    CHECK(malio_voxel_grid(g_h, l, nullptr, 0, /*filter_size_surf=*/0.5f, nullptr, 0, &n_down));
    std::printf("LiDAR %d: %zu raw points -> %u after the voxel grid\n", l, raw.size(), n_down);
  }
  uint32_t n_scan = 0;
  CHECK(malio_upload_scan_device(g_h, table.data(), table_off, tcomp, &n_scan));

  // ---- the map: the reference's own tree on the host, its point set mirrored on the device (INTEGRATION.md §2b)
  // on the heap: the object embeds its rebuild logger (~80 MB), as a global it is in laserMapping.cpp
  KD_TREE<PointType>& ikdtree = *new KD_TREE<PointType>(0.5f, 0.6f, 0.5f);
  PointVector map_pts;
  {
    std::mt19937 gen(1);
    std::uniform_real_distribution<float> u(-1.f, 1.f);
    for (int i = 0; i < 200000; ++i) {       // a ground plane and a wall, the surfaces the synthetic scans see
      PointType p;
      const bool wall = (i % 3) == 0;
      p.x = wall ? 12.f + 0.01f * u(gen) : 30.f * u(gen);
      p.y = 30.f * u(gen);
      p.z = wall ? 5.f * (u(gen) + 1.f) : -1.5f + 0.01f * u(gen);
      p.normal_y = 0.001f;
      map_pts.push_back(p);
    }
  }
  ikdtree.Build(map_pts);
  {
    std::vector<float> xyz(3 * map_pts.size()), ny(map_pts.size());
    for (size_t i = 0; i < map_pts.size(); ++i) { xyz[3 * i] = map_pts[i].x; xyz[3 * i + 1] = map_pts[i].y; xyz[3 * i + 2] = map_pts[i].z; ny[i] = map_pts[i].normal_y; }
    CHECK(malio_map_build(g_h, xyz.data(), ny.data(), nullptr, (uint32_t)map_pts.size()));
  }

  // ---- the filter step (laserMapping.cpp:1052): state and covariance as IMU_init leaves them
  malio_state x;
  std::memset(&x, 0, sizeof(x));
  x.rot[0] = 1.0;
  for (int l = 0; l < L; ++l) { std::memcpy(x.ext[l].q, q_id, sizeof(q_id)); std::memcpy(x.ext[l].t, t_ext[l], sizeof(t_ext[l])); }
  x.grav[2] = -9.809;
  const int n_dof = 17 + 6 * L;
  std::vector<double> P((size_t)n_dof * n_dof, 0.0);
  for (int k = 0; k < n_dof; ++k) P[(size_t)k * n_dof + k] = 1e-4;
  malio_update_report rep;
  std::memset(&rep, 0, sizeof(rep));
  CHECK(malio_ieskf_update(g_h, &x, P.data(), /*NUM_MAX_ITERATIONS=*/3, /*LASER_POINT_COV=*/0.001, &rep));
  std::printf("update: %d passes, %d searches, N_eff %u, device %.3f ms, host solve %.3f ms, pos = (%.4f %.4f %.4f)\n", rep.passes, rep.searches,
              rep.n_eff_last, rep.ms_device_total, rep.ms_host_solve, x.pos[0], x.pos[1], x.pos[2]);

  // ---- map_incremental (laserMapping.cpp:398-446): the decision on the device, the tree calls on the host, the mirror calls after them
  malio_pass_state ps;
  std::memcpy(ps.rot, x.rot, sizeof(ps.rot)); std::memcpy(ps.pos, x.pos, sizeof(ps.pos));
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) ps.ext[l] = x.ext[l < L ? l : 0];
  std::vector<uint8_t> cls(n_scan);
  std::vector<float> world(3 * (size_t)n_scan);
  CHECK(malio_map_incremental(g_h, &ps, /*filter_size_map_min=*/0.5, /*flg_EKF_inited=*/1, cls.data(), world.data()));
  PointVector PointToAdd, PointNoNeedDownsample;
  for (uint32_t i = 0; i < n_scan; ++i) {
    if (cls[i] != MALIO_MAP_ADD && cls[i] != MALIO_MAP_ADD_NO_DOWNSAMPLE) continue;
    PointType p;
    p.x = world[3 * i]; p.y = world[3 * i + 1]; p.z = world[3 * i + 2]; p.normal_y = 0.001f;
    (cls[i] == MALIO_MAP_ADD ? PointToAdd : PointNoNeedDownsample).push_back(p);
  }
  ikdtree.Add_Points(PointToAdd, true);                                   // :443
  malio::VoxelSync sync;
  malio::collect_voxel_sync<KD_TREE<PointType>, BoxPointType>(ikdtree, PointToAdd, 0.5f, sync, [](const PointType&) { return 0; }, /*threads=*/8);
  if (sync.outside_own_box) std::fprintf(stderr, "down-sample size not exactly representable: fall back to a full snapshot this scan\n");
  CHECK(malio_map_sync_voxels(g_h, sync.boxes.data(), (uint32_t)sync.counts.size(), sync.xyz.data(), sync.normal_y.data(), nullptr,
                              (uint32_t)sync.normal_y.size(), nullptr));
  ikdtree.Add_Points(PointNoNeedDownsample, false);                       // :444
  if (!PointNoNeedDownsample.empty()) {
    std::vector<float> xyz(3 * PointNoNeedDownsample.size()), ny(PointNoNeedDownsample.size(), 0.001f);
    for (size_t i = 0; i < PointNoNeedDownsample.size(); ++i) { xyz[3 * i] = PointNoNeedDownsample[i].x; xyz[3 * i + 1] = PointNoNeedDownsample[i].y; xyz[3 * i + 2] = PointNoNeedDownsample[i].z; }
    CHECK(malio_map_add_points(g_h, xyz.data(), ny.data(), nullptr, (uint32_t)PointNoNeedDownsample.size()));
  }
  uint32_t live = 0, slots = 0;
  CHECK(malio_map_info(g_h, &live, &slots));
  std::printf("map: tree holds %d valid points, device %u live points in %u slots; %zu + %zu points added\n", ikdtree.validnum(), live, slots,
              PointToAdd.size(), PointNoNeedDownsample.size());
  malio_destroy(g_h);
  return (int)live == ikdtree.validnum() ? 0 : 2;
}
