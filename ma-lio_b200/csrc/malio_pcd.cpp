// malio_pcd.cpp — the saved map's file format: pcl::PCDWriter::writeBinary for pcl::PointXYZINormal, the call that writes
// pcl_wait_save every pcd_save_interval scans and at shutdown (laserMapping.cpp:484, :1090).  Host code; the header text and
// the 32-byte record layout live only here, for malio_write_pcd_binary and malio_world_save_pcd alike.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "malio_internal.h"

namespace malio_pcd {

std::string header(uint64_t n) {
  const std::string ns = std::to_string(n);
  return "# .PCD v0.7 - Point Cloud Data file format\n"
         "VERSION 0.7\n"
         "FIELDS x y z intensity normal_x normal_y normal_z curvature\n"
         "SIZE 4 4 4 4 4 4 4 4\n"
         "TYPE F F F F F F F F\n"
         "COUNT 1 1 1 1 1 1 1 1\n"
         "WIDTH " + ns + "\n"
         "HEIGHT 1\n"
         "VIEWPOINT 0 0 0 1 0 0 0\n"
         "POINTS " + ns + "\n"
         "DATA binary\n";
}

int write_binary(const char* path, uint64_t n, const Fetch& fetch, std::string& err) {
  if (!path) { err = "pcd: null path"; return MALIO_ERR_INVALID_ARG; }
  if (n == 0) { err = "pcd: empty cloud (the reference never writes one, laserMapping.cpp:478, :1083)"; return MALIO_ERR_INVALID_ARG; }
  if (n > 0xFFFFFFFFull) { err = "pcd: more than 2^32-1 points (PCL's width is 32-bit)"; return MALIO_ERR_CAPACITY; }
  FILE* f = std::fopen(path, "wb");
  if (!f) { err = std::string("pcd: cannot open ") + path + " for writing"; return MALIO_ERR_INVALID_ARG; }
  const std::string hdr = header(n);
  int rc = std::fwrite(hdr.data(), 1, hdr.size(), f) == hdr.size() ? MALIO_OK : MALIO_ERR_INVALID_ARG;
  if (rc) err = std::string("pcd: write failed on ") + path;
  // PointXYZINormal as PCL stores it: x y z intensity normal_x normal_y normal_z curvature; only xyz and intensity are set by
  // RGBpointBodyToWorld (laserMapping.cpp:149-163), every other field keeps its default 0
  std::vector<float> rec((size_t)CHUNK * 8, 0.f);
  for (uint64_t first = 0; first < n && rc == MALIO_OK; first += CHUNK) {
    const uint64_t cnt = (n - first) < (uint64_t)CHUNK ? (n - first) : (uint64_t)CHUNK;
    const float* xyzi = nullptr;
    if ((rc = fetch(first, cnt, &xyzi)) != MALIO_OK) { err = "pcd: could not fetch the points"; break; }
    for (uint64_t i = 0; i < cnt; ++i) std::memcpy(&rec[8 * i], xyzi + 4 * i, 4 * sizeof(float));
    if (std::fwrite(rec.data(), 32, cnt, f) != cnt) { rc = MALIO_ERR_INVALID_ARG; err = std::string("pcd: write failed on ") + path; }
  }
  if (std::fclose(f) != 0 && rc == MALIO_OK) { rc = MALIO_ERR_INVALID_ARG; err = std::string("pcd: write failed on ") + path; }
  if (rc != MALIO_OK) std::remove(path);   // no partial file
  return rc;
}

}  // namespace malio_pcd

extern "C" int malio_write_pcd_binary(const char* path, const float* xyzi, uint64_t n) {
  if (!path || !xyzi) return MALIO_ERR_INVALID_ARG;
  std::string err;
  return malio_pcd::write_binary(path, n, [xyzi](uint64_t first, uint64_t, const float** out) {
    *out = xyzi + 4 * first;
    return (int)MALIO_OK;
  }, err);
}
