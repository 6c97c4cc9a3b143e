// malio_pcd.cpp — the saved map's file format: pcl::PCDWriter::writeBinary for pcl::PointXYZINormal, the call that writes
// pcl_wait_save every pcd_save_interval scans and at shutdown (laserMapping.cpp:484, :1090).  Host code; the header text and
// the 32-byte record layout live only here, for malio_write_pcd_binary and malio_world_save_pcd alike.  malio_read_pcd reads
// such a file back (and the other binary layouts PCL writes) for malio_prior_map_load.  malio_write_grid_pgm writes the 2-D
// occupancy grid (malio_grid.cu) as map_server's PGM + YAML pair.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <sstream>
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

namespace {

// the header of a binary PCD file: field offsets within a record, the record size and the point count
struct PcdLayout {
  long off[4] = {-1, -1, -1, -1};   // x, y, z, intensity: byte offset in the record, -1 when absent
  uint64_t rec = 0, n = 0;
  long data = 0;                     // byte offset of the first record
};

int parse_header(FILE* f, PcdLayout& L, std::string& err) {
  std::vector<std::string> fields, types;
  std::vector<uint64_t> sizes, counts;
  uint64_t width = 0, height = 0, points = 0;
  bool has_w = false, has_h = false, has_p = false;
  char line[4096];
  for (int lines = 0; lines < 64; ++lines) {
    if (!std::fgets(line, sizeof(line), f)) { err = "pcd: header ends before its DATA line"; return MALIO_ERR_INVALID_ARG; }
    std::istringstream ss(line);
    std::string key;
    if (!(ss >> key) || key[0] == '#') continue;
    std::vector<std::string> v;
    for (std::string w; ss >> w;) v.push_back(w);
    auto nums = [&](std::vector<uint64_t>& out) {
      for (const std::string& w : v) {
        if (w.empty() || w.find_first_not_of("0123456789") != std::string::npos || w.size() > 12) return false;
        out.push_back(std::stoull(w));
      }
      return true;
    };
    auto one = [&](uint64_t& out) { std::vector<uint64_t> t; if (v.size() != 1 || !nums(t)) return false; out = t[0]; return true; };
    bool ok = true;
    if (key == "FIELDS") fields = v;
    else if (key == "SIZE") ok = nums(sizes);
    else if (key == "TYPE") types = v;
    else if (key == "COUNT") ok = nums(counts);
    else if (key == "WIDTH") ok = has_w = one(width);
    else if (key == "HEIGHT") ok = has_h = one(height);
    else if (key == "POINTS") ok = has_p = one(points);
    else if (key == "DATA") {
      if (v.size() != 1 || v[0] != "binary") { err = "pcd: DATA " + (v.empty() ? std::string("?") : v[0]) + " (only binary is read)"; return MALIO_ERR_INVALID_ARG; }
      if (fields.empty() || sizes.size() != fields.size() || types.size() != fields.size() || !has_w || !has_h || !has_p) {
        err = "pcd: malformed header (FIELDS / SIZE / TYPE / WIDTH / HEIGHT / POINTS)"; return MALIO_ERR_INVALID_ARG;
      }
      if (counts.empty()) counts.assign(fields.size(), 1);
      if (counts.size() != fields.size()) { err = "pcd: COUNT does not match FIELDS"; return MALIO_ERR_INVALID_ARG; }
      if (width * height != points) { err = "pcd: POINTS differs from WIDTH x HEIGHT"; return MALIO_ERR_INVALID_ARG; }
      static const char* names[4] = {"x", "y", "z", "intensity"};
      for (size_t i = 0; i < fields.size(); ++i) {
        if (sizes[i] == 0 || sizes[i] > 8 || counts[i] == 0 || counts[i] > 1u << 16) { err = "pcd: field " + fields[i] + " has no fixed size"; return MALIO_ERR_INVALID_ARG; }
        for (int k = 0; k < 4; ++k)
          if (fields[i] == names[k]) {
            if (types[i] != "F" || sizes[i] != 4 || counts[i] != 1) { err = "pcd: field " + fields[i] + " must be TYPE F, SIZE 4, COUNT 1"; return MALIO_ERR_INVALID_ARG; }
            L.off[k] = (long)L.rec;
          }
        L.rec += sizes[i] * counts[i];
      }
      if (L.off[0] < 0 || L.off[1] < 0 || L.off[2] < 0) { err = "pcd: fields x y z are required"; return MALIO_ERR_INVALID_ARG; }
      L.n = points;
      L.data = std::ftell(f);
      return MALIO_OK;
    } else if (key != "VERSION" && key != "VIEWPOINT") { err = "pcd: unknown header line " + key; return MALIO_ERR_INVALID_ARG; }
    if (!ok) { err = "pcd: malformed " + key + " line"; return MALIO_ERR_INVALID_ARG; }
  }
  err = "pcd: no DATA line in the first 64 lines";
  return MALIO_ERR_INVALID_ARG;
}

}  // namespace

// The occupancy grid in map_server's format: a binary PGM (map_saver's trinary values, the top row at the largest y) and the
// YAML that names it.  Every value is checked before either file is opened; on any failure both are removed.
extern "C" int malio_write_grid_pgm(const char* pgm_path, const char* yaml_path, const uint8_t* cls, uint32_t nx, uint32_t ny,
                                    float res, int32_t i0, int32_t j0) {
  if (!pgm_path || !yaml_path || !cls || nx == 0 || ny == 0 || !(res > 0.f) || !std::isfinite(res)) return MALIO_ERR_INVALID_ARG;
  const uint64_t cells = (uint64_t)nx * ny;
  for (uint64_t c = 0; c < cells; ++c)
    if (cls[c] != MALIO_GRID_FREE && cls[c] != MALIO_GRID_OCCUPIED && cls[c] != MALIO_GRID_UNKNOWN) return MALIO_ERR_INVALID_ARG;
  int rc = MALIO_OK;
  if (FILE* f = std::fopen(pgm_path, "wb")) {
    const std::string hdr = "P5\n" + std::to_string(nx) + " " + std::to_string(ny) + "\n255\n";
    if (std::fwrite(hdr.data(), 1, hdr.size(), f) != hdr.size()) rc = MALIO_ERR_INVALID_ARG;
    std::vector<uint8_t> row(nx);
    for (uint32_t r = 0; r < ny && rc == MALIO_OK; ++r) {
      const uint8_t* src = cls + (uint64_t)(ny - 1 - r) * nx;   // file row 0 is the region's last cell row (largest y)
      for (uint32_t i = 0; i < nx; ++i)
        row[i] = src[i] == MALIO_GRID_OCCUPIED ? 0 : (src[i] == MALIO_GRID_FREE ? 254 : 205);
      if (std::fwrite(row.data(), 1, nx, f) != nx) rc = MALIO_ERR_INVALID_ARG;
    }
    if (std::fclose(f) != 0) rc = MALIO_ERR_INVALID_ARG;
  } else {
    return MALIO_ERR_INVALID_ARG;
  }
  if (rc == MALIO_OK) {
    const char* slash = std::strrchr(pgm_path, '/');
    char buf[512];
    std::snprintf(buf, sizeof(buf),
                  "resolution: %.9g\norigin: [%.17g, %.17g, 0.0]\nnegate: 0\noccupied_thresh: 0.65\nfree_thresh: 0.196\n",
                  (double)res, (double)i0 * (double)res, (double)j0 * (double)res);
    const std::string yaml = std::string("image: ") + (slash ? slash + 1 : pgm_path) + "\nmode: trinary\n" + buf;
    if (FILE* f = std::fopen(yaml_path, "wb")) {
      if (std::fwrite(yaml.data(), 1, yaml.size(), f) != yaml.size()) rc = MALIO_ERR_INVALID_ARG;
      if (std::fclose(f) != 0) rc = MALIO_ERR_INVALID_ARG;
      if (rc != MALIO_OK) std::remove(yaml_path);
    } else {
      rc = MALIO_ERR_INVALID_ARG;
    }
  }
  if (rc != MALIO_OK) std::remove(pgm_path);
  return rc;
}

extern "C" int malio_read_pcd(const char* path, float* xyzi, uint64_t cap, uint64_t* n_out) {
  if (!path || !n_out || (cap && !xyzi)) return MALIO_ERR_INVALID_ARG;
  FILE* f = std::fopen(path, "rb");
  if (!f) return MALIO_ERR_INVALID_ARG;
  PcdLayout L;
  std::string err;
  int rc = parse_header(f, L, err);
  if (rc == MALIO_OK) {
    std::fseek(f, 0, SEEK_END);
    const long end = std::ftell(f);
    if (end < L.data || (uint64_t)(end - L.data) / L.rec < L.n) rc = MALIO_ERR_INVALID_ARG;   // truncated
  }
  if (rc == MALIO_OK) {
    *n_out = L.n;
    if (xyzi && cap < L.n) rc = MALIO_ERR_CAPACITY;
  }
  if (rc == MALIO_OK && xyzi && L.n) {
    std::fseek(f, L.data, SEEK_SET);
    const uint64_t chunk = 1u << 16;
    std::vector<unsigned char> buf(chunk * L.rec);
    for (uint64_t first = 0; first < L.n && rc == MALIO_OK; first += chunk) {
      const uint64_t cnt = (L.n - first) < chunk ? (L.n - first) : chunk;
      if (std::fread(buf.data(), L.rec, cnt, f) != cnt) { rc = MALIO_ERR_INVALID_ARG; break; }
      for (uint64_t i = 0; i < cnt; ++i) {
        float* o = xyzi + 4 * (first + i);
        for (int k = 0; k < 4; ++k) {
          if (L.off[k] >= 0) std::memcpy(o + k, &buf[i * L.rec + L.off[k]], 4);
          else o[k] = 0.f;
        }
      }
    }
  }
  std::fclose(f);
  return rc;
}
