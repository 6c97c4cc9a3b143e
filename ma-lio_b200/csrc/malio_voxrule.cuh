// malio_voxrule.cuh — the two per-entry rules of the saved voxel map that more than one unit evaluates on the device:
// malio_voxmap.cu (downloads, saves, changes) and malio_grid.cu (the occupancy grid of the map in place).  One expression
// each, so that a grid of the map and a grid of its download see the same bits.
#ifndef MALIO_VOXRULE_CUH_
#define MALIO_VOXRULE_CUH_

#include <cuda_runtime.h>

#include <cstdint>

namespace malio_voxrule {

// the centroid of an entry: its float sums over its count, component by component (vg_centroid_kernel's arithmetic)
__device__ __forceinline__ float4 centroid(float4 s, uint32_t cnt) {
  const float cf = (float)cnt;
  return make_float4(s.x / cf, s.y / cf, s.z / cf, s.w / cf);
}

// (hit, miss) of entry e; zeros for a map that was never carved (hm NULL)
__device__ __forceinline__ uint2 evidence(const uint2* hm, uint32_t e) { return hm ? hm[e] : make_uint2(0u, 0u); }
// the keep rule (malio_carve_keep): a voxel is dropped when miss >= min_miss and (double)miss > ratio * (double)hit
__device__ __forceinline__ bool dropped(uint2 v, uint32_t min_miss, double ratio) {
  return v.y >= min_miss && (double)v.y > ratio * (double)v.x;
}

}  // namespace malio_voxrule

#endif  // MALIO_VOXRULE_CUH_
