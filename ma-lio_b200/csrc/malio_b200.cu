// malio_b200.cu — sm_90a kernels + device-side state of libmalio_b200.so.
//
// Hot path of MA-LIO's measurement update, H100-native (DESIGN.md has the data layout and rooflines):
//   K1 knn_kernel      KD_TREE::Nearest_Search / Search   (ikd_Tree.cpp:426-461, 1073-1255)
//   K2 fit/tau/gate    h_share_model S1 + esti_plane (once per search) + evalPointUncertainty (once per scan)
//                      (laserMapping.cpp:559-612, 725-743; common_lib.h:144-190; associate_uct.hpp:153-175)
//   K3 reduce_kernel   h_share_model S3-S4 rows fused with esekfom.hpp:622-635 (H^T R^-1 H, H^T R^-1 h)
// Compiled with -fmad=false: every float/double expression below is evaluated with the same IEEE operations,
// in the same order, as the reference's x86-64 build (no FMA, CMakeLists.txt:8) so that k-NN index sets are
// bit-exact and the selection gates do not flip; explicit fma() is used only in the FP64 accumulation of K3.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "malio_internal.h"
#include "malio_device.cuh"


using namespace malio_devstate;
namespace {

// ------------------------------------------------------------------ small device algebra (mirrors Eigen's op order)
__device__ __forceinline__ void cross3(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
// Quaternion * vector as Eigen's _transformVector: v + w*uv + qv x uv, uv = 2 (qv x v); q = (w,x,y,z)
__device__ __forceinline__ void q_rot(const double q[4], const double v[3], double o[3]) {
  const double qv[3] = {q[1], q[2], q[3]};
  double uv[3], c2[3];
  cross3(qv, v, uv);
  uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
  cross3(qv, uv, c2);
  o[0] = v[0] + q[0] * uv[0] + c2[0];
  o[1] = v[1] + q[0] * uv[1] + c2[1];
  o[2] = v[2] + q[0] * uv[2] + c2[2];
}
__device__ __forceinline__ void q_rot_conj(const double q[4], const double v[3], double o[3]) {
  const double qc[4] = {q[0], -q[1], -q[2], -q[3]};
  q_rot(qc, v, o);
}
// toRotationMatrix of the conjugate of q, row-major
__device__ __forceinline__ void q_conj_to_R(const double q[4], double R[9]) {
  const double w = q[0], x = -q[1], y = -q[2], z = -q[3];
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
  R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

__device__ __forceinline__ void mat3_mul(const double R[9], const double v[3], double o[3]) {
  o[0] = fma(R[2], v[2], fma(R[1], v[1], R[0] * v[0]));
  o[1] = fma(R[5], v[2], fma(R[4], v[1], R[3] * v[0]));
  o[2] = fma(R[8], v[2], fma(R[7], v[1], R[6] * v[0]));
}
__device__ __forceinline__ void cross3_fma(const double a[3], const double b[3], double o[3]) {
  o[0] = fma(a[1], b[2], -(a[2] * b[1]));
  o[1] = fma(a[2], b[0], -(a[0] * b[2]));
  o[2] = fma(a[0], b[1], -(a[1] * b[0]));
}
// laserMapping.cpp:569-579: point in its LiDAR frame -> LiDAR-0 body frame b, IMU frame m, world g
__device__ __forceinline__ void transform_point(const PassConst& pc, float px, float py, float pz, int lid,
                                                double b[3], double m[3], double g[3]) {
  b[0] = px; b[1] = py; b[2] = pz;
  if (lid != 0) {
    double a[3], t[3], d[3];
    q_rot(pc.eq[lid], b, a);
    a[0] += pc.et[lid][0]; a[1] += pc.et[lid][1]; a[2] += pc.et[lid][2];
    q_rot(pc.cq[lid], a, t);
    d[0] = (t[0] + pc.ct[lid][0]) - pc.et[0][0];
    d[1] = (t[1] + pc.ct[lid][1]) - pc.et[0][1];
    d[2] = (t[2] + pc.ct[lid][2]) - pc.et[0][2];
    q_rot_conj(pc.eq[0], d, b);
  }
  q_rot(pc.eq[0], b, m);
  m[0] += pc.et[0][0]; m[1] += pc.et[0][1]; m[2] += pc.et[0][2];
  q_rot(pc.rot, m, g);
  g[0] += pc.pos[0]; g[1] += pc.pos[1]; g[2] += pc.pos[2];
}

// Device-side fault word (bit 0: a traversal stack overflowed, i.e. the snapshot is deeper than the max_depth the caller
// declared at upload).  Kernels only ever set bits; measure() / knn() read it back with their results and fail loudly.
__device__ uint32_t g_fault_word = 0;
constexpr uint32_t FAULT_STACK_OVERFLOW = 1u;

// ------------------------------------------------------------------ K1: k-NN over the flattened ikd-Tree snapshot
// calc_box_dist (ikd_Tree.cpp:1702-1720).  For lo <= hi at most one of `p < lo`, `p > hi` fires per axis and
// (p-lo)^2 == (lo-p)^2 exactly, so  t = max(lo-p, p-hi, 0);  m += t*t  (in x,y,z order, adding an exact 0 when
// neither fires) gives the reference's float result bit for bit with fewer, branch-free instructions.
__device__ __forceinline__ float box_dist(float px, float py, float pz, float x0, float x1, float y0, float y1,
                                          float z0, float z1) {
  const float tx = fmaxf(fmaxf(x0 - px, px - x1), 0.0f);
  const float ty = fmaxf(fmaxf(y0 - py, py - y1), 0.0f);
  const float tz = fmaxf(fmaxf(z0 - pz, pz - z1), 0.0f);
  float m = tx * tx;
  m += ty * ty;
  m += tz * tz;
  return m;
}
// PointType_CMP::operator< (ikd_Tree.h:102-108):  fabs(dist - a.dist) < 1e-10 ? point.x < a.point.x : dist < a.dist.
// The reference promotes the float difference to double before comparing with 1e-10; 1e-10f rounds UP
// (1.0000000134e-10), so for a float v:  (double)v < 1e-10  <=>  v < 1e-10f.  Pure-float compare, same truth table.
struct HItem { float d, x; uint32_t i; };
__device__ __forceinline__ bool h_lt(const HItem& a, const HItem& b) {
  return (fabsf(a.d - b.d) < 1e-10f) ? (a.x < b.x) : (a.d < b.d);
}

// MANUAL_HEAP (ikd_Tree.h:111-201) specialised to capacity k = 5 and held in registers: slots h0..h4 with the
// binary-heap shape {0:(1,2), 1:(3,4)}.  Each routine below is MoveDown / FloatUp written out for one heap size,
// comparison for comparison, so the slot contents match the reference's array at every step.
struct Heap5 {
  HItem h0, h1, h2, h3, h4;
  int cnt;
  // push while cnt < 5: heap[cnt] = p; FloatUp(cnt)
  __device__ __forceinline__ void push_fill(const HItem& p) {
    if (cnt == 0) { h0 = p; }
    else if (cnt == 1) { if (h_lt(h0, p)) { h1 = h0; h0 = p; } else h1 = p; }
    else if (cnt == 2) { if (h_lt(h0, p)) { h2 = h0; h0 = p; } else h2 = p; }
    else if (cnt == 3) {
      if (h_lt(h1, p)) { h3 = h1; if (h_lt(h0, p)) { h1 = h0; h0 = p; } else h1 = p; } else h3 = p;
    } else {
      if (h_lt(h1, p)) { h4 = h1; if (h_lt(h0, p)) { h1 = h0; h0 = p; } else h1 = p; } else h4 = p;
    }
    cnt++;
  }
  // pop() at size 5: heap[0] = heap[4]; size = 4; MoveDown(0)
  __device__ __forceinline__ void pop5() {
    const HItem tmp = h4;
    const bool c12 = h_lt(h1, h2);            // l = 1; if (l+1 < 4 && heap[1] < heap[2]) l = 2
    const HItem hl = c12 ? h2 : h1;
    if (h_lt(tmp, hl)) {
      h0 = hl;
      if (c12) { h2 = tmp; }                  // idx = 2, l = 5 >= 4
      else {                                  // idx = 1, l = 3 < 4, l+1 = 4 not < 4
        if (h_lt(tmp, h3)) { h1 = h3; h3 = tmp; } else h1 = tmp;
      }
    } else h0 = tmp;
    cnt = 4;
  }
  // steady state: pop() then push(p) with the heap full
  __device__ __forceinline__ void replace_top(const HItem& p) {
    pop5();
    if (h_lt(h1, p)) { h4 = h1; if (h_lt(h0, p)) { h1 = h0; h0 = p; } else h1 = p; } else h4 = p;   // FloatUp(4)
    cnt = 5;
  }
  __device__ __forceinline__ void pop4() {   // size 4 -> 3
    const HItem tmp = h3;
    const bool c12 = h_lt(h1, h2);            // l+1 = 2 < 3
    const HItem hl = c12 ? h2 : h1;
    if (h_lt(tmp, hl)) { h0 = hl; if (c12) h2 = tmp; else h1 = tmp; }   // next l = 3 or 5, both >= 3
    else h0 = tmp;
    cnt = 3;
  }
  __device__ __forceinline__ void pop3() {   // size 3 -> 2: l = 1 < 2, l+1 = 2 not < 2
    const HItem tmp = h2;
    if (h_lt(tmp, h1)) { h0 = h1; h1 = tmp; } else h0 = tmp;
    cnt = 2;
  }
  __device__ __forceinline__ void pop2() { h0 = h1; cnt = 1; }   // size 2 -> 1: l = 1 not < 1
  __device__ __forceinline__ void pop_any() {
    if (cnt == 5) pop5(); else if (cnt == 4) pop4(); else if (cnt == 3) pop3(); else if (cnt == 2) pop2(); else cnt = 0;
  }
};

// Exact emulation of one Nearest_Search call: KD_TREE::Search's traversal with the MANUAL_HEAP emulated slot
// for slot.  Used for the (rare) queries on which the fast path below saw a tie hazard.
__device__ __noinline__ void knn_exact_query(const float4* __restrict__ nodes, float qx, float qy, float qz,
                                             uint32_t oi[MALIO_K], float od[MALIO_K], int& found_out) {
  Heap5 hp;
  hp.cnt = 0;
  hp.h0 = hp.h1 = hp.h2 = hp.h3 = hp.h4 = HItem{INFINITY, 0.f, 0xFFFFFFFFu};
  uint32_t st_n[MALIO_MAX_TREE_DEPTH];
  float st_d[MALIO_MAX_TREE_DEPTH];
  int sp = 0;
  float top = INFINITY;           // q.top().dist once the heap holds k items; +inf (accept all) before
  uint32_t cur = 0;
  bool go = true;
  while (go) {
    const float4* nd = nodes + 4 * (size_t)cur;
    const float4 a = __ldg(nd), b4 = __ldg(nd + 1), c4 = __ldg(nd + 2), d4 = __ldg(nd + 3);
    const uint32_t link = __float_as_uint(a.w);
    if (!(link & MALIO_LINK_POINT_DELETED)) {
      const float dist = (qx - a.x) * (qx - a.x) + (qy - a.y) * (qy - a.y) + (qz - a.z) * (qz - a.z);
      if (hp.cnt < MALIO_K) {
        hp.push_fill(HItem{dist, a.x, cur});
        if (hp.cnt == MALIO_K) top = hp.h0.d;
      } else if (dist < top) {
        hp.replace_top(HItem{dist, a.x, cur});
        top = hp.h0.d;
      }
    }
    const bool hl = link & MALIO_LINK_HAS_LEFT, hr = link & MALIO_LINK_HAS_RIGHT;
    const float dl = hl ? box_dist(qx, qy, qz, b4.x, b4.y, b4.z, b4.w, c4.x, c4.y) : INFINITY;
    const float dr = hr ? box_dist(qx, qy, qz, c4.z, c4.w, d4.x, d4.y, d4.z, d4.w) : INFINITY;
    const uint32_t li = cur + 1, ri = link & MALIO_LINK_INDEX_MASK;
    const bool left_first = dl <= dr;
    const uint32_t n_near = left_first ? li : ri, n_far = left_first ? ri : li;
    const float d_near = left_first ? dl : dr, d_far = left_first ? dr : dl;
    if (d_far < top) {
      if (sp < MALIO_MAX_TREE_DEPTH) { st_n[sp] = n_far; st_d[sp] = d_far; sp++; }
      else atomicOr(&g_fault_word, FAULT_STACK_OVERFLOW);
    }
    if (d_near < top) { cur = n_near; continue; }
    go = false;
    while (sp > 0) {
      --sp;
      if (st_d[sp] < top) { cur = st_n[sp]; go = true; break; }
    }
  }
  const int found = hp.cnt;
#pragma unroll
  for (int j = MALIO_K - 1; j >= 0; --j) {
    if (j < found) { oi[j] = hp.h0.i; od[j] = hp.h0.d; hp.pop_any(); }
    else { oi[j] = 0xFFFFFFFFu; od[j] = INFINITY; }
  }
  found_out = found;
}

// One query per active lane.  Traversal order and pruning are exactly KD_TREE::Search's (near child first
// when dist_left <= dist_right, strict '<' everywhere, first-visited wins), the far child waits on a
// per-thread stack with its box distance and is re-tested against the then-current k-th distance when popped.
//
// Fast path / exact path.  The reference keeps candidates in a binary max-heap ordered by PointType_CMP.  As long
// as no two candidates held at the same time have |d_a - d_b| < 1e-10 (in particular no equal distances), that
// comparator is the plain order on d, the heap is a priority queue over a strict total order, and its
// observable behaviour (top().dist, what pop() evicts, the ascending output) is that of a sorted list.  The fast
// path keeps the 5 best in registers sorted by d, checks every accepted candidate against the 5 held distances
// for the 1e-10 window, and on a hit re-runs that query through knn_exact_query (slot-for-slot heap emulation).
// Results are therefore the reference's, bit for bit, in every case; hazards are ~1e-6 per query on jittered data.
//
// Only the first `lanes` lanes of every warp carry a query (narrow logical warps for very small N).
//   MODE 0: queries come from the scan (transform with pc), also writes world + the k-NN gate
//   MODE 1: stand-alone queries (world-frame float3), no gate
// Traversal stack: SMEM_STACK = true keeps it in shared memory ([depth][thread] layout, 8 B entries; snapshots up to
// KNN_SMEM_DEPTH-1 levels deep) — the unwinding loop is a chain of dependent stack reads, and in local memory those
// reads fall out of L1 behind the node traffic and cost an L2 round trip each; SMEM_STACK = false is the
// local-memory fallback for deeper trees.
constexpr int KNN_POP_WIDTH = 4;
constexpr int KNN_SMEM_DEPTH = 36;   // entries per thread in shared memory, KNN_POP_WIDTH sentinels included

// The traversal itself, called by every lane in `wmask` (converged); lanes with active == false only take part in
// the per-iteration vote.  Returns the reference's Nearest_Search result for the lane's query in oi/od/found.
template <bool SMEM_STACK>
__device__ __forceinline__ void knn_tree_lane(const float4* __restrict__ nodes, float qx, float qy, float qz, bool active,
                                              unsigned wmask, uint32_t oi[MALIO_K], float od[MALIO_K], int& found) {
  // 5 best so far, ascending; +inf sentinels make the fill phase (q.size() < k) the same code path
  float d0 = INFINITY, d1 = INFINITY, d2 = INFINITY, d3 = INFINITY, d4 = INFINITY;
  uint32_t i0 = 0xFFFFFFFFu, i1 = 0xFFFFFFFFu, i2 = 0xFFFFFFFFu, i3 = 0xFFFFFFFFu, i4 = 0xFFFFFFFFu;
  bool hazard = false;
  __shared__ uint2 s_stack[SMEM_STACK ? KNN_SMEM_DEPTH * KNN_THREADS : 1];
  uint2 l_stack[SMEM_STACK ? 1 : MALIO_MAX_TREE_DEPTH + KNN_POP_WIDTH];
#define ST(k) (SMEM_STACK ? s_stack[(k) * KNN_THREADS + threadIdx.x] : l_stack[(k)])
  // KNN_POP_WIDTH sentinels at the bottom: a sentinel always passes `d < top` and ends the traversal; having as
  // many as the pop width lets the unwinding loop read a full group without a bounds check
#pragma unroll
  for (int k = 0; k < KNN_POP_WIDTH; ++k) ST(k) = make_uint2(0xFFFFFFFFu, __float_as_uint(-1.0f));
  int sp = KNN_POP_WIDTH;
  uint32_t cur = 0;
  bool done = !active;
  // One node visit per iteration for every unfinished lane; the vote at the bottom makes the warp reconverge
  // each iteration (lanes that descend would otherwise run ahead of lanes that are unwinding their stack).
  for (;;) {
    if (!done) {
      const float4* nd = nodes + 4 * (size_t)cur;
      const float4 a = __ldg(nd), b4 = __ldg(nd + 1), c4 = __ldg(nd + 2), e4 = __ldg(nd + 3);
      const uint32_t link = __float_as_uint(a.w);
      // calc_dist (ikd_Tree.cpp:1694-1699)
      const float dist = (qx - a.x) * (qx - a.x) + (qy - a.y) * (qy - a.y) + (qz - a.z) * (qz - a.z);
      // both children's box distances, unconditionally (absent children carry a zero box and are masked below):
      // straight-line code lets the box arithmetic overlap the candidate insertion instead of sitting behind branches
      const float bl = box_dist(qx, qy, qz, b4.x, b4.y, b4.z, b4.w, c4.x, c4.y);
      const float br = box_dist(qx, qy, qz, c4.z, c4.w, e4.x, e4.y, e4.z, e4.w);
      // candidate: accepted iff the point is live and dist < k-th best (d4 == +inf while q.size() < k).
      // Branch-free sorted insertion; with acc == false every select keeps its old value.
      const bool acc = !(link & MALIO_LINK_POINT_DELETED) && (dist < d4);
      hazard |= acc & ((fabsf(dist - d0) < 1e-10f) | (fabsf(dist - d1) < 1e-10f) | (fabsf(dist - d2) < 1e-10f) |
                       (fabsf(dist - d3) < 1e-10f) | (fabsf(dist - d4) < 1e-10f));
      const bool c0 = acc & (dist < d0), c1 = acc & (dist < d1), c2 = acc & (dist < d2), c3 = acc & (dist < d3);
      d4 = acc ? (c3 ? d3 : dist) : d4;   i4 = acc ? (c3 ? i3 : cur) : i4;
      d3 = c3 ? (c2 ? d2 : dist) : d3;    i3 = c3 ? (c2 ? i2 : cur) : i3;
      d2 = c2 ? (c1 ? d1 : dist) : d2;    i2 = c2 ? (c1 ? i1 : cur) : i2;
      d1 = c1 ? (c0 ? d0 : dist) : d1;    i1 = c1 ? (c0 ? i0 : cur) : i1;
      d0 = c0 ? dist : d0;                i0 = c0 ? cur : i0;
      const float dl = (link & MALIO_LINK_HAS_LEFT) ? bl : INFINITY;
      const float dr = (link & MALIO_LINK_HAS_RIGHT) ? br : INFINITY;
      const uint32_t li = cur + 1, ri = link & MALIO_LINK_INDEX_MASK;
      const bool left_first = dl <= dr;
      const uint32_t n_near = left_first ? li : ri, n_far = left_first ? ri : li;
      const float d_near = left_first ? dl : dr, d_far = left_first ? dr : dl;
      // d4 == +inf while fewer than k are held, so `d < d4` also covers `q.size() < k` for present children
      if (d_far < d4) {
        constexpr int LIMIT = SMEM_STACK ? KNN_SMEM_DEPTH : MALIO_MAX_TREE_DEPTH + KNN_POP_WIDTH;
        if (sp < LIMIT) { ST(sp) = make_uint2(n_far, __float_as_uint(d_far)); sp++; }
        else atomicOr(&g_fault_word, FAULT_STACK_OVERFLOW);   // deeper than declared: the result is not trusted, the call fails
      }
      if (d_near < d4) { cur = n_near; }
      else {
        // unwind: the reference re-tests one pending far child per returning recursion level; here the top
        // KNN_POP_WIDTH entries are read together (independent shared-memory loads, one latency) and the first
        // live one from the top is taken — same entry, same order, a quarter of the dependent round trips
        uint2 e;
        for (;;) {
          const uint2 e1 = ST(sp - 1), e2 = ST(sp - 2), e3 = ST(sp - 3), e4 = ST(sp - 4);
          const bool k1 = __uint_as_float(e1.y) < d4, k2 = __uint_as_float(e2.y) < d4, k3 = __uint_as_float(e3.y) < d4,
                     k4 = __uint_as_float(e4.y) < d4;
          if (k1 | k2 | k3 | k4) {
            e = k1 ? e1 : (k2 ? e2 : (k3 ? e3 : e4));
            sp -= k1 ? 1 : (k2 ? 2 : (k3 ? 3 : 4));
            break;
          }
          sp -= 4;
        }
        cur = e.x;
        done = (e.x == 0xFFFFFFFFu);
      }
    }
    if (__all_sync(wmask, done)) break;
  }
#undef ST
  if (!active) { found = 0; return; }
  if (!hazard) {
    oi[0] = i0; oi[1] = i1; oi[2] = i2; oi[3] = i3; oi[4] = i4;
    od[0] = d0; od[1] = d1; od[2] = d2; od[3] = d3; od[4] = d4;
    found = (i0 != 0xFFFFFFFFu) + (i1 != 0xFFFFFFFFu) + (i2 != 0xFFFFFFFFu) + (i3 != 0xFFFFFFFFu) + (i4 != 0xFFFFFFFFu);
  } else {
    knn_exact_query(nodes, qx, qy, qz, oi, od, found);
  }
}

// query of position p: MODE 0 = scan point through the state (also yields the world point), MODE 1 = stand-alone
template <int MODE>
__device__ __forceinline__ void load_query(const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm,
                                           const float* __restrict__ queries, uint32_t p, const PassConst& pc,
                                           float& qx, float& qy, float& qz) {
  if (MODE == 0) {
    const malio_scan_pt pt = pts[perm ? perm[p] : p];
    double b[3], m[3], g[3];
    transform_point(pc, pt.x, pt.y, pt.z, pt.lidar, b, m, g);
    qx = (float)g[0]; qy = (float)g[1]; qz = (float)g[2];
  } else {
    const uint32_t src = perm ? perm[p] : p;
    qx = queries[3 * (size_t)src]; qy = queries[3 * (size_t)src + 1]; qz = queries[3 * (size_t)src + 2];
  }
}

template <int MODE, bool SMEM_STACK>
__global__ void __launch_bounds__(KNN_THREADS)
knn_kernel(const float4* __restrict__ nodes, uint32_t n_nodes, const malio_scan_pt* __restrict__ pts,
           const uint32_t* __restrict__ perm, const float* __restrict__ queries, uint32_t N, int lanes, PassConst pc,
           float max_sqdist, float4* __restrict__ world, uint32_t* __restrict__ nn_idx,
           float* __restrict__ nn_d2, uint8_t* __restrict__ sel) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * KNN_THREADS + threadIdx.x) >> 5;
  const uint32_t p = warp * (uint32_t)lanes + lane;
  const bool valid = ((int)lane < lanes) && (p < N);
  const unsigned wmask = __ballot_sync(0xffffffffu, valid);
  if (!valid) return;
  float qx, qy, qz;
  load_query<MODE>(pts, perm, queries, p, pc, qx, qy, qz);
  if (MODE == 0) world[p] = make_float4(qx, qy, qz, 0.f);
  uint32_t oi[MALIO_K];
  float od[MALIO_K];
  int found = 0;
  if (n_nodes > 0) {
    knn_tree_lane<SMEM_STACK>(nodes, qx, qy, qz, true, wmask, oi, od, found);
  } else {
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) { oi[j] = 0xFFFFFFFFu; od[j] = INFINITY; }
  }
#pragma unroll
  for (int j = 0; j < MALIO_K; ++j) {
    nn_idx[(size_t)j * N + p] = oi[j];
    nn_d2[(size_t)j * N + p] = od[j];
  }
  if (MODE == 0) sel[p] = (found < MALIO_K) ? 0 : (od[MALIO_K - 1] > max_sqdist ? 0 : 1);   // laserMapping.cpp:587
}

// List mode: the same traversal for the positions the cell-list fast path (below) could not settle — tie hazards,
// queries whose 5th neighbour lies beyond the searched cell block, queries outside the grid.  A fixed grid walks
// the list (its length is only known on the device); the world point was already written by the fast path.
template <int MODE, bool SMEM_STACK>
__global__ void __launch_bounds__(KNN_THREADS)
knn_list_kernel(const float4* __restrict__ nodes, uint32_t n_nodes, const malio_scan_pt* __restrict__ pts,
                const uint32_t* __restrict__ perm, const float* __restrict__ queries, uint32_t N, PassConst pc,
                float max_sqdist, const uint32_t* __restrict__ plist, const uint32_t* __restrict__ pcount,
                uint32_t* __restrict__ nn_idx, float* __restrict__ nn_d2, uint8_t* __restrict__ sel,
                uint32_t* __restrict__ count_out) {
  const uint32_t count = *pcount;
  if (blockIdx.x == 0 && threadIdx.x == 0) { count_out[0] = count; count_out[2] = count_out[1]; }   // [1] = ring-2 counter
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t lanes = 8;   // few, unrelated queries: narrow logical warps (less divergence, more warps)
  const uint32_t warp = (blockIdx.x * KNN_THREADS + threadIdx.x) >> 5, nwarps = (gridDim.x * KNN_THREADS) >> 5;
  for (uint32_t base = warp * lanes; base < count; base += nwarps * lanes) {
    const bool valid = (lane < lanes) && (base + lane < count);
    const uint32_t p = valid ? plist[base + lane] : 0u;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (valid) load_query<MODE>(pts, perm, queries, p, pc, qx, qy, qz);
    uint32_t oi[MALIO_K];
    float od[MALIO_K];
    int found = 0;
    if (n_nodes > 0) {
      knn_tree_lane<SMEM_STACK>(nodes, qx, qy, qz, valid, 0xffffffffu, oi, od, found);
    } else {
#pragma unroll
      for (int j = 0; j < MALIO_K; ++j) { oi[j] = 0xFFFFFFFFu; od[j] = INFINITY; }
    }
    if (valid) {
#pragma unroll
      for (int j = 0; j < MALIO_K; ++j) {
        nn_idx[(size_t)j * N + p] = oi[j];
        nn_d2[(size_t)j * N + p] = od[j];
      }
      if (MODE == 0) sel[p] = (found < MALIO_K) ? 0 : (od[MALIO_K - 1] > max_sqdist ? 0 : 1);   // laserMapping.cpp:587
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------ snapshot in compact form: boxes rebuilt on the device
// malio_upload_map_compact ships 16 B per node (point + link).  The 64-byte records the traversal reads (both children's
// boxes inside the parent) are rebuilt here: a node's box is the tight bounding box of the live points of its subtree
// = what KD_TREE::Update leaves in node_range_* (ikd_Tree.cpp:1469-1635).  Bottom-up, one thread per node: a thread
// stores its finished box into its parent's record and the LAST child to arrive (counter) carries the parent upwards.
constexpr uint32_t TREE_NO_PARENT = 0xFFFFFFFFu;
__global__ void tree_init_kernel(const float4* __restrict__ mpts, uint32_t n, float4* __restrict__ nodes,
                                 uint32_t* __restrict__ parent) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 a = mpts[i];
  nodes[4 * (size_t)i] = a;
  const uint32_t link = __float_as_uint(a.w);
  if (link & MALIO_LINK_HAS_LEFT) parent[i + 1] = i;
  if (link & MALIO_LINK_HAS_RIGHT) parent[link & MALIO_LINK_INDEX_MASK] = i;
  if (i == 0) parent[0] = TREE_NO_PARENT;
}
__global__ void tree_refit_kernel(const float4* __restrict__ mpts, uint32_t n, float4* nodes, const uint32_t* __restrict__ parent,
                                  uint32_t* __restrict__ arrived) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 a = mpts[i];
  const uint32_t link = __float_as_uint(a.w);
  if (link & (MALIO_LINK_HAS_LEFT | MALIO_LINK_HAS_RIGHT)) return;   // leaves start the climb
  const bool live = !(link & MALIO_LINK_POINT_DELETED);
  float x0 = live ? a.x : INFINITY, x1 = live ? a.x : -INFINITY, y0 = live ? a.y : INFINITY, y1 = live ? a.y : -INFINITY,
        z0 = live ? a.z : INFINITY, z1 = live ? a.z : -INFINITY;
  uint32_t cur = i;
  for (;;) {
    const uint32_t par = parent[cur];
    if (par == TREE_NO_PARENT) break;
    const float4 pa = mpts[par];
    const uint32_t plink = __float_as_uint(pa.w);
    const bool is_left = (plink & MALIO_LINK_HAS_LEFT) && cur == par + 1;
    float* rec = reinterpret_cast<float*>(nodes + 4 * (size_t)par);
    float* box = rec + (is_left ? 4 : 10);      // lbox at floats 4..9, rbox at 10..15
    box[0] = x0; box[1] = x1; box[2] = y0; box[3] = y1; box[4] = z0; box[5] = z1;
    const uint32_t need = ((plink & MALIO_LINK_HAS_LEFT) ? 1u : 0u) + ((plink & MALIO_LINK_HAS_RIGHT) ? 1u : 0u);
    // release our box / acquire the sibling's in the one atomic of this level (the climb is a chain of these round trips)
    uint32_t before;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(before) : "l"(arrived + par) : "memory");
    if (before + 1u < need) break;   // the sibling's thread carries the parent
    if (need == 2) {   // merge the sibling's box, written by another thread: read it from L2
      const float* sib = rec + (is_left ? 10 : 4);
      x0 = fminf(x0, __ldcg(sib + 0)); x1 = fmaxf(x1, __ldcg(sib + 1));
      y0 = fminf(y0, __ldcg(sib + 2)); y1 = fmaxf(y1, __ldcg(sib + 3));
      z0 = fminf(z0, __ldcg(sib + 4)); z1 = fmaxf(z1, __ldcg(sib + 5));
    }
    if (!(plink & MALIO_LINK_POINT_DELETED)) {
      x0 = fminf(x0, pa.x); x1 = fmaxf(x1, pa.x); y0 = fminf(y0, pa.y); y1 = fmaxf(y1, pa.y);
      z0 = fminf(z0, pa.z); z1 = fmaxf(z1, pa.z);
    }
    cur = par;
  }
}
// full-record upload: the compact mirror (point + link, 16 B stride) the plane fit and the cell-list build read
__global__ void tree_extract_kernel(const float4* __restrict__ nodes, uint32_t n, float4* __restrict__ mpts) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) mpts[i] = __ldg(nodes + 4 * (size_t)i);
}

// ------------------------------------------------------------------ K1g: cell-list k-NN, the fast path of K1
// Nearest_Search's RESULT (the 5 smallest squared distances, ascending) does not depend on how the tree is walked
// unless distances tie: acceptance is `dist < q.top().dist` (ikd_Tree.cpp:1099), so with pairwise distinct distances
// among the six closest points any exact search returns the same list.  The traversal order only matters for ties
// (first visited wins; PointType_CMP's 1e-10 window, ikd_Tree.h:102-108).  So: the live snapshot points are binned
// once per upload into a uniform grid (cell edge h), a query scans the 3x3x3 cell block around its own cell — 9
// contiguous x-rows of the cell-sorted point array, no dependent chain — keeping the 6 smallest distances, computed
// with calc_dist's exact float expression.  The block contains every point closer than r = (1 + min frac) h, so if
// the 5th distance is below r (minus a margin that covers float rounding of the cell arithmetic) and the six
// smallest distances are pairwise more than 1e-10 apart, the list IS the reference's.  Otherwise the 5x5x5 block
// is tried (r = (2 + min frac) h), and what is still unsettled — ties, very sparse neighbourhoods, queries outside
// the grid — goes to knn_list_kernel, i.e. through the exact ikd-Tree-order traversal above.


__global__ void grid_count_kernel(const float4* __restrict__ nodes, uint32_t n, GridConst G, uint32_t* __restrict__ cnt,
                                  uint32_t* __restrict__ cell_of) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 a = __ldg(nodes + i);   // compact mirror: 16 B stride
  if (__float_as_uint(a.w) & MALIO_LINK_POINT_DELETED) { cell_of[i] = 0xFFFFFFFFu; return; }
  // monotone in each coordinate (subtract, multiply by a positive constant, floor, clamp): what the radius guarantee needs
  int cx = (int)floorf((a.x - G.ox) * G.inv_h), cy = (int)floorf((a.y - G.oy) * G.inv_h), cz = (int)floorf((a.z - G.oz) * G.inv_h);
  cx = min(max(cx, 0), G.nx - 1); cy = min(max(cy, 0), G.ny - 1); cz = min(max(cz, 0), G.nz - 1);
  const uint32_t c = grid_cell_index(G, cx, cy, cz);
  cell_of[i] = c;
  atomicAdd(cnt + c, 1u);
}
// exclusive scan of the cell counts, three small kernels: chunk-local scan (+ chunk totals, occupied-cell count;
// the counts are zeroed to serve as scatter cursors), scan of the <= 8192 chunk totals, add-back
__global__ void __launch_bounds__(1024) grid_scan_local_kernel(uint32_t* __restrict__ cnt, uint32_t* __restrict__ start,
                                                               uint32_t* __restrict__ ctot, uint32_t* __restrict__ stats) {
  __shared__ uint32_t s_w[32];
  __shared__ uint32_t s_occ[32];
  const uint32_t base = (blockIdx.x * 1024u + threadIdx.x) * 4u;
  const uint4 v = *reinterpret_cast<const uint4*>(cnt + base);
  *reinterpret_cast<uint4*>(cnt + base) = make_uint4(0u, 0u, 0u, 0u);
  const uint32_t sum = v.x + v.y + v.z + v.w;
  uint32_t occ = (v.x != 0) + (v.y != 0) + (v.z != 0) + (v.w != 0);
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= (unsigned)o) inc += t; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) occ += __shfl_xor_sync(0xffffffffu, occ, o);
  if ((threadIdx.x & 31) == 31) s_w[threadIdx.x >> 5] = inc;
  if ((threadIdx.x & 31) == 0) s_occ[threadIdx.x >> 5] = occ;
  __syncthreads();
  if (threadIdx.x < 32) {   // warp 0: exclusive scan of the 32 warp totals, sum of the occupied-cell counts
    const uint32_t wt = s_w[threadIdx.x];
    uint32_t wi = wt, oc = s_occ[threadIdx.x];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o); if (threadIdx.x >= (unsigned)o) wi += t; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) oc += __shfl_xor_sync(0xffffffffu, oc, o);
    s_w[threadIdx.x] = wi - wt;
    if (threadIdx.x == 31) ctot[blockIdx.x] = wi;
    if (threadIdx.x == 0 && oc) atomicAdd(stats, oc);
  }
  __syncthreads();
  uint32_t run = s_w[threadIdx.x >> 5] + inc - sum;
  uint4 o4;
  o4.x = run; run += v.x; o4.y = run; run += v.y; o4.z = run; run += v.z; o4.w = run;
  *reinterpret_cast<uint4*>(start + base) = o4;
}
__global__ void __launch_bounds__(1024) grid_scan_tot_kernel(const uint32_t* __restrict__ ctot, uint32_t nchunk,
                                                             uint32_t* __restrict__ cbase, uint32_t* __restrict__ stats) {
  __shared__ uint32_t s_w[32];
  uint32_t v[8], sum = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) { const uint32_t i = threadIdx.x * 8 + k; v[k] = i < nchunk ? ctot[i] : 0u; sum += v[k]; }
  uint32_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= (unsigned)o) inc += t; }
  if ((threadIdx.x & 31) == 31) s_w[threadIdx.x >> 5] = inc;
  __syncthreads();
  uint32_t wbase = 0;
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wbase += s_w[w];
  uint32_t run = wbase + inc - sum;
#pragma unroll
  for (int k = 0; k < 8; ++k) { const uint32_t i = threadIdx.x * 8 + k; if (i < nchunk) cbase[i] = run; run += v[k]; }
  if (threadIdx.x == 1023) stats[1] = run;   // number of live points
}
__global__ void __launch_bounds__(1024) grid_scan_add_kernel(uint32_t* __restrict__ start, const uint32_t* __restrict__ cbase) {
  const uint32_t base = (blockIdx.x * 1024u + threadIdx.x) * 4u;
  const uint32_t b = cbase[blockIdx.x];
  uint4 v = *reinterpret_cast<uint4*>(start + base);
  v.x += b; v.y += b; v.z += b; v.w += b;
  *reinterpret_cast<uint4*>(start + base) = v;
}
__global__ void grid_scatter_kernel(const float4* __restrict__ nodes, uint32_t n, const uint32_t* __restrict__ cell_of,
                                    const uint32_t* __restrict__ start, uint32_t* __restrict__ cursor,
                                    float4* __restrict__ cell_pts) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = cell_of[i];
  if (c == 0xFFFFFFFFu) return;
  const float4 a = __ldg(nodes + i);   // compact mirror: 16 B stride
  const uint32_t slot = start[c] + atomicAdd(cursor + c, 1u);
  cell_pts[slot] = make_float4(a.x, a.y, a.z, __uint_as_float(i));
}

// the 6 smallest squared distances seen so far (ascending) and the snapshot indices of the first 5
struct Top6 {
  float d0, d1, d2, d3, d4, d5;
  uint32_t i0, i1, i2, i3, i4;
  __device__ __forceinline__ void reset() {
    d0 = d1 = d2 = d3 = d4 = d5 = INFINITY;
    i0 = i1 = i2 = i3 = i4 = 0xFFFFFFFFu;
  }
  __device__ __forceinline__ void insert(float dist, uint32_t idx) {   // precondition: dist < d5
    const bool c0 = dist < d0, c1 = dist < d1, c2 = dist < d2, c3 = dist < d3, c4 = dist < d4;
    d5 = c4 ? d4 : dist;
    d4 = c4 ? (c3 ? d3 : dist) : d4;   i4 = c4 ? (c3 ? i3 : idx) : i4;
    d3 = c3 ? (c2 ? d2 : dist) : d3;   i3 = c3 ? (c2 ? i2 : idx) : i3;
    d2 = c2 ? (c1 ? d1 : dist) : d2;   i2 = c2 ? (c1 ? i1 : idx) : i2;
    d1 = c1 ? (c0 ? d0 : dist) : d1;   i1 = c1 ? (c0 ? i0 : idx) : i1;
    d0 = c0 ? dist : d0;               i0 = c0 ? idx : i0;
  }
  // any two of the six within PointType_CMP's window (ascending list: adjacent gaps suffice)
  __device__ __forceinline__ bool tie_hazard() const {
    return (fabsf(d1 - d0) < 1e-10f) | (fabsf(d2 - d1) < 1e-10f) | (fabsf(d3 - d2) < 1e-10f) |
           (fabsf(d4 - d3) < 1e-10f) | (fabsf(d5 - d4) < 1e-10f);
  }
};

// Ring 2 (5x5x5 cells), one WARP per query.  These are the few queries (sparse neighbourhoods) whose 5th neighbour was
// not proven inside the 3x3x3 block; a single thread would need ~125 candidates x a dependent insertion chain (tens of
// microseconds of pure latency), so the candidates of one query are spread over the 32 lanes (the 25 runs flattened:
// lane j of every group of 32 candidates finds its run by a 5-step search over the prefix of the run lengths), every
// lane keeps its own 6 best, and the warp extracts the 6 overall smallest by six rounds of arg-min over the lane
// heads.  Equal heads in two lanes are a tie -> exact traversal.  Called by all 32 lanes with the same query.
template <int MODE>
__device__ __forceinline__ void ring2_query_warp(const float4* __restrict__ cell_pts, const uint32_t* __restrict__ cell_start,
                                                 const GridConst& G, float qx, float qy, float qz, uint32_t p, uint32_t N,
                                                 float max_sqdist, uint32_t* __restrict__ nn_idx, float* __restrict__ nn_d2,
                                                 uint8_t* __restrict__ sel, uint32_t* __restrict__ fb_list,
                                                 uint32_t* __restrict__ fb_count) {
  const uint32_t lane = threadIdx.x & 31u;
  const float ux = (qx - G.ox) * G.inv_h, uy = (qy - G.oy) * G.inv_h, uz = (qz - G.oz) * G.inv_h;
  const float flx = floorf(ux), fly = floorf(uy), flz = floorf(uz);
  const int cx = (int)flx, cy = (int)fly, cz = (int)flz;       // in [-1, n]: ring 1 only lists in-grid queries
  const float fx = ux - flx, fy = uy - fly, fz = uz - flz;
  const float fmin = fminf(fminf(fminf(fx, 1.f - fx), fminf(fy, 1.f - fy)), fminf(fz, 1.f - fz));
  uint32_t rs = 0, re = 0;
  if (lane < 25) {
    const uint32_t row = grid_cell_index(G, cx, cy + (int)(lane % 5) - 2, cz + (int)(lane / 5) - 2);
    rs = __ldg(cell_start + row - 2);
    re = __ldg(cell_start + row + 3);
  }
  Top6 t;
  t.reset();
  // flatten the 25 runs: lane j of every group of 32 candidates finds its run by a 5-step search over the exclusive
  // prefix of the run lengths (held one per lane), so the whole block costs ceil(total / 32) memory round trips
  const uint32_t len = re - rs;
  uint32_t inc = len;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (uint32_t)o) inc += v; }
  const uint32_t excl = inc - len, total = __shfl_sync(0xffffffffu, inc, 31);
  for (uint32_t base = 0; base < total; base += 32) {
    const uint32_t j = base + lane;
    uint32_t r = 0;
#pragma unroll
    for (int step = 16; step > 0; step >>= 1) {
      const uint32_t cand = r + step;
      const uint32_t ex = __shfl_sync(0xffffffffu, excl, cand & 31u);
      if (cand < 32u && ex <= j) r = cand;
    }
    const uint32_t ex_r = __shfl_sync(0xffffffffu, excl, r), rs_r = __shfl_sync(0xffffffffu, rs, r);
    if (j < total) {
      const float4 c = __ldg(cell_pts + rs_r + (j - ex_r));
      const float dist = (qx - c.x) * (qx - c.x) + (qy - c.y) * (qy - c.y) + (qz - c.z) * (qz - c.z);   // calc_dist
      if (dist < t.d5) t.insert(dist, __float_as_uint(c.w));
    }
  }
  // six rounds: smallest lane head overall, popped from the lane that holds it
  float od[6];
  uint32_t oi[6];
  bool hazard = false;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    float m = t.d0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const uint32_t who = __ballot_sync(0xffffffffu, t.d0 == m && m < INFINITY);
    if (__popc(who) > 1) hazard = true;
    const int src = who ? __ffs(who) - 1 : 0;
    od[k] = m;
    oi[k] = __shfl_sync(0xffffffffu, t.i0, src);
    if (who && (int)lane == src) {
      t.d0 = t.d1; t.d1 = t.d2; t.d2 = t.d3; t.d3 = t.d4; t.d4 = t.d5; t.d5 = INFINITY;
      t.i0 = t.i1; t.i1 = t.i2; t.i2 = t.i3; t.i3 = t.i4; t.i4 = 0xFFFFFFFFu;
    }
  }
  hazard |= (fabsf(od[1] - od[0]) < 1e-10f) | (fabsf(od[2] - od[1]) < 1e-10f) | (fabsf(od[3] - od[2]) < 1e-10f) |
            (fabsf(od[4] - od[3]) < 1e-10f) | (fabsf(od[5] - od[4]) < 1e-10f);
  const float rg = (2.f + fmin - GRID_MARGIN) * G.h;
  const bool settled = (od[4] < rg * rg) & !hazard;
  if (lane == 0) {
    if (settled) {
#pragma unroll
      for (int k = 0; k < MALIO_K; ++k) { nn_idx[(size_t)k * N + p] = oi[k]; nn_d2[(size_t)k * N + p] = od[k]; }
      if (MODE == 0) sel[p] = (od[4] > max_sqdist) ? 0 : 1;   // laserMapping.cpp:587 (five were found)
    } else {
      fb_list[atomicAdd(fb_count, 1u)] = p;
    }
  }
}

// One query per thread (3x3x3 cells).  Queries whose 5th neighbour is not proven inside the block are retried on the
// 5x5x5 block by the whole warp (ring2_query_warp) before the kernel ends; tie hazards and out-of-grid queries go to the
// traversal list.  The nine cell ranges are fetched up front, the candidates are read with independent 16-byte loads in
// batches of four straight into registers.  No dynamic shared memory, so occupancy is bounded by registers only and the
// latency of a batch is hidden by other warps.
#ifndef MALIO_GD_THREADS
#define MALIO_GD_THREADS 128
#endif
#ifndef MALIO_GD_BATCH
#define MALIO_GD_BATCH 4
#endif
constexpr int GD_THREADS = MALIO_GD_THREADS;
constexpr int GD_BATCH = MALIO_GD_BATCH;     // independent candidate loads in flight per thread
template <int MODE>
__global__ void __launch_bounds__(GD_THREADS)
knn_direct_kernel(const float4* __restrict__ cell_pts, const uint32_t* __restrict__ cell_start, GridConst G,
                  const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm,
                  const float* __restrict__ queries, uint32_t N, PassConst pc, float max_sqdist,
                  float4* __restrict__ world, uint32_t* __restrict__ nn_idx, float* __restrict__ nn_d2,
                  uint8_t* __restrict__ sel, uint32_t* __restrict__ r2_count, uint32_t* __restrict__ fb_list,
                  uint32_t* __restrict__ fb_count, unsigned long long* __restrict__ cand_total) {
  uint32_t n_cand = 0;   // candidates this thread scanned (statistics for the roofline; only summed when asked for)
  const uint32_t p = blockIdx.x * GD_THREADS + threadIdx.x;
  bool want_r2 = false;
  float qx = 0.f, qy = 0.f, qz = 0.f;
  if (p < N) {
    load_query<MODE>(pts, perm, queries, p, pc, qx, qy, qz);
    if (MODE == 0) world[p] = make_float4(qx, qy, qz, 0.f);
    const float ux = (qx - G.ox) * G.inv_h, uy = (qy - G.oy) * G.inv_h, uz = (qz - G.oz) * G.inv_h;
    const float flx = floorf(ux), fly = floorf(uy), flz = floorf(uz);
    // own cell in [-1, n] per axis: the 5x5x5 block then stays inside the GRID_PAD = 3 border of empty cells
    const bool in_grid = flx >= -1.f && fly >= -1.f && flz >= -1.f && flx <= (float)G.nx && fly <= (float)G.ny && flz <= (float)G.nz;
    bool settled = false, hazard = false;
    Top6 t;
    t.reset();
    if (in_grid) {
      const int cx = (int)flx, cy = (int)fly, cz = (int)flz;
      const float fx = ux - flx, fy = uy - fly, fz = uz - flz;
      const float fmin = fminf(fminf(fminf(fx, 1.f - fx), fminf(fy, 1.f - fy)), fminf(fz, 1.f - fz));
      uint32_t ra[9], rb[9];
#pragma unroll
      for (int r = 0; r < 9; ++r) {
        const uint32_t row = grid_cell_index(G, cx, cy + (r % 3) - 1, cz + (r / 3) - 1);
        ra[r] = __ldg(cell_start + row - 1);
        rb[r] = __ldg(cell_start + row + 2);
      }
#pragma unroll
      for (int r = 0; r < 9; ++r) {
        uint32_t a = ra[r];
        const uint32_t b = rb[r];
        n_cand += b - a;
        while (a < b) {
          const uint32_t left = b - a;
          // GD_BATCH independent loads in flight (indices past the run are clamped to its first entry and ignored below)
          float4 c[GD_BATCH];
#pragma unroll
          for (int k = 0; k < GD_BATCH; ++k) c[k] = __ldg(cell_pts + (left > (uint32_t)k ? a + k : a));
#pragma unroll
          for (int k = 0; k < GD_BATCH; ++k) {
            if (left > (uint32_t)k) {
              const float dist = (qx - c[k].x) * (qx - c[k].x) + (qy - c[k].y) * (qy - c[k].y) + (qz - c[k].z) * (qz - c[k].z);   // calc_dist
              if (dist < t.d5) t.insert(dist, __float_as_uint(c[k].w));
            }
          }
          a += GD_BATCH;
        }
      }
      const float rg = (1.f + fmin - GRID_MARGIN) * G.h;
      hazard = t.tie_hazard();
      settled = (t.d4 < rg * rg) & !hazard;
    }
    if (settled) {
      nn_idx[p] = t.i0;                  nn_d2[p] = t.d0;
      nn_idx[(size_t)N + p] = t.i1;      nn_d2[(size_t)N + p] = t.d1;
      nn_idx[(size_t)2 * N + p] = t.i2;  nn_d2[(size_t)2 * N + p] = t.d2;
      nn_idx[(size_t)3 * N + p] = t.i3;  nn_d2[(size_t)3 * N + p] = t.d3;
      nn_idx[(size_t)4 * N + p] = t.i4;  nn_d2[(size_t)4 * N + p] = t.d4;
      if (MODE == 0) sel[p] = (t.d4 > max_sqdist) ? 0 : 1;
    } else if (in_grid && !hazard) {
      want_r2 = true;
    } else {
      fb_list[atomicAdd(fb_count, 1u)] = p;
    }
  }
  unsigned r2mask = __ballot_sync(0xffffffffu, want_r2);
  if (r2mask && (threadIdx.x & 31u) == 0) atomicAdd(r2_count, (uint32_t)__popc(r2mask));
  while (r2mask) {
    const int src = __ffs(r2mask) - 1;
    r2mask &= r2mask - 1;
    const float bx = __shfl_sync(0xffffffffu, qx, src), by = __shfl_sync(0xffffffffu, qy, src), bz = __shfl_sync(0xffffffffu, qz, src);
    const uint32_t bp = __shfl_sync(0xffffffffu, p, src);
    ring2_query_warp<MODE>(cell_pts, cell_start, G, bx, by, bz, bp, N, max_sqdist, nn_idx, nn_d2, sel, fb_list, fb_count);
  }
  if (cand_total) {
    const uint32_t act = __activemask();
    const uint32_t tot = __reduce_add_sync(act, n_cand);
    if ((threadIdx.x & 31u) == (uint32_t)(__ffs(act) - 1)) atomicAdd(cand_total, (unsigned long long)tot);
  }
}

// Key scan: the 3x3x3 scan with ONE 32-bit key per kept candidate and G lanes per query (G = 2, 4; the template also covers 1, 8).
//
// (1) Keys.  The thread-per-query scan above spends most of its instructions on the sorted insertion of (distance, index)
// pairs (5 compares + ~20 selects per candidate, executed by the whole warp whenever one lane inserts).  Here a candidate is
// the key  (float bits of dist with the low 10 mantissa bits cleared) | row << 6 | offset-in-row : squared distances are
// non-negative, so their bit patterns order like the numbers, the low bits make every key of a query unique, and the six
// smallest keys are kept by a branch-free min/max chain (11 instructions).  The truncation keeps 13 mantissa bits; exactness
// is restored afterwards: the five winners are re-read, their distances recomputed with calc_dist's expression and sorted
// exactly.  Every candidate that was NOT kept has dist >= T5 := the truncated distance of the 6th key, so the five are the
// true five nearest whenever T5 - e4 >= 1e-10 (e4 = their largest exact distance; 1e-10 = PointType_CMP's window).  Otherwise
// (~0.06 % of the queries: 5th and 6th distance agree in 13 bits) the query is redone by the exact warp-cooperative 5x5x5
// scan, as are the queries whose 5th neighbour is not proven inside the block; ties among the five go to the traversal list.
// Rows longer than 64 candidates do not fit the 6-bit offset: such queries (maps far denser than the 2..9 points per cell
// the index is tuned for) are handed to the list as well.  Results are identical to the scan above by construction.
//
// (2) Groups.  A 100k-query search is 0.59 waves of a thread-per-query kernel: it lasts as long as ONE warp's dependent chain
// however few queries a GPU holds.  With G lanes per query the chain is G times shorter and there are G times more warps;
// every lane keeps the six smallest keys of its share, six rounds of arg-min over the lane heads merge them (keys are unique,
// so the owner of the minimum is unique).  The per-query preamble (state transform in double, cell coordinates, the nine row
// ranges) is done once per query by the first 128/G threads of the block and handed over through shared memory.
constexpr uint32_t KEY_LOW = 0x3FFu;                 // row (4 bits) << 6 | offset (6 bits)
constexpr uint32_t KEY_ROW_MAX = 64;                 // candidates per row the offset field can number
struct Keys6 {
  uint32_t k0, k1, k2, k3, k4, k5;
  __device__ __forceinline__ void reset() { k0 = k1 = k2 = k3 = k4 = k5 = 0xFFFFFFFFu; }
  __device__ __forceinline__ void insert(uint32_t x) {
    uint32_t m = max(k0, x); k0 = min(k0, x);
    uint32_t t = max(k1, m); k1 = min(k1, m); m = t;
    t = max(k2, m); k2 = min(k2, m); m = t;
    t = max(k3, m); k3 = min(k3, m); m = t;
    t = max(k4, m); k4 = min(k4, m); m = t;
    k5 = min(k5, m);
  }
  __device__ __forceinline__ void pop() { k0 = k1; k1 = k2; k2 = k3; k3 = k4; k4 = k5; k5 = 0xFFFFFFFFu; }
};
template <int MODE, int G, bool PRE>
__global__ void __launch_bounds__(GD_THREADS)
knn_keys_kernel(const float4* __restrict__ cell_pts, const uint32_t* __restrict__ cell_start, GridConst Gc,
                const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm,
                const float* __restrict__ queries, uint32_t N, PassConst pc, float max_sqdist,
                float4* __restrict__ world, uint32_t* __restrict__ nn_idx, float* __restrict__ nn_d2,
                uint8_t* __restrict__ sel, uint32_t* __restrict__ r2_count, uint32_t* __restrict__ fb_list,
                uint32_t* __restrict__ fb_count, unsigned long long* __restrict__ cand_total) {
  constexpr int QPB = GD_THREADS / G;          // queries per block
  constexpr int B = G == 1 ? 4 : 2;            // independent candidate loads in flight per lane
  __shared__ float4 s_q[QPB];                  // x, y, z, containment radius^2 (-1: outside the grid, -2: row too long for the key)
  __shared__ uint2 s_rng[9][QPB];              // first candidate, length of the nine x-rows
  if (threadIdx.x < QPB) {
    const uint32_t p = blockIdx.x * QPB + threadIdx.x;
    uint32_t n_cand = 0;
    float4 q = make_float4(0.f, 0.f, 0.f, -1.f);
    uint2 rng[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) rng[r] = make_uint2(0u, 0u);
    if (p < N) {
      load_query<MODE>(pts, perm, queries, p, pc, q.x, q.y, q.z);
      if (MODE == 0) world[p] = make_float4(q.x, q.y, q.z, 0.f);
      const float ux = (q.x - Gc.ox) * Gc.inv_h, uy = (q.y - Gc.oy) * Gc.inv_h, uz = (q.z - Gc.oz) * Gc.inv_h;
      const float flx = floorf(ux), fly = floorf(uy), flz = floorf(uz);
      const bool in_grid = flx >= -1.f && fly >= -1.f && flz >= -1.f && flx <= (float)Gc.nx && fly <= (float)Gc.ny && flz <= (float)Gc.nz;
      if (in_grid) {
        const int cx = (int)flx, cy = (int)fly, cz = (int)flz;
        const float fx = ux - flx, fy = uy - fly, fz = uz - flz;
        const float fmin = fminf(fminf(fminf(fx, 1.f - fx), fminf(fy, 1.f - fy)), fminf(fz, 1.f - fz));
        const float rg = (1.f + fmin - GRID_MARGIN) * Gc.h;
        q.w = rg * rg;
        uint32_t longest = 0;
#pragma unroll
        for (int r = 0; r < 9; ++r) {
          const uint32_t row = grid_cell_index(Gc, cx, cy + (r % 3) - 1, cz + (r / 3) - 1);
          const uint32_t a = __ldg(cell_start + row - 1), b = __ldg(cell_start + row + 2);
          rng[r] = make_uint2(a, b - a);
          n_cand += b - a;
          longest = max(longest, b - a);
        }
        if (longest > KEY_ROW_MAX) {
          q.w = -2.f;
#pragma unroll
          for (int r = 0; r < 9; ++r) rng[r].y = 0u;
        }
      }
    }
    s_q[threadIdx.x] = q;
#pragma unroll
    for (int r = 0; r < 9; ++r) s_rng[r][threadIdx.x] = rng[r];
    if (cand_total) {
      const uint32_t act = __activemask();
      const uint32_t tot = __reduce_add_sync(act, n_cand);
      if ((threadIdx.x & 31u) == (uint32_t)(__ffs(act) - 1)) atomicAdd(cand_total, (unsigned long long)tot);
    }
  }
  __syncthreads();
  const uint32_t ql = threadIdx.x / G, sub = threadIdx.x % G;
  const uint32_t p = blockIdx.x * QPB + ql;
  const float4 q = s_q[ql];
  Keys6 t;
  t.reset();
  if (PRE) {
    // the first candidate of this lane in every row: nine independent loads in flight at once (with G >= 4 that is most of the
    // block: rows hold ~4 candidates), instead of nine dependent load -> insert round trips
    float4 c0[9];
    uint32_t len[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) {
      const uint2 rg = s_rng[r][ql];
      len[r] = rg.y;
      c0[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (sub < rg.y) c0[r] = __ldg(cell_pts + rg.x + sub);
    }
#pragma unroll
    for (int r = 0; r < 9; ++r) {
      const float dist = (q.x - c0[r].x) * (q.x - c0[r].x) + (q.y - c0[r].y) * (q.y - c0[r].y) + (q.z - c0[r].z) * (q.z - c0[r].z);   // calc_dist
      const uint32_t key = (__float_as_uint(dist) & ~KEY_LOW) | (uint32_t)(r << 6) | sub;
      t.insert(sub < len[r] ? key : 0xFFFFFFFFu);
    }
  }
#pragma unroll
  for (int r = 0; r < 9; ++r) {
    const uint2 rg = s_rng[r][ql];
    const float4* __restrict__ run = cell_pts + rg.x;
    for (uint32_t off = sub + (PRE ? G : 0); off < rg.y; off += G * B) {
      float4 c[B];
      uint32_t o[B];
#pragma unroll
      for (int k = 0; k < B; ++k) {
        o[k] = off + k * G;
        c[k] = __ldg(run + (o[k] < rg.y ? o[k] : off));   // past the run: re-read the first one, its key is voided below
      }
#pragma unroll
      for (int k = 0; k < B; ++k) {
        const float dist = (q.x - c[k].x) * (q.x - c[k].x) + (q.y - c[k].y) * (q.y - c[k].y) + (q.z - c[k].z) * (q.z - c[k].z);   // calc_dist
        const uint32_t key = (__float_as_uint(dist) & ~KEY_LOW) | (uint32_t)(r << 6) | o[k];
        t.insert(o[k] < rg.y ? key : 0xFFFFFFFFu);
      }
    }
  }
  // ---- merge: six rounds of arg-min over the G lane heads (xor shuffles below G stay inside the aligned group)
  uint32_t mk[6];
  if (G == 1) {
    mk[0] = t.k0; mk[1] = t.k1; mk[2] = t.k2; mk[3] = t.k3; mk[4] = t.k4; mk[5] = t.k5;
  } else {
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      uint32_t m = t.k0;
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
      mk[k] = m;
      if (t.k0 == m) t.pop();       // keys are unique inside a query; several lanes popping the all-ones filler is harmless
    }
  }
  // ---- exact distances of the five winners (calc_dist's expression), sorted exactly
  float e[5];
  uint32_t id[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    e[k] = INFINITY; id[k] = 0xFFFFFFFFu;
    if (mk[k] != 0xFFFFFFFFu) {
      const float4 c = __ldg(cell_pts + s_rng[(mk[k] >> 6) & 15u][ql].x + (mk[k] & 63u));
      e[k] = (q.x - c.x) * (q.x - c.x) + (q.y - c.y) * (q.y - c.y) + (q.z - c.z) * (q.z - c.z);
      id[k] = __float_as_uint(c.w);
    }
  }
#define MALIO_CE(a, b)                                                               \
  {                                                                                  \
    const bool sw = e[a] > e[b];                                                     \
    const float ea = sw ? e[b] : e[a], eb = sw ? e[a] : e[b];                        \
    const uint32_t ia = sw ? id[b] : id[a], ib = sw ? id[a] : id[b];                 \
    e[a] = ea; e[b] = eb; id[a] = ia; id[b] = ib;                                    \
  }
  MALIO_CE(0, 1) MALIO_CE(3, 4) MALIO_CE(2, 4) MALIO_CE(2, 3) MALIO_CE(1, 4) MALIO_CE(0, 3) MALIO_CE(0, 2) MALIO_CE(1, 3) MALIO_CE(1, 2)
#undef MALIO_CE
  const bool tie = (fabsf(e[1] - e[0]) < 1e-10f) | (fabsf(e[2] - e[1]) < 1e-10f) | (fabsf(e[3] - e[2]) < 1e-10f) | (fabsf(e[4] - e[3]) < 1e-10f);
  const float t5 = mk[5] == 0xFFFFFFFFu ? INFINITY : __uint_as_float(mk[5] & ~KEY_LOW);
  const bool set_exact = (t5 - e[4]) >= 1e-10f;         // every candidate outside the five is farther than e4 by the tie window
  const bool in_grid = q.w >= 0.f;
  const bool settled = in_grid & !tie & set_exact & (e[4] < q.w);
  bool want_r2 = false;
  if (p < N) {
    if (settled) {
#pragma unroll
      for (int k = 0; k < MALIO_K; ++k)
        if ((k % G) == (int)sub) { nn_idx[(size_t)k * N + p] = id[k]; nn_d2[(size_t)k * N + p] = e[k]; }
      if (MODE == 0 && sub == 0) sel[p] = (e[4] > max_sqdist) ? 0 : 1;   // laserMapping.cpp:587 (five were found)
    } else if (sub == 0) {
      if (in_grid && !tie) want_r2 = true;        // not proven inside the 3x3x3 block, or the 13-bit keys could not separate 5th and 6th
      else fb_list[atomicAdd(fb_count, 1u)] = p;  // outside the grid, over-long row, or a tie among the five
    }
  }
  const uint32_t lane = threadIdx.x & 31u;
  unsigned r2mask = __ballot_sync(0xffffffffu, want_r2);
  if (r2mask && lane == 0) atomicAdd(r2_count, (uint32_t)__popc(r2mask));
  while (r2mask) {
    const int src = __ffs(r2mask) - 1;
    r2mask &= r2mask - 1;
    const float bx = __shfl_sync(0xffffffffu, q.x, src), by = __shfl_sync(0xffffffffu, q.y, src), bz = __shfl_sync(0xffffffffu, q.z, src);
    const uint32_t bp = __shfl_sync(0xffffffffu, p, src);
    ring2_query_warp<MODE>(cell_pts, cell_start, Gc, bx, by, bz, bp, N, max_sqdist, nn_idx, nn_d2, sel, fb_list, fb_count);
  }
}

// ------------------------------------------------------------------ K1r: tree-free exact search (device-resident map mode)
// When the map lives on the device as a point set kept in step with the host's ikd-Tree by deltas (malio_mapops.cu), there
// is no flattened tree to walk.  The queries the 3x3x3 / 5x5x5 scans leave open — sparse neighbourhoods, queries outside the
// grid, tie hazards — are settled by one warp per query scanning cell blocks of growing half-width r: the block contains
// every point closer than (r + min frac - margin) h, so the list is final once the 5th distance is below that radius, or once
// the block covers the whole grid.  Same float distance expression as everywhere (calc_dist).  Ties (two of the six best
// within PointType_CMP's 1e-10 window) cannot be resolved the reference's way without its traversal order: they are broken
// by the smaller slot index, deterministically, and COUNTED (malio_counters.knn_tie_queries) — the documented exemption of
// SURVEY.md §7 ("ties at the k-th boundary resolve by first visited wins ... the harness must detect and exempt exact ties").
struct Top6T {
  float d0, d1, d2, d3, d4, d5;
  uint32_t i0, i1, i2, i3, i4, i5;
  __device__ __forceinline__ void reset() {
    d0 = d1 = d2 = d3 = d4 = d5 = INFINITY;
    i0 = i1 = i2 = i3 = i4 = i5 = 0xFFFFFFFFu;
  }
  static __device__ __forceinline__ bool lt(float da, uint32_t ia, float db, uint32_t ib) { return da < db || (da == db && ia < ib); }
  __device__ __forceinline__ void insert(float dist, uint32_t idx) {   // precondition: lt(dist, idx, d5, i5)
    const bool c0 = lt(dist, idx, d0, i0), c1 = lt(dist, idx, d1, i1), c2 = lt(dist, idx, d2, i2), c3 = lt(dist, idx, d3, i3), c4 = lt(dist, idx, d4, i4);
    d5 = c4 ? d4 : dist;               i5 = c4 ? i4 : idx;
    d4 = c4 ? (c3 ? d3 : dist) : d4;   i4 = c4 ? (c3 ? i3 : idx) : i4;
    d3 = c3 ? (c2 ? d2 : dist) : d3;   i3 = c3 ? (c2 ? i2 : idx) : i3;
    d2 = c2 ? (c1 ? d1 : dist) : d2;   i2 = c2 ? (c1 ? i1 : idx) : i2;
    d1 = c1 ? (c0 ? d0 : dist) : d1;   i1 = c1 ? (c0 ? i0 : idx) : i1;
    d0 = c0 ? dist : d0;               i0 = c0 ? idx : i0;
  }
  __device__ __forceinline__ void pop() {
    d0 = d1; d1 = d2; d2 = d3; d3 = d4; d4 = d5; d5 = INFINITY;
    i0 = i1; i1 = i2; i2 = i3; i3 = i4; i4 = i5; i5 = 0xFFFFFFFFu;
  }
};
template <int MODE>
__device__ __forceinline__ void ring_search_warp(const float4* __restrict__ cell_pts, const uint32_t* __restrict__ cell_start,
                                                 const GridConst& G, float qx, float qy, float qz, uint32_t p, uint32_t N,
                                                 float max_sqdist, uint32_t* __restrict__ nn_idx, float* __restrict__ nn_d2,
                                                 uint8_t* __restrict__ sel, uint32_t* __restrict__ tie_count) {
  const uint32_t lane = threadIdx.x & 31u;
  float od[6];
  uint32_t oi[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) { od[k] = INFINITY; oi[k] = 0xFFFFFFFFu; }
  const bool finite = isfinite(qx) && isfinite(qy) && isfinite(qz);
  if (finite) {
    const float lim = 1.0e9f;
    const float ux = fminf(fmaxf((qx - G.ox) * G.inv_h, -lim), lim), uy = fminf(fmaxf((qy - G.oy) * G.inv_h, -lim), lim),
                uz = fminf(fmaxf((qz - G.oz) * G.inv_h, -lim), lim);
    const float flx = floorf(ux), fly = floorf(uy), flz = floorf(uz);
    const long long cx = (long long)flx, cy = (long long)fly, cz = (long long)flz;
    const float fx = ux - flx, fy = uy - fly, fz = uz - flz;
    const float fmin = fminf(fminf(fminf(fx, 1.f - fx), fminf(fy, 1.f - fy)), fminf(fz, 1.f - fz));
    // rounding of (q - o) * inv_h grows with its magnitude: ~2^-22 relative
    const float margin = GRID_MARGIN + 4.0e-7f * fmaxf(fmaxf(fabsf(ux), fabsf(uy)), fabsf(uz));
    auto outside = [](long long c, int n) -> long long { return c < 0 ? -c : (c > (long long)n - 1 ? c - ((long long)n - 1) : 0); };
    long long r = outside(cx, G.nx);
    r = r > outside(cy, G.ny) ? r : outside(cy, G.ny);
    r = r > outside(cz, G.nz) ? r : outside(cz, G.nz);
    if (r < 3) r = 3;
    for (;;) {
      const int x0 = (int)(cx - r > 0 ? cx - r : 0), x1 = (int)(cx + r < G.nx - 1 ? cx + r : G.nx - 1);
      const int y0 = (int)(cy - r > 0 ? cy - r : 0), y1 = (int)(cy + r < G.ny - 1 ? cy + r : G.ny - 1);
      const int z0 = (int)(cz - r > 0 ? cz - r : 0), z1 = (int)(cz + r < G.nz - 1 ? cz + r : G.nz - 1);
      const bool covers_all = (cx - r <= 0) && (cx + r >= G.nx - 1) && (cy - r <= 0) && (cy + r >= G.ny - 1) && (cz - r <= 0) && (cz + r >= G.nz - 1);
      Top6T t;
      t.reset();
      if (x0 <= x1 && y0 <= y1 && z0 <= z1) {
        const uint32_t ycnt = (uint32_t)(y1 - y0 + 1), nrows = ycnt * (uint32_t)(z1 - z0 + 1);
        for (uint32_t rowbase = 0; rowbase < nrows; rowbase += 32) {
          const uint32_t row = rowbase + lane;
          uint32_t rs = 0, re = 0;
          if (row < nrows) {
            const int y = y0 + (int)(row % ycnt), z = z0 + (int)(row / ycnt);
            rs = __ldg(cell_start + grid_cell_index(G, x0, y, z));
            re = __ldg(cell_start + grid_cell_index(G, x1, y, z) + 1);
          }
          const uint32_t len = re - rs;
          uint32_t inc = len;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (uint32_t)o) inc += v; }
          const uint32_t excl = inc - len, total = __shfl_sync(0xffffffffu, inc, 31);
          for (uint32_t base = 0; base < total; base += 32) {
            const uint32_t j = base + lane;
            uint32_t rr = 0;
#pragma unroll
            for (int step = 16; step > 0; step >>= 1) {
              const uint32_t cand = rr + step;
              const uint32_t ex = __shfl_sync(0xffffffffu, excl, cand & 31u);
              if (cand < 32u && ex <= j) rr = cand;
            }
            const uint32_t ex_r = __shfl_sync(0xffffffffu, excl, rr), rs_r = __shfl_sync(0xffffffffu, rs, rr);
            if (j < total) {
              const float4 c = __ldg(cell_pts + rs_r + (j - ex_r));
              const float dist = (qx - c.x) * (qx - c.x) + (qy - c.y) * (qy - c.y) + (qz - c.z) * (qz - c.z);   // calc_dist
              const uint32_t idx = __float_as_uint(c.w);
              if (Top6T::lt(dist, idx, t.d5, t.i5)) t.insert(dist, idx);
            }
          }
        }
      }
      // six rounds of (distance, slot) arg-min over the lane heads
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        float m = t.d0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
        uint32_t mi = (t.d0 == m) ? t.i0 : 0xFFFFFFFFu;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mi = min(mi, __shfl_xor_sync(0xffffffffu, mi, o));
        od[k] = m; oi[k] = (m < INFINITY) ? mi : 0xFFFFFFFFu;
        if (m < INFINITY && t.d0 == m && t.i0 == mi) t.pop();
      }
      const float rg = ((float)r + fmin - margin) * G.h;
      if (covers_all || od[4] < rg * rg) break;
      r = r + (r >> 1) + 1;
    }
  }
  if (lane == 0) {
    const bool tie = (od[1] < INFINITY && fabsf(od[1] - od[0]) < 1e-10f) | (od[2] < INFINITY && fabsf(od[2] - od[1]) < 1e-10f) |
                     (od[3] < INFINITY && fabsf(od[3] - od[2]) < 1e-10f) | (od[4] < INFINITY && fabsf(od[4] - od[3]) < 1e-10f) |
                     (od[5] < INFINITY && fabsf(od[5] - od[4]) < 1e-10f);
    if (tie) atomicAdd(tie_count, 1u);
#pragma unroll
    for (int k = 0; k < MALIO_K; ++k) { nn_idx[(size_t)k * N + p] = oi[k]; nn_d2[(size_t)k * N + p] = od[k]; }
    if (MODE == 0) sel[p] = (oi[4] == 0xFFFFFFFFu) ? 0 : (od[4] > max_sqdist ? 0 : 1);   // laserMapping.cpp:587
  }
}
template <int MODE>
__global__ void __launch_bounds__(KNN_THREADS)
knn_ring_kernel(const float4* __restrict__ cell_pts, const uint32_t* __restrict__ cell_start, GridConst G,
                const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm, const float* __restrict__ queries,
                uint32_t N, PassConst pc, float max_sqdist, const uint32_t* __restrict__ plist, const uint32_t* __restrict__ pcount,
                uint32_t* __restrict__ nn_idx, float* __restrict__ nn_d2, uint8_t* __restrict__ sel, uint32_t* __restrict__ count_out,
                uint32_t* __restrict__ tie_count) {
  const uint32_t count = *pcount;
  if (blockIdx.x == 0 && threadIdx.x == 0) { count_out[0] = count; count_out[2] = count_out[1]; }
  const uint32_t warp = (blockIdx.x * KNN_THREADS + threadIdx.x) >> 5, nwarps = (gridDim.x * KNN_THREADS) >> 5;
  for (uint32_t k = warp; k < count; k += nwarps) {
    const uint32_t p = plist[k];
    float qx, qy, qz;
    load_query<MODE>(pts, perm, queries, p, pc, qx, qy, qz);
    ring_search_warp<MODE>(cell_pts, cell_start, G, qx, qy, qz, p, N, max_sqdist, nn_idx, nn_d2, sel, tie_count);
  }
}

// ------------------------------------------------------------------ query ordering (internal only; outputs stay in caller order)
// Spatially coherent warps matter (neighbouring queries walk the same upper tree levels: L1 hits, similar visit
// counts), the exact order does not.  A general radix sort of ~1e5 keys is launch/latency-bound (CUB: 6 kernels,
// ~57 us here), so this is a hand-written counting sort on a 16-bit cell key:
//   cell = 2 m; key = z(2 bits) | Morton(x 7 bits, y 7 bits)   (wraps every 256 m / 8 m: only locality matters)
//               or  LiDAR(2 bits) | z(2 bits) | Morton(x 6 bits, y 6 bits) for large scans (see count_kernel)
//   count_kernel   key per point + histogram (integer atomics)
//   scan_kernel    exclusive prefix over the 65 536 bins (64 block-local scans + 64 totals)
//   scatter_kernel slot = offset[key] + atomic cursor  -> tmp (order inside a bin is arrival order ...)
//   rank_kernel    ... so each point re-derives its slot as its rank among its bin-mates by point index: the final
//                  permutation is a pure function of the input (bit-reproducible reduction order downstream)
constexpr int SORT_BINS = 1 << 16;
__device__ __forceinline__ uint32_t spread7(uint32_t v) {   // 7 bits -> every other bit
  v &= 0x7Fu;
  v = (v | (v << 4)) & 0x070Fu;
  v = (v | (v << 2)) & 0x1333u;
  v = (v | (v << 1)) & 0x1555u;
  return v;
}
template <int MODE>
__global__ void count_kernel(const malio_scan_pt* __restrict__ pts, const float* __restrict__ queries, uint32_t N,
                             PassConst pc, int lid_major, uint16_t* __restrict__ keys, uint32_t* __restrict__ hist) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float x, y, z;
  uint32_t lid_key = 0;
  if (MODE == 0) {
    const malio_scan_pt pt = pts[i];
    double b[3], m[3], g[3];
    transform_point(pc, pt.x, pt.y, pt.z, pt.lidar, b, m, g);
    x = (float)g[0]; y = (float)g[1]; z = (float)g[2];
    lid_key = pt.lidar < 3 ? pt.lidar : 3u;
  } else {
    x = queries[3 * (size_t)i]; y = queries[3 * (size_t)i + 1]; z = queries[3 * (size_t)i + 2];
  }
  const uint32_t ix = (uint32_t)(int)floorf(x * 0.5f), iy = (uint32_t)(int)floorf(y * 0.5f), iz = (uint32_t)(int)floorf(z * 0.5f);
  // Small scans (the fused pass keeps all rows of a block in shared memory): pure cell order, best for the k-NN.
  // Large scans (rows go through global memory tile by tile): LiDAR id as the major key, so that the reduction can keep
  // one LiDAR's accumulators in registers while it walks its tiles.
  const uint32_t key = lid_major ? ((lid_key << 14) | ((iz & 3u) << 12) | (spread7(iy & 0x3Fu) << 1) | spread7(ix & 0x3Fu))
                                 : (((iz & 3u) << 14) | (spread7(iy) << 1) | spread7(ix));
  keys[i] = (uint16_t)key;
  atomicAdd(hist + key, 1u);
}
// 64 blocks x 1024 bins: block-local exclusive scan (coalesced uint4 loads) + the block's total; consumers add the
// prefix of the 64 totals themselves (bin_base below) — no second scan kernel, no grid-wide dependency
constexpr int SCAN_BLOCKS = 64, SCAN_THREADS = 256;
static_assert(SCAN_BLOCKS * SCAN_THREADS * 4 == SORT_BINS, "scan tiling");
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(const uint32_t* __restrict__ hist, uint32_t* __restrict__ offs,
                                                            uint32_t* __restrict__ cursor, uint32_t* __restrict__ btot) {
  __shared__ uint32_t s_w[SCAN_THREADS / 32];
  const uint32_t base = (blockIdx.x * SCAN_THREADS + threadIdx.x) * 4;
  const uint4 v = *reinterpret_cast<const uint4*>(hist + base);
  const uint32_t sum = v.x + v.y + v.z + v.w;
  uint32_t inc = sum;   // inclusive warp scan
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= (unsigned)o) inc += t; }
  if ((threadIdx.x & 31) == 31) s_w[threadIdx.x >> 5] = inc;
  __syncthreads();
  uint32_t wbase = 0;
  for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wbase += s_w[w];
  uint32_t run = wbase + inc - sum;
  uint4 o4;
  o4.x = run; run += v.x; o4.y = run; run += v.y; o4.z = run; run += v.z; o4.w = run;
  *reinterpret_cast<uint4*>(offs + base) = o4;
  *reinterpret_cast<uint4*>(cursor + base) = make_uint4(0u, 0u, 0u, 0u);
  if (threadIdx.x == SCAN_THREADS - 1) btot[blockIdx.x] = wbase + inc;
}
// prefix of the 64 block totals into shared memory (every consumer block recomputes it: 64 adds)
__device__ __forceinline__ void load_bin_base(const uint32_t* __restrict__ btot, uint32_t* s_base) {
  if (threadIdx.x < 32) {
    const uint32_t a = btot[threadIdx.x], b = btot[32 + threadIdx.x];
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o);
      if (threadIdx.x >= (unsigned)o) { ia += ta; ib += tb; }
    }
    const uint32_t tot_a = __shfl_sync(0xffffffffu, ia, 31);
    s_base[threadIdx.x] = ia - a;
    s_base[32 + threadIdx.x] = tot_a + ib - b;
  }
  __syncthreads();
}
__global__ void scatter_kernel(const uint16_t* __restrict__ keys, uint32_t N, const uint32_t* __restrict__ offs,
                               const uint32_t* __restrict__ btot, uint32_t* __restrict__ cursor, uint32_t* __restrict__ perm,
                               uint32_t* __restrict__ arrival) {
  __shared__ uint32_t s_base[SCAN_BLOCKS];
  load_bin_base(btot, s_base);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const uint32_t key = keys[i];
  const uint32_t a = atomicAdd(cursor + key, 1u);
  perm[s_base[key >> 10] + offs[key] + a] = i;
  arrival[i] = a;
}
// one thread per point: its final slot inside its bin is the number of bin-mates with a smaller index
// (bins hold ~10 points, at most a few dozen: a short, fully parallel O(cnt) scan per point).  Bins above RANK_LIMIT points
// (thousands of queries inside one 2 m cell: un-down-sampled or tiny clouds) would make that quadratic: they keep the
// arrival order of the scatter instead — still a valid permutation, only the bit-reproducibility of the internal order
// (and with it of the last bits of the reduction) is given up for such inputs.
constexpr uint32_t RANK_LIMIT = 2048;
__global__ void rank_kernel(const uint16_t* __restrict__ keys, uint32_t N, const uint32_t* __restrict__ offs,
                            const uint32_t* __restrict__ btot, const uint32_t* __restrict__ hist,
                            const uint32_t* __restrict__ tmp, const uint32_t* __restrict__ arrival, uint32_t* __restrict__ perm,
                            const malio_scan_pt* __restrict__ pts, malio_scan_pt* __restrict__ pts_sorted) {
  __shared__ uint32_t s_base[SCAN_BLOCKS];
  load_bin_base(btot, s_base);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const uint32_t key = keys[i];
  const uint32_t off = s_base[key >> 10] + offs[key], cnt = hist[key];
  uint32_t rank = 0;
  if (cnt > RANK_LIMIT) rank = arrival[i];
  else for (uint32_t j = 0; j < cnt; ++j) rank += (tmp[off + j] < i) ? 1u : 0u;
  perm[off + rank] = i;
  if (pts_sorted) pts_sorted[off + rank] = pts[i];   // position-ordered copy: the per-pass kernels read it without the perm hop
}

// ------------------------------------------------------------------ K2: plane fit, gates, point-wise uncertainty
// Eigen::ColPivHouseholderQR<Matrix<float,5,3>>::solve(b) with b = -1 (common_lib.h:156-157,174), float, no FMA.
__device__ __forceinline__ void qr_solve_5x3(float A[5][3], float x[3]) {
  const float eps = 1.1920928955078125e-07f;   // FLT_EPSILON
  float hC[3] = {0.f, 0.f, 0.f};
  int perm[3] = {0, 1, 2};
  float nU[3], nD[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 5; ++i) s += A[i][k] * A[i][k];
    nD[k] = sqrtf(s);
    nU[k] = nD[k];
  }
  const float maxn = fmaxf(nU[0], fmaxf(nU[1], nU[2]));
  const float threshold_helper = (maxn * eps) * (maxn * eps) / 5.0f;
  const float downdate_thr = sqrtf(eps);
  int nonzero = 3;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int biggest = k;
#pragma unroll
    for (int j = k + 1; j < 3; ++j) {
      float cur = nU[k];
#pragma unroll
      for (int jj = k + 1; jj < 3; ++jj) if (biggest == jj) cur = nU[jj];
      if (nU[j] > cur) biggest = j;
    }
    float bn = nU[k];
#pragma unroll
    for (int jj = k + 1; jj < 3; ++jj) if (biggest == jj) bn = nU[jj];
    if (nonzero == 3 && bn * bn < threshold_helper * (float)(5 - k)) nonzero = k;
#pragma unroll
    for (int j = k + 1; j < 3; ++j) {
      if (biggest == j) {
#pragma unroll
        for (int i = 0; i < 5; ++i) { float t = A[i][k]; A[i][k] = A[i][j]; A[i][j] = t; }
        float t = nU[k]; nU[k] = nU[j]; nU[j] = t;
        t = nD[k]; nD[k] = nD[j]; nD[j] = t;
        int ti = perm[k]; perm[k] = perm[j]; perm[j] = ti;
      }
    }
    float tailSq = 0.f;
#pragma unroll
    for (int i = k + 1; i < 5; ++i) tailSq += A[i][k] * A[i][k];
    const float c0 = A[k][k];
    float beta, tau;
    if (tailSq <= 1.17549435e-38f) {   // numeric_limits<float>::min()
      tau = 0.f; beta = c0;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) A[i][k] = 0.f;
    } else {
      beta = sqrtf(c0 * c0 + tailSq);
      if (c0 >= 0.f) beta = -beta;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) A[i][k] = A[i][k] / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    A[k][k] = beta;
    hC[k] = tau;
    if (tau != 0.f) {
#pragma unroll
      for (int j = k + 1; j < 3; ++j) {
        float tmp = 0.f;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) tmp += A[i][k] * A[i][j];
        tmp += A[k][j];
        A[k][j] -= tau * tmp;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) A[i][j] -= tau * A[i][k] * tmp;
      }
    }
#pragma unroll
    for (int j = k + 1; j < 3; ++j) {
      if (nU[j] != 0.f) {
        float temp = fabsf(A[k][j]) / nU[j];
        temp = (1.f + temp) * (1.f - temp);
        temp = temp < 0.f ? 0.f : temp;
        const float r = nU[j] / nD[j];
        const float temp2 = temp * r * r;
        if (temp2 <= downdate_thr) {
          float s = 0.f;
#pragma unroll
          for (int i = k + 1; i < 5; ++i) s += A[i][j] * A[i][j];
          nD[j] = sqrtf(s);
          nU[j] = nD[j];
        } else {
          nU[j] *= sqrtf(temp);
        }
      }
    }
  }
  float c[5] = {-1.f, -1.f, -1.f, -1.f, -1.f};
  x[0] = x[1] = x[2] = 0.f;
  if (nonzero == 0) return;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (k < nonzero && hC[k] != 0.f) {
      float tmp = 0.f;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) tmp += A[i][k] * c[i];
      tmp += c[k];
      c[k] -= hC[k] * tmp;
#pragma unroll
      for (int i = k + 1; i < 5; ++i) c[i] -= hC[k] * A[i][k] * tmp;
    }
  }
#pragma unroll
  for (int i = 2; i >= 0; --i) {
    if (i < nonzero) {
      float s = c[i];
#pragma unroll
      for (int j = i + 1; j < 3; ++j) if (j < nonzero) s -= A[i][j] * c[j];
      c[i] = s / A[i][i];
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < nonzero) {
#pragma unroll
      for (int q = 0; q < 3; ++q) if (perm[i] == q) x[q] = c[i];
    }
  }
}

// trace of evalPointUncertainty's 3x3 (associate_uct.hpp:153-175) in closed form:
//   G = [ q_w I | -[q]x | T(0:3,0:3) ], q = T (0.05 p, 1);  Sigma_in = blkdiag(1e4 cov, 0.1 I)
//   trace = sum_{i<3} (F (1e4 cov) F^T)_ii + 0.1 |T(0:3,0:3)|_F^2,  F = [ q_w I | -[q]x ]
// Row i of F has three non-zeros, so (F S F^T)_ii is a 3x3 quadratic form: 27 terms instead of the dense 9x9
// product.  `e` is one table entry as uploaded: T (16) then cov (36).
__device__ __forceinline__ double point_cov_trace(float px, float py, float pz, const double* __restrict__ e) {
  const double pc0 = px * 0.05, pc1 = py * 0.05, pc2 = pz * 0.05;
  double q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = e[4 * i] * pc0 + e[4 * i + 1] * pc1 + e[4 * i + 2] * pc2 + e[4 * i + 3] * 1.0;
  const double* cov = e + 16;
  // non-zero columns / values of the rows of F = [q3 I | -skew(q)]
  const int col[3][3] = {{0, 4, 5}, {1, 3, 5}, {2, 3, 4}};
  const double val[3][3] = {{q[3], q[2], -q[1]}, {q[3], -q[2], q[0]}, {q[3], q[1], -q[0]}};
  double tr = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      double m = 0.0;
#pragma unroll
      for (int b = 0; b < 3; ++b) m += val[i][b] * (cov[6 * col[i][b] + col[i][a]] * 10000.0);
      tr += m * val[i][a];
    }
  }
  double fro = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) fro += (e[4 * i + j] * 0.1) * e[4 * i + j];
  return tr + fro;
}

struct MinMax4 { double umin, umax, tmin, tmax; uint32_t cnt; };

// order-preserving map double <-> uint64 (so that min/max can use integer atomics: exact and order-independent)
__host__ __device__ __forceinline__ unsigned long long dkey(double v) {
  unsigned long long b;
  memcpy(&b, &v, 8);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double dkey_inv(unsigned long long k) {
  const unsigned long long b = (k & 0x8000000000000000ull) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
  double v;
  memcpy(&v, &b, 8);
  return v;
}

__device__ __forceinline__ MinMax4 warp_reduce(MinMax4 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.umin = fmin(v.umin, __shfl_xor_sync(0xffffffffu, v.umin, o));
    v.umax = fmax(v.umax, __shfl_xor_sync(0xffffffffu, v.umax, o));
    v.tmin = fmin(v.tmin, __shfl_xor_sync(0xffffffffu, v.tmin, o));
    v.tmax = fmax(v.tmax, __shfl_xor_sync(0xffffffffu, v.tmax, o));
    v.cnt += __shfl_xor_sync(0xffffffffu, v.cnt, o);
  }
  return v;
}

// ---- K2a (search passes only): plane fit of the 5 neighbours.  esti_plane depends on the neighbours alone, not on
// the state, so its result is computed once per search and reused by the passes that re-use Nearest_Points
// (the reference recomputes it every pass, laserMapping.cpp:596, with the same outcome).
//   plane[p] = (n_x, n_y, n_z, d) ;  ucov[p] = plane_cov ;  sel[p] &= plane ok
__device__ __forceinline__ void fit_point(const float4* __restrict__ nodes, const float* __restrict__ node_cov, uint32_t N,
                                          const ParamConst& prm, const uint32_t* __restrict__ nn_idx,
                                          uint8_t* __restrict__ sel, float4* __restrict__ plane,
                                          double* __restrict__ ucov, uint32_t p) {
  float A[5][3], W[5];
#pragma unroll
  for (int j = 0; j < MALIO_K; ++j) {
    const uint32_t idx = nn_idx[(size_t)j * N + p];
    const float4 a = __ldg(nodes + idx);   // compact mirror of the snapshot: 16 B stride
    A[j][0] = a.x; A[j][1] = a.y; A[j][2] = a.z;
    W[j] = __ldg(node_cov + idx);
  }
  // esti_plane (common_lib.h:144-190)
  double cov_sum = 0.0, unit_cov = 0.0;
#pragma unroll
  for (int j = 0; j < MALIO_K; ++j) cov_sum += fabs(prm.cov_threshold - (double)W[j]);
  if ((double)W[0] > 0.00001) {
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j)
      unit_cov += ((prm.cov_threshold - (double)W[j]) / cov_sum) * ((prm.cov_threshold - (double)W[j]) / cov_sum) * (double)W[j];
  }
  float Aq[5][3];
#pragma unroll
  for (int j = 0; j < 5; ++j) { Aq[j][0] = A[j][0]; Aq[j][1] = A[j][1]; Aq[j][2] = A[j][2]; }
  float nv[3];
  qr_solve_5x3(Aq, nv);
  const float n = sqrtf(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
  const float pa = nv[0] / n, pb = nv[1] / n, pcn = nv[2] / n;
  const float pd = (float)(1.0 / (double)n);
  bool ok = true;
#pragma unroll
  for (int j = 0; j < MALIO_K; ++j)
    if (fabsf(pa * A[j][0] + pb * A[j][1] + pcn * A[j][2] + pd) > prm.plane_th) ok = false;
  plane[p] = make_float4(pa, pb, pcn, pd);
  ucov[p] = unit_cov;
  if (!ok) sel[p] = 0;
}
__global__ void __launch_bounds__(PLANE_THREADS)
fit_kernel(const float4* __restrict__ nodes, const float* __restrict__ node_cov, uint32_t N, ParamConst prm,
           const uint32_t* __restrict__ nn_idx, uint8_t* __restrict__ sel, float4* __restrict__ plane,
           double* __restrict__ ucov) {
  const uint32_t p = blockIdx.x * PLANE_THREADS + threadIdx.x;
  if (p >= N || !sel[p]) return;
  fit_point(nodes, node_cov, N, prm, nn_idx, sel, plane, ucov, p);
}

// ---- K2b (once per scan): point-wise uncertainty.  evalPointUncertainty depends on the point and its table entry
// only; the entry index is clamped differently for selected (:694-696) and non-selected (:737-739) points, so both
// traces are kept:  tau2[p] = (tau_selected, tau_not_selected).
__device__ __forceinline__ void tau_point(const malio_scan_pt& pt, const PassConst& pc, const double* __restrict__ table,
                                          double2* __restrict__ tau2, uint32_t p) {
  const int lid = pt.lidar;
  const int tsize = (int)(pc.table_off[lid + 1] - pc.table_off[lid]);
  const int ti = (int)pt.table_idx;
  const int ti_sel = (ti >= tsize) ? tsize - 2 : ti;
  const int ti_non = (ti >= tsize - 1) ? tsize - 2 : ti;
  const double t_sel = point_cov_trace(pt.x, pt.y, pt.z, table + (size_t)(pc.table_off[lid] + ti_sel) * TABLE_DOUBLES);
  const double t_non = (ti_non == ti_sel) ? t_sel
                       : point_cov_trace(pt.x, pt.y, pt.z, table + (size_t)(pc.table_off[lid] + ti_non) * TABLE_DOUBLES);
  tau2[p] = make_double2(t_sel, t_non);
}
__global__ void __launch_bounds__(PLANE_THREADS)
tau_kernel(const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm, uint32_t N, PassConst pc,
           const double* __restrict__ table, double2* __restrict__ tau2) {
  const uint32_t p = blockIdx.x * PLANE_THREADS + threadIdx.x;
  if (p >= N) return;
  const malio_scan_pt pt = pts[perm ? perm[p] : p];
  tau_point(pt, pc, table, tau2, p);
}

// ---- K2c (every pass): transform, point-to-plane residual, residual gate, min/max of the two weights.
// d_mmkey layout: dkey of {min_u, -max_u, min_tau, -max_tau}: one (integer) MIN all-reduce serves all four
struct GateOut { double u, tau; float pd2; int lid; bool selected; };
// one point of the gate: returns its contribution to the min/max of the two weights in mm
__device__ __forceinline__ void gate_point(const malio_scan_pt& pt, uint32_t p, const PassConst& pc,
                                           const float4* __restrict__ plane, const double* __restrict__ ucov,
                                           const double2* __restrict__ tau2, uint8_t* __restrict__ sel,
                                           float4* __restrict__ world, float* __restrict__ pd2_out, double* __restrict__ tau,
                                           float* __restrict__ normal_y, double* __restrict__ rows12,
                                           uint8_t* __restrict__ lid8, MinMax4& mm, double* __restrict__ srow = nullptr,
                                           GateOut* __restrict__ go = nullptr) {
  double b[3], m[3], g[3];
  transform_point(pc, pt.x, pt.y, pt.z, pt.lidar, b, m, g);
  const float wx = (float)g[0], wy = (float)g[1], wz = (float)g[2];
  world[p] = make_float4(wx, wy, wz, 0.f);
  bool selected = sel[p] != 0;
  if (selected) {
    const float4 pl = plane[p];
    const float pd2 = pl.x * wx + pl.y * wy + pl.z * wz + pl.w;                  // laserMapping.cpp:598
    const double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
    const float s = (float)(1 - 0.9 * (double)fabsf(pd2) / sqrt(nb));           // :599
    selected = (double)s > 0.1;
    pd2_out[p] = pd2;
    if (!selected) sel[p] = 0;
    if (selected) {
      // un-weighted Jacobian row, compact: [ n | A | B | C ]  (laserMapping.cpp:665-693)
      const int lid = pt.lidar;
      const double nvec[3] = {(double)pl.x, (double)pl.y, (double)pl.z};
      // C0 = R(s.rot)^T n (:676);  A = [m]x C0 (:677);  l = 0: C = C0, B = [b]x R(qE0)^T C (:683-684);
      // l != 0: C = R(qC_l)^T C0, B = [p]x R(qE_l)^T C (:687-690).  [v]x (R C) = v x (R C): evaluated as matrix-vector
      // products and cross products with FMAs — equal to the reference's (skew * R) * C to rounding (bar: 1e-9 on the system)
      double C[3], A[3], B[3] = {0.0, 0.0, 0.0};
      mat3_mul(pc.RsT, nvec, C);
      cross3_fma(m, C, A);
      double Cc[3] = {0.0, 0.0, 0.0};
      if (pc.ext_en) {
        double w[3];
        if (lid == 0) {
          mat3_mul(pc.ReT[0], C, w);
          cross3_fma(b, w, B);
        } else {
          double C2[3];
          mat3_mul(pc.RcT[lid], C, C2);
          C[0] = C2[0]; C[1] = C2[1]; C[2] = C2[2];
          mat3_mul(pc.ReT[lid], C, w);
          const double v[3] = {(double)pt.x, (double)pt.y, (double)pt.z};
          cross3_fma(v, w, B);
        }
        Cc[0] = C[0]; Cc[1] = C[1]; Cc[2] = C[2];
      }
      double2* dst = reinterpret_cast<double2*>(rows12 + (size_t)p * 12);
      dst[0] = make_double2(nvec[0], nvec[1]); dst[1] = make_double2(nvec[2], A[0]); dst[2] = make_double2(A[1], A[2]);
      dst[3] = make_double2(B[0], B[1]);       dst[4] = make_double2(B[2], Cc[0]);   dst[5] = make_double2(Cc[1], Cc[2]);
      lid8[p] = (uint8_t)lid;
      if (srow) {   // the fused pass keeps the row on chip across the min/max barrier
        srow[0] = nvec[0]; srow[1] = nvec[1]; srow[2] = nvec[2]; srow[3] = A[0]; srow[4] = A[1]; srow[5] = A[2];
        srow[6] = B[0]; srow[7] = B[1]; srow[8] = B[2]; srow[9] = Cc[0]; srow[10] = Cc[1]; srow[11] = Cc[2];
      }
      if (go) go->pd2 = pd2;
    }
  }
  const double2 t2 = tau2[p];
  if (go) { go->selected = selected; go->lid = pt.lidar; go->u = selected ? ucov[p] : 0.0; go->tau = t2.x; }
  if (selected) {
    const double u = ucov[p];
    mm.umin = fmin(mm.umin, u); mm.umax = fmax(mm.umax, u); mm.cnt += 1;
    if (pc.ext_en) {   // :694-703; with extrinsic_est_en == false R and normal_y are left untouched
      tau[p] = t2.x;
      normal_y[p] = (float)t2.x;
      mm.tmin = fmin(mm.tmin, t2.x); mm.tmax = fmax(mm.tmax, t2.x);
    }
  } else {
    normal_y[p] = (float)t2.y;   // :735-741
  }
}
// block-level min/max, then one integer atomicMin per quantity and block on the order-preserving keys:
// min/max are exact under any ordering, so this is deterministic without a serial fold.
template <int THREADS>
__device__ __forceinline__ void minmax_block_commit(MinMax4 mm, unsigned long long* __restrict__ d_mmkey,
                                                    uint32_t* __restrict__ d_cnt) {
  __shared__ MinMax4 s_w[THREADS / 32];
  mm = warp_reduce(mm);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = mm;
  __syncthreads();
  if (threadIdx.x == 0) {
    MinMax4 r = s_w[0];
    for (int w = 1; w < THREADS / 32; ++w) {
      r.umin = fmin(r.umin, s_w[w].umin); r.umax = fmax(r.umax, s_w[w].umax);
      r.tmin = fmin(r.tmin, s_w[w].tmin); r.tmax = fmax(r.tmax, s_w[w].tmax);
      r.cnt += s_w[w].cnt;
    }
    if (r.cnt) {
      atomicMin(d_mmkey + 0, dkey(r.umin)); atomicMin(d_mmkey + 1, dkey(-r.umax));
      atomicMin(d_mmkey + 2, dkey(r.tmin)); atomicMin(d_mmkey + 3, dkey(-r.tmax));
      atomicAdd(d_cnt, r.cnt);
    }
  }
}
__global__ void __launch_bounds__(GATE_THREADS)
gate_kernel(const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm, uint32_t N, PassConst pc,
            const float4* __restrict__ plane, const double* __restrict__ ucov, const double2* __restrict__ tau2,
            uint8_t* __restrict__ sel, float4* __restrict__ world, float* __restrict__ pd2_out,
            double* __restrict__ tau, float* __restrict__ normal_y, double* __restrict__ rows12,
            uint8_t* __restrict__ lid8, unsigned long long* __restrict__ d_mmkey, uint32_t* __restrict__ d_cnt) {
  const uint32_t p = blockIdx.x * GATE_THREADS + threadIdx.x;
  MinMax4 mm{1000.0, 0.0, 9999.0, 0.0, 0u};   // laserMapping.cpp:615-616, 646-647
  if (p < N) {
    const malio_scan_pt pt = pts[perm ? perm[p] : p];
    gate_point(pt, p, pc, plane, ucov, tau2, sel, world, pd2_out, tau, normal_y, rows12, lid8, mm);
  }
  minmax_block_commit<GATE_THREADS>(mm, d_mmkey, d_cnt);
}

// ------------------------------------------------------------------ K3: weights + fused H^T R^-1 [H | h] reduction
// The gate kernel leaves, per selected point, the un-weighted Jacobian row in compact form
//   J12 = [ n | [m]x C0 | B | C ]     (laserMapping.cpp:665-693; 12 of the 24 columns are non-zero)
// and the LiDAR id that says where B and C sit (columns 6+3l and 6+3(L+l)).  Here each row gets its plane weight
// a_i (:651-656) and noise rho_i (:716-721, clamp esekfom.hpp:624-626) and the block accumulates, per LiDAR l,
//     Gc_l = sum_{i in l} (a J12 / rho^)_a * [ a J12 | z | rho^ a J12_0..2 ]_b          (12 x 16, upper 4x4 blocks)
// i.e. esekfom.hpp:622-635 restricted to the non-zero columns (3.7x fewer FP64 operations than the dense 24 x 28
// form; FP64 issue is the limiter of this kernel).  The host scatters the three compact systems into the c x c one.
// The localization weight (a scalar, :745-759) factors out and is applied on the host.
__device__ __forceinline__ void point_weights(const ParamConst& prm, double u, double tau_i, int ext_en,
                                              double umin, double umax, double tmin, double tmax,
                                              double& a, double& rho) {
  // :651-656
  a = u;
  if (a == 0) a = 1;
  else if (umax == umin) a = (prm.plane_cov_max + prm.plane_cov_min) / 2;
  else a = 1 / ((prm.plane_cov_max - prm.plane_cov_min) * (a - umin) / (umax - umin) + prm.plane_cov_min);
  // :716-721 (FIC).  Degenerate 0/0 defined as mid-range (the reference yields NaN; SURVEY.md quirk 8)
  double R = ext_en ? tau_i : 0.0;
  if (R < tmin + (tmax - tmin) * prm.range_min) R = prm.point_cov_min;
  else if (R > tmin + (tmax - tmin) * prm.range_max) R = prm.point_cov_max;
  else {
    const double den = (prm.range_max - prm.range_min) * (tmax - tmin);
    if (den == 0.0) R = (prm.point_cov_max + prm.point_cov_min) / 2;
    else R = (prm.point_cov_max - prm.point_cov_min) * (R - (tmin + (tmax - tmin) * prm.range_min)) / den + prm.point_cov_min;
  }
  if (R < 0.0001) R = 0.001;   // esekfom.hpp:624-626
  rho = R;
}

// task t (0..8) -> upper-triangular 4x4 block (row group gi < 3, col group gj >= gi, gj < 4) of a 12 x 16 system
__device__ __forceinline__ void red_task(int t, int& gi, int& gj) {
  gi = (t >= 4) + (t >= 7);
  gj = t - (gi == 0 ? 0 : (gi == 1 ? 3 : 5));
}

// The body of the reduction for one block: tiles [tile_begin, tile_end) (contiguous, so that with the LiDAR-major
// internal order a block sees one LiDAR for many tiles), result in the block's slot.  Each of the 126 worker threads
// owns one 4x4 block (task) of the compact 12 x 16 system and every RED_KS-th row; its 16 accumulators stay in
// registers for as long as the LiDAR does not change and are folded over the row-splits (fixed order) into the slot
// only then.
__device__ __forceinline__ void reduce_flush(const double acc[16], bool worker, int l, double* __restrict__ s_flush,
                                             double* __restrict__ slot) {
  if (worker) {
#pragma unroll
    for (int k = 0; k < 16; ++k) s_flush[k * (RED_TASKS * RED_KS) + threadIdx.x] = acc[k];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < RED_TASKS * 16; e += RED_THREADS) {
    const int tk = e / 16, k = e % 16;
    double sum = 0.0;
#pragma unroll
    for (int q = 0; q < RED_KS; ++q) sum += s_flush[k * (RED_TASKS * RED_KS) + tk * RED_KS + q];
    slot[(l * RED_TASKS + tk) * 16 + k] += sum;
  }
  __syncthreads();
}
__device__ __forceinline__ void reduce_block(uint32_t N, const ParamConst& prm, int ext_en, const uint8_t* __restrict__ sel,
                                             const uint8_t* __restrict__ lid8, const double* __restrict__ rows12,
                                             const float* __restrict__ pd2v, const double* __restrict__ ucov,
                                             const double* __restrict__ tau, const unsigned long long* __restrict__ d_mm,
                                             uint32_t tile_begin, uint32_t tile_end, double* __restrict__ slot) {
  extern __shared__ double smem[];
  double* s_hs = smem;                                       // [128][RED_HS_STRIDE]  a J12 / rho^
  double* s_hx = s_hs + RED_THREADS * RED_HS_STRIDE;         // [128][RED_HX_STRIDE]  [a J12 | z | rho^ a J12_0..2]
  double* s_flush = s_hx + RED_THREADS * RED_HX_STRIDE;      // [16][RED_TASKS * RED_KS]  (entry-major: conflict-free)
  __shared__ uint32_t s_wcnt[MALIO_MAX_LIDAR][RED_THREADS / 32];
  __shared__ uint32_t s_seg[MALIO_MAX_LIDAR + 1];
  const int task = threadIdx.x / RED_KS, ks = threadIdx.x % RED_KS;
  const bool worker = task < RED_TASKS;
  int gi = 0, gj = 0;
  if (worker) red_task(task, gi, gj);
  for (int e = threadIdx.x; e < MALIO_RED_DOUBLES; e += RED_THREADS) slot[e] = 0.0;
  const double umin = dkey_inv(d_mm[0]), umax = -dkey_inv(d_mm[1]), tmin = dkey_inv(d_mm[2]), tmax = -dkey_inv(d_mm[3]);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t cnt_total = 0;
  int cur_l = -1;            // block-uniform: every thread derives it from s_seg
  double acc[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) acc[k] = 0.0;
  __syncthreads();
  for (uint32_t tile = tile_begin; tile < tile_end; ++tile) {
    // ---- phase A: weight this thread's row, then place it in the tile's LiDAR-sorted order
    const uint32_t p = tile * RED_THREADS + threadIdx.x;
    const bool ok = (p < N) && sel[p];
    const int l = ok ? (int)lid8[p] : -1;
    double h[12], z = 0.0, rho = 1.0, a = 0.0;
    if (ok) {
      point_weights(prm, ucov[p], ext_en ? tau[p] : 0.0, ext_en, umin, umax, tmin, tmax, a, rho);
      const double2* src = reinterpret_cast<const double2*>(rows12 + (size_t)p * 12);
#pragma unroll
      for (int k = 0; k < 6; ++k) { const double2 v = src[k]; h[2 * k] = v.x * a; h[2 * k + 1] = v.y * a; }   // :714
      z = ((-1) * (double)pd2v[p]) * a;                                                                  // :707,715
    }
    const uint32_t b0 = __ballot_sync(0xffffffffu, l == 0), b1 = __ballot_sync(0xffffffffu, l == 1),
                   b2 = __ballot_sync(0xffffffffu, l == 2);
    if (lane == 0) { s_wcnt[0][wid] = __popc(b0); s_wcnt[1][wid] = __popc(b1); s_wcnt[2][wid] = __popc(b2); }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t run = 0;
      for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
        s_seg[ll] = run;
        for (int w = 0; w < RED_THREADS / 32; ++w) { const uint32_t c = s_wcnt[ll][w]; s_wcnt[ll][w] = run; run += c; }
      }
      s_seg[MALIO_MAX_LIDAR] = run;
    }
    __syncthreads();
    if (ok) {
      const uint32_t bal = l == 0 ? b0 : (l == 1 ? b1 : b2);
      const uint32_t dst = s_wcnt[l][wid] + __popc(bal & ((1u << lane) - 1u));
      double* hs = s_hs + dst * RED_HS_STRIDE;
      double* hx = s_hx + dst * RED_HX_STRIDE;
      const double inv_rho = 1.0 / rho;   // HT(:,i) / R_i (esekfom.hpp:627) as a multiply: <= 1 ulp per term
#pragma unroll
      for (int k = 0; k < 12; ++k) { hs[k] = h[k] * inv_rho; hx[k] = h[k]; }
      hx[12] = z; hx[13] = rho * h[0]; hx[14] = rho * h[1]; hx[15] = rho * h[2];
    }
    __syncthreads();
    cnt_total += s_seg[MALIO_MAX_LIDAR];
    // ---- phase B: per LiDAR segment, 9 block tasks x RED_KS row-splits
#pragma unroll 1
    for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
      const uint32_t beg = s_seg[ll], end = s_seg[ll + 1];
      if (beg == end) continue;
      if (ll != cur_l) {
        if (cur_l >= 0) reduce_flush(acc, worker, cur_l, s_flush, slot);
        cur_l = ll;
#pragma unroll
        for (int k = 0; k < 16; ++k) acc[k] = 0.0;
      }
      if (worker) {
        for (uint32_t q = beg + ks; q < end; q += RED_KS) {
          const double* aa = s_hs + q * RED_HS_STRIDE + 4 * gi;
          const double* bb = s_hx + q * RED_HX_STRIDE + 4 * gj;
          const double a0 = aa[0], a1 = aa[1], a2 = aa[2], a3 = aa[3];
          const double c0 = bb[0], c1 = bb[1], c2 = bb[2], c3 = bb[3];
          acc[0] = fma(a0, c0, acc[0]);   acc[1] = fma(a0, c1, acc[1]);   acc[2] = fma(a0, c2, acc[2]);   acc[3] = fma(a0, c3, acc[3]);
          acc[4] = fma(a1, c0, acc[4]);   acc[5] = fma(a1, c1, acc[5]);   acc[6] = fma(a1, c2, acc[6]);   acc[7] = fma(a1, c3, acc[7]);
          acc[8] = fma(a2, c0, acc[8]);   acc[9] = fma(a2, c1, acc[9]);   acc[10] = fma(a2, c2, acc[10]); acc[11] = fma(a2, c3, acc[11]);
          acc[12] = fma(a3, c0, acc[12]); acc[13] = fma(a3, c1, acc[13]); acc[14] = fma(a3, c2, acc[14]); acc[15] = fma(a3, c3, acc[15]);
        }
      }
    }
    __syncthreads();   // the staging area is rewritten by the next tile
  }
  if (cur_l >= 0) reduce_flush(acc, worker, cur_l, s_flush, slot);
  if (threadIdx.x == 0) { slot[MALIO_RED_BLOCKS * 16] = (double)cnt_total; slot[MALIO_RED_BLOCKS * 16 + 1] = 0.0; }
}
// contiguous tile range of block b when n_tiles are dealt to `grid` blocks (the host picks grid = ceil(n_tiles / per_block))
__device__ __forceinline__ void block_tiles(uint32_t n_tiles, uint32_t& t0, uint32_t& t1) {
  const uint32_t per_block = (n_tiles + gridDim.x - 1) / gridDim.x;
  t0 = blockIdx.x * per_block;
  t1 = t0 + per_block < n_tiles ? t0 + per_block : n_tiles;
  if (t0 > n_tiles) t0 = n_tiles;
}
__global__ void __launch_bounds__(RED_THREADS)
reduce_kernel(uint32_t N, ParamConst prm, int ext_en, const uint8_t* __restrict__ sel, const uint8_t* __restrict__ lid8,
              const double* __restrict__ rows12, const float* __restrict__ pd2v, const double* __restrict__ ucov,
              const double* __restrict__ tau, const unsigned long long* __restrict__ d_mm, uint32_t n_tiles,
              double* __restrict__ block_red) {
  uint32_t t0, t1;
  block_tiles(n_tiles, t0, t1);
  reduce_block(N, prm, ext_en, sel, lid8, rows12, pd2v, ucov, tau, d_mm, t0, t1, block_red + (size_t)blockIdx.x * MALIO_RED_DOUBLES);
}

// ------------------------------------------------------------------ one measurement pass in ONE cooperative launch
// K2 + K3 fused (single-GPU path):  [tau once per scan] [plane fit once per search] gate -> grid barrier -> weights +
// H^T R^-1 [H|h] accumulation -> grid barrier -> distributed fixed-order fold, written both to device memory and straight
// into pinned, mapped host memory, followed by a sequence flag the host spins on.  Compared with the three launches +
// D2H copy + stream synchronisation it replaces, this removes every launch gap and the copy/sync latency from the
// per-pass critical path; arithmetic and summation order are unchanged (bit-identical results).
// The kernel is launched with cudaLaunchCooperativeKernel (all blocks co-resident), the barriers are plain
// device-scope counters that only ever grow (the host passes the value they had before the launch).
// Multi-GPU: the two exchanges of a pass (MIN of the four min/max keys before the weights, SUM of the reduced system at
// the end) go through per-rank mailboxes in device memory that every peer maps with CUDA IPC and writes over
// NVLink/NVSwitch from inside pass_kernel — no NCCL call, no extra launch, the cross-GPU latency of a pass is two
// one-way store + flag hops.  Layout of one rank's mailbox: [parity 2][kind: MIN 64 B | SUM 3584 B][source rank 8].
struct PeerArgs {
  unsigned char* mail[MAIL_MAX_WORLD];   // mail[r] = rank r's mailbox as mapped into THIS process (mail[rank] is local)
  int rank, world;
};
__device__ __forceinline__ unsigned char* mail_min_slot(unsigned char* box, uint32_t seq, int src) {
  return box + (seq & 1u) * MAIL_PARITY_BYTES + src * MAIL_MIN_BYTES;
}
__device__ __forceinline__ unsigned char* mail_sum_slot(unsigned char* box, uint32_t seq, int src) {
  return box + (seq & 1u) * MAIL_PARITY_BYTES + MAIL_MAX_WORLD * MAIL_MIN_BYTES + src * MAIL_SUM_BYTES;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// spin until *p == want; gives up after ~2 s (a peer that never launched) and reports it
__device__ __forceinline__ bool wait_seq_sys(const uint32_t* p, uint32_t want) {
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (uint32_t it = 0;; ++it) {
    if (ld_acquire_sys_u32(p) == want) return true;
    if ((it & 0xFFFu) == 0xFFFu) {
      unsigned long long t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > 2000000000ull) return false;
    }
  }
}
struct PassArgs {
  const malio_scan_pt* pts; const uint32_t* perm; uint32_t N;
  const double* table; const float4* nodes; const float* node_cov; const uint32_t* nn_idx;
  uint8_t* sel; float4* world; float4* plane; double* ucov; double2* tau2; float* pd2; double* tau; float* normal_y;
  double* rows12; uint8_t* lid8;
  int do_tau, do_fit;
  unsigned long long *mmkey, *mmkey_next; uint32_t *cnt_cell, *cnt_next, *gstats;
  uint32_t* bar;           // [0] barrier 1 arrivals, [1] barrier 2 arrivals, [2] folded entries  (monotone), [3] release flag of barrier 1 (multi-GPU)
  PeerArgs peer;
  uint32_t bar_base[3];
  uint32_t n_tiles;
  double* block_red; double* d_res;
  double* h_res;           // mapped host memory: MALIO_RED_DOUBLES result | 4 min/max keys | flag
  uint32_t seq;
  unsigned long long* dbg; // optional [grid][8] %globaltimer stamps at the phase boundaries (MALIO_PASS_TRACE=1)
  unsigned long long* xwait;   // multi-GPU: [0] ns spent in the MIN exchange (push + wait for every peer), [1] same for the SUM exchange, [2] passes
};
__device__ __forceinline__ void pass_stamp(const PassArgs& a, int k) {
  if (a.dbg && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    a.dbg[(size_t)blockIdx.x * 8 + k] = t;
  }
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// all threads of all blocks call this; returns when `expected` arrivals have been counted
// Gives up after ~2 s (a block of the grid that never became resident) and raises the fault word of the mapped result buffer,
// which measure() reports.
__device__ __forceinline__ void grid_barrier(uint32_t* counter, uint32_t target, uint32_t* fault) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned long long t0 = 0;
    for (uint32_t it = 0; (int32_t)(ld_acquire_u32(counter) - target) < 0; ++it) {
      if ((it & 0x3FFFu) == 0x3FFFu) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t0 == 0) t0 = t1;
        else if (t1 - t0 > 2000000000ull) { *reinterpret_cast<volatile uint32_t*>(fault) = 2u; break; }
      }
    }
  }
  __syncthreads();
}
// FAST: every block owns at most PASS_FAST_TILES tiles and keeps their Jacobian rows in shared memory from the gate to
// the accumulation (no global round trip, no staging pass); rows stay in their own positions and the workers pick the
// rows of the LiDAR they are accumulating by a per-row tag, so no prefix sums or compaction barriers are needed.
// !FAST: any number of tiles per block, rows go through global memory (reduce_block).
#ifndef MALIO_PASS_TILES
#define MALIO_PASS_TILES 2
#endif
#ifndef MALIO_PASS_MINB
#define MALIO_PASS_MINB 4
#endif
constexpr int PASS_FAST_TILES = MALIO_PASS_TILES;   // tiles of 128 points a block keeps on chip (fast path)
constexpr int PASS_MIN_BLOCKS = MALIO_PASS_MINB;    // co-resident blocks per SM the kernel is compiled for
constexpr int PASS_ROW_STRIDE = 15;        // doubles per staged row: a*J12 (12) | 1/rho^ | z | rho^   (odd: conflict-free)
constexpr int PASS_FAST_SMEM_DOUBLES = PASS_FAST_TILES * RED_THREADS * PASS_ROW_STRIDE + RED_TASKS * RED_KS * 16;
static_assert(PASS_FAST_SMEM_DOUBLES <= RED_SMEM_DOUBLES, "the fast path must fit the generic path's shared memory");
template <bool FAST>
__global__ void __launch_bounds__(RED_THREADS, FAST ? PASS_MIN_BLOCKS : 4)
pass_kernel(PassArgs a, PassConst pc, ParamConst prm) {
  uint32_t t0, t1;
  block_tiles(a.n_tiles, t0, t1);
  extern __shared__ double smem[];
  // FAST: rows stay in their own slots; per (tile, LiDAR) the slots that hold a row are listed (compacted) so that the
  // accumulation loop runs over rows of one LiDAR only, every lane busy
  __shared__ uint8_t s_list[PASS_FAST_TILES * RED_THREADS];
  __shared__ uint16_t s_wc[PASS_FAST_TILES][MALIO_MAX_LIDAR][RED_THREADS / 32];   // selected rows per tile, LiDAR, warp
  GateOut go[PASS_FAST_TILES];
  uint32_t bal[PASS_FAST_TILES];   // ballot of this thread's LiDAR within its warp (FAST)
  pass_stamp(a, 0);
  // ---- phase 1: per point, same tile -> block mapping as the accumulation below
  {
    MinMax4 mm{1000.0, 0.0, 9999.0, 0.0, 0u};   // laserMapping.cpp:615-616, 646-647
#pragma unroll
    for (int k = 0; k < (FAST ? PASS_FAST_TILES : 1); ++k) go[k].selected = false;
    if (FAST) {
#pragma unroll
      for (int k = 0; k < PASS_FAST_TILES; ++k) {
        const uint32_t tile = t0 + k;
        const uint32_t p = tile * RED_THREADS + threadIdx.x;
        if (tile < t1 && p < a.N) {
          const malio_scan_pt pt = a.pts[a.perm ? a.perm[p] : p];
          if (a.do_tau) tau_point(pt, pc, a.table, a.tau2, p);
          if (a.do_fit && a.sel[p]) fit_point(a.nodes, a.node_cov, a.N, prm, a.nn_idx, a.sel, a.plane, a.ucov, p);
          gate_point(pt, p, pc, a.plane, a.ucov, a.tau2, a.sel, a.world, a.pd2, a.tau, a.normal_y, a.rows12, a.lid8, mm,
                     smem + (size_t)(k * RED_THREADS + threadIdx.x) * PASS_ROW_STRIDE, &go[k]);
        }
        const int l = go[k].selected ? go[k].lid : -1;
        const uint32_t b0 = __ballot_sync(0xffffffffu, l == 0), b1 = __ballot_sync(0xffffffffu, l == 1),
                       b2 = __ballot_sync(0xffffffffu, l == 2);
        bal[k] = l == 0 ? b0 : (l == 1 ? b1 : b2);
        if ((threadIdx.x & 31) == 0) {
          s_wc[k][0][threadIdx.x >> 5] = (uint16_t)__popc(b0); s_wc[k][1][threadIdx.x >> 5] = (uint16_t)__popc(b1);
          s_wc[k][2][threadIdx.x >> 5] = (uint16_t)__popc(b2);
        }
      }
    } else {
      for (uint32_t tile = t0; tile < t1; ++tile) {
        const uint32_t p = tile * RED_THREADS + threadIdx.x;
        if (p < a.N) {
          const malio_scan_pt pt = a.pts[a.perm ? a.perm[p] : p];
          if (a.do_tau) tau_point(pt, pc, a.table, a.tau2, p);
          if (a.do_fit && a.sel[p]) fit_point(a.nodes, a.node_cov, a.N, prm, a.nn_idx, a.sel, a.plane, a.ucov, p);
          gate_point(pt, p, pc, a.plane, a.ucov, a.tau2, a.sel, a.world, a.pd2, a.tau, a.normal_y, a.rows12, a.lid8, mm);
        }
      }
    }
    minmax_block_commit<RED_THREADS>(mm, a.mmkey, a.cnt_cell);
  }
  pass_stamp(a, 1);
  if (a.peer.world <= 1) {
    grid_barrier(a.bar + 0, a.bar_base[0] + gridDim.x, reinterpret_cast<uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9));
  } else {
    // barrier 1 fused with the cross-GPU MIN: every block arrives; warp 0 of block 0 waits for the local arrivals, pushes
    // this GPU's four keys into every peer's mailbox, waits for the peers' keys, writes the global minima into the local
    // key cell and only then releases the local blocks
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); atomicAdd(a.bar + 0, 1u); }
    if (blockIdx.x == 0 && threadIdx.x < 32) {
      const int lane = threadIdx.x, me = a.peer.rank, W = a.peer.world;
      if (lane == 0) while ((int32_t)(ld_acquire_u32(a.bar + 0) - (a.bar_base[0] + gridDim.x)) < 0) { }
      __syncwarp();
      unsigned long long xw0 = 0;
      if (lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xw0));
      unsigned long long k[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) k[c] = __ldcg(a.mmkey + c);
      bool ok = true;
      if (lane < W && lane != me) {
        unsigned char* dst = mail_min_slot(a.peer.mail[lane], a.seq, me);
        volatile unsigned long long* dk = reinterpret_cast<volatile unsigned long long*>(dst);
#pragma unroll
        for (int c = 0; c < 4; ++c) dk[c] = k[c];
        st_release_sys_u32(reinterpret_cast<uint32_t*>(dst + 40), a.seq);
        const unsigned char* src = mail_min_slot(a.peer.mail[me], a.seq, lane);
        ok = wait_seq_sys(reinterpret_cast<const uint32_t*>(src + 40), a.seq);
        const volatile unsigned long long* sk = reinterpret_cast<const volatile unsigned long long*>(src);
#pragma unroll
        for (int c = 0; c < 4; ++c) k[c] = sk[c];
      } else if (lane >= W) {
#pragma unroll
        for (int c = 0; c < 4; ++c) k[c] = ~0ull;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int c = 0; c < 4; ++c) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, k[c], o); k[c] = v < k[c] ? v : k[c]; }
      }
      const bool all_ok = __all_sync(0xffffffffu, ok);
      if (lane == 0) {
        unsigned long long xw1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xw1));
        a.xwait[0] += xw1 - xw0;      // only this thread of this GPU ever writes these words
        a.xwait[2] += 1;
#pragma unroll
        for (int c = 0; c < 4; ++c) a.mmkey[c] = k[c];
        if (!all_ok) *reinterpret_cast<volatile uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9) = 1u;   // peer timeout
        __threadfence();
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.bar + 3), "r"(a.seq) : "memory");
      }
    }
    if (threadIdx.x == 0) while (ld_acquire_u32(a.bar + 3) != a.seq) { }
    __syncthreads();
  }
  pass_stamp(a, 2);
  if (blockIdx.x == 0 && threadIdx.x == 0) {   // arm the other parity's min/max cell for the next pass
    a.mmkey_next[0] = dkey(1000.0); a.mmkey_next[1] = dkey(-0.0);
    a.mmkey_next[2] = dkey(9999.0); a.mmkey_next[3] = dkey(-0.0);
    *a.cnt_next = 0;
    a.gstats[2] = 0; a.gstats[4] = 0;
  }
  // ---- phase 2: weights + accumulation into this block's slot
  double* slot = a.block_red + (size_t)blockIdx.x * MALIO_RED_DOUBLES;
  if (FAST) {
    double* s_flush = smem + PASS_FAST_TILES * RED_THREADS * PASS_ROW_STRIDE;
    const double umin = dkey_inv(a.mmkey[0]), umax = -dkey_inv(a.mmkey[1]), tmin = dkey_inv(a.mmkey[2]), tmax = -dkey_inv(a.mmkey[3]);
    uint32_t mine = 0;
    // segment table of the block: seg[k][l] = [beg, end) inside tile k's list (every thread derives it from s_wc)
    uint32_t seg_beg[PASS_FAST_TILES][MALIO_MAX_LIDAR], seg_end[PASS_FAST_TILES][MALIO_MAX_LIDAR];
#pragma unroll
    for (int k = 0; k < PASS_FAST_TILES; ++k) {
      uint32_t run = 0;
#pragma unroll
      for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
        seg_beg[k][l] = run;
#pragma unroll
        for (int w = 0; w < RED_THREADS / 32; ++w) run += s_wc[k][l][w];
        seg_end[k][l] = run;
      }
    }
#pragma unroll
    for (int k = 0; k < PASS_FAST_TILES; ++k) {
      if (go[k].selected) {
        double aw, rho;
        point_weights(prm, go[k].u, pc.ext_en ? go[k].tau : 0.0, pc.ext_en, umin, umax, tmin, tmax, aw, rho);
        double* row = smem + (size_t)(k * RED_THREADS + threadIdx.x) * PASS_ROW_STRIDE;
#pragma unroll
        for (int c = 0; c < 12; ++c) row[c] = row[c] * aw;                       // laserMapping.cpp:714
        row[12] = 1.0 / rho;   // HT(:,i) / R_i (esekfom.hpp:627) as a multiply: <= 1 ulp per term
        row[13] = ((-1) * (double)go[k].pd2) * aw;                               // :707,715
        row[14] = rho;
        // compacted position of this row among the tile's rows of its LiDAR
        const int l = go[k].lid, wid = threadIdx.x >> 5;
        uint32_t pos = l == 0 ? seg_beg[k][0] : (l == 1 ? seg_beg[k][1] : seg_beg[k][2]);
        for (int w = 0; w < wid; ++w) pos += s_wc[k][l][w];
        pos += __popc(bal[k] & ((1u << (threadIdx.x & 31)) - 1u));
        s_list[k * RED_THREADS + pos] = (uint8_t)threadIdx.x;
        ++mine;
      }
    }
    __shared__ uint32_t s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    if (mine) atomicAdd(&s_cnt, mine);
    const int task = threadIdx.x / RED_KS, ks = threadIdx.x % RED_KS;
    const bool worker = task < RED_TASKS;
    int gi = 0, gj = 0;
    if (worker) red_task(task, gi, gj);
    // thread e < 144 ends up holding entry (task e / 16, element e % 16) of each LiDAR's compact system, e >= 128 wraps
    // onto threads 0..15 as a second entry: two result registers per LiDAR and thread
    double res0[MALIO_MAX_LIDAR], res1[MALIO_MAX_LIDAR];
#pragma unroll
    for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
      res0[ll] = 0.0; res1[ll] = 0.0;
      if (ll < pc.L) {
        double acc[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) acc[k] = 0.0;
        if (worker) {
#pragma unroll
          for (int k = 0; k < PASS_FAST_TILES; ++k) {
            for (uint32_t i = seg_beg[k][ll] + ks; i < seg_end[k][ll]; i += RED_KS) {
              const uint32_t q = k * RED_THREADS + s_list[k * RED_THREADS + i];
              const double* row = smem + (size_t)q * PASS_ROW_STRIDE;
              const double ir = row[12];
              const double a0 = row[4 * gi] * ir, a1 = row[4 * gi + 1] * ir, a2 = row[4 * gi + 2] * ir, a3 = row[4 * gi + 3] * ir;
              double c0, c1, c2, c3;
              if (gj < 3) { c0 = row[4 * gj]; c1 = row[4 * gj + 1]; c2 = row[4 * gj + 2]; c3 = row[4 * gj + 3]; }
              else { const double rho = row[14]; c0 = row[13]; c1 = rho * row[0]; c2 = rho * row[1]; c3 = rho * row[2]; }
              acc[0] = fma(a0, c0, acc[0]);   acc[1] = fma(a0, c1, acc[1]);   acc[2] = fma(a0, c2, acc[2]);   acc[3] = fma(a0, c3, acc[3]);
              acc[4] = fma(a1, c0, acc[4]);   acc[5] = fma(a1, c1, acc[5]);   acc[6] = fma(a1, c2, acc[6]);   acc[7] = fma(a1, c3, acc[7]);
              acc[8] = fma(a2, c0, acc[8]);   acc[9] = fma(a2, c1, acc[9]);   acc[10] = fma(a2, c2, acc[10]); acc[11] = fma(a2, c3, acc[11]);
              acc[12] = fma(a3, c0, acc[12]); acc[13] = fma(a3, c1, acc[13]); acc[14] = fma(a3, c2, acc[14]); acc[15] = fma(a3, c3, acc[15]);
            }
          }
#pragma unroll
          for (int k = 0; k < 16; ++k) s_flush[k * (RED_TASKS * RED_KS) + threadIdx.x] = acc[k];
        }
        __syncthreads();
        {   // fold the RED_KS row-splits in a fixed order
          const int e0 = threadIdx.x, e1 = threadIdx.x + RED_THREADS;
          double sum = 0.0;
#pragma unroll
          for (int q = 0; q < RED_KS; ++q) sum += s_flush[(e0 % 16) * (RED_TASKS * RED_KS) + (e0 / 16) * RED_KS + q];
          res0[ll] = sum;
          if (e1 < RED_TASKS * 16) {
            sum = 0.0;
#pragma unroll
            for (int q = 0; q < RED_KS; ++q) sum += s_flush[(e1 % 16) * (RED_TASKS * RED_KS) + (e1 / 16) * RED_KS + q];
            res1[ll] = sum;
          }
        }
        __syncthreads();
      }
    }
#pragma unroll
    for (int ll = 0; ll < MALIO_MAX_LIDAR; ++ll) {
      slot[ll * RED_TASKS * 16 + threadIdx.x] = res0[ll];
      if (threadIdx.x + RED_THREADS < RED_TASKS * 16) slot[ll * RED_TASKS * 16 + threadIdx.x + RED_THREADS] = res1[ll];
    }
    if (threadIdx.x == 0) { slot[MALIO_RED_BLOCKS * 16] = (double)s_cnt; slot[MALIO_RED_BLOCKS * 16 + 1] = 0.0; }
  } else {
    reduce_block(a.N, prm, pc.ext_en, a.sel, a.lid8, a.rows12, a.pd2, a.ucov, a.tau, a.mmkey, t0, t1, slot);
  }
  pass_stamp(a, 3);
  grid_barrier(a.bar + 1, a.bar_base[1] + gridDim.x, reinterpret_cast<uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9));
  pass_stamp(a, 4);
  // ---- phase 3: fold the slots, one warp per entry, in fold_kernel's order
  const uint32_t lane = threadIdx.x & 31u, wpb = RED_THREADS / 32;
  uint32_t folded = 0;
  for (uint32_t e = blockIdx.x * wpb + (threadIdx.x >> 5); e < MALIO_RED_DOUBLES; e += gridDim.x * wpb) {
    double sum = 0.0;
    for (uint32_t bk = lane; bk < gridDim.x; bk += 32) sum += a.block_red[(size_t)bk * MALIO_RED_DOUBLES + e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) a.d_res[e] = sum;
    ++folded;
  }
  if (folded) {   // warp-uniform
    uint32_t done = 0;
    if (lane == 0) {
      __threadfence();
      done = atomicAdd(a.bar + 2, folded) + folded;
    }
    done = __shfl_sync(0xffffffffu, done, 0);
    if (done == a.bar_base[2] + MALIO_RED_DOUBLES) {
      // this warp folded the last entry: ship result + min/max keys to the mapped host buffer (posted PCIe writes, one
      // system-scope fence), then the sequence flag the host is spinning on
      __threadfence();
      if (a.peer.world > 1) {
        // cross-GPU SUM: this GPU's folded system goes into slot [me] of every mailbox (its own included), then the
        // slots of all ranks are added in rank order — the same order on every GPU, so all ranks hold identical bits
        const int me = a.peer.rank, W = a.peer.world;
        unsigned long long xs0 = 0;
        if (lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xs0));
        // payload with ordinary (weak) stores: they pipeline over NVLink; the system-scope fence + the release flag below publish
        // them.  (volatile = strong system-scope stores cost ~0.5 us EACH here: 17 us per pass at N = 2, ~60 us at N = 8.)
        {
          double v[(MALIO_RED_DOUBLES + 31) / 32];
#pragma unroll
          for (uint32_t j = 0; j < (MALIO_RED_DOUBLES + 31) / 32; ++j) { const uint32_t e = lane + 32 * j; v[j] = e < MALIO_RED_DOUBLES ? __ldcg(a.d_res + e) : 0.0; }
          for (int r = 0; r < W; ++r) {
            double* dst = reinterpret_cast<double*>(mail_sum_slot(a.peer.mail[r], a.seq, me));
#pragma unroll
            for (uint32_t j = 0; j < (MALIO_RED_DOUBLES + 31) / 32; ++j) { const uint32_t e = lane + 32 * j; if (e < MALIO_RED_DOUBLES) dst[e] = v[j]; }
          }
        }
        __threadfence_system();
        __syncwarp();
        bool ok = true;
        if ((int)lane < W && (int)lane != me) {
          st_release_sys_u32(reinterpret_cast<uint32_t*>(mail_sum_slot(a.peer.mail[lane], a.seq, me) + MAIL_SUM_SEQ_OFF), a.seq);
          ok = wait_seq_sys(reinterpret_cast<const uint32_t*>(mail_sum_slot(a.peer.mail[me], a.seq, (int)lane) + MAIL_SUM_SEQ_OFF), a.seq);
        }
        if (!__all_sync(0xffffffffu, ok) && lane == 0) *reinterpret_cast<volatile uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 9) = 1u;
        if (lane == 0) {
          unsigned long long xs1;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(xs1));
          a.xwait[1] += xs1 - xs0;    // the last-folding warp of the grid: one writer per pass
        }
        __syncwarp();     // every lane's peer has published (acquire loads above); L2 is the coherence point for the peers' writes
        for (uint32_t e = lane; e < MALIO_RED_DOUBLES; e += 32) {
          double sum = 0.0;
          for (int r = 0; r < W; ++r) sum += __ldcg(reinterpret_cast<const double*>(mail_sum_slot(a.peer.mail[me], a.seq, r)) + e);
          a.d_res[e] = sum;
          a.h_res[e] = sum;
        }
      } else {
        for (uint32_t e = lane; e < MALIO_RED_DOUBLES; e += 32) a.h_res[e] = __ldcg(a.d_res + e);
      }
      if (lane < 4) reinterpret_cast<unsigned long long*>(a.h_res + MALIO_RED_DOUBLES)[lane] = a.mmkey[lane];
      // k-NN list statistics of the last search as knn_list_kernel published them ([3] traversal list, [5] 5x5x5 retries)
      if (lane == 4) { uint32_t* hg = reinterpret_cast<uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 4); hg[3] = a.gstats[3]; hg[5] = a.gstats[5]; hg[6] = g_fault_word; hg[7] = a.gstats[7]; }
      __threadfence_system();
      __syncwarp();
      if (lane == 0) *reinterpret_cast<volatile uint32_t*>(a.h_res + MALIO_RED_DOUBLES + 8) = a.seq;
    }
  }
  pass_stamp(a, 5);
}

// second stage: one warp per entry of the reduced system folds the per-block slots in a fixed order
// (lane-strided partial sums, then a shuffle tree) -> bit-reproducible result, no FP64 atomics
__global__ void __launch_bounds__(256)
fold_kernel(const double* __restrict__ block_red, uint32_t n_slots, double* __restrict__ d_res,
            unsigned long long* __restrict__ next_mmkey, uint32_t* __restrict__ next_cnt, uint32_t* __restrict__ gstats) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {   // arm the other parity's min/max cell for the next pass
    gstats[2] = 0; gstats[4] = 0;              // and the k-NN fast path's unsettled / ring-2 counters
    next_mmkey[0] = dkey(1000.0); next_mmkey[1] = dkey(-0.0);    // laserMapping.cpp:615-616
    next_mmkey[2] = dkey(9999.0); next_mmkey[3] = dkey(-0.0);    // :646-647
    *next_cnt = 0;
  }
  const uint32_t e = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (e >= MALIO_RED_DOUBLES) return;
  double s = 0.0;
  for (uint32_t bk = lane; bk < n_slots; bk += 32) s += block_red[(size_t)bk * MALIO_RED_DOUBLES + e];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) d_res[e] = s;
}

// rows for the degenerate branch (esekfom.hpp:574-582): the first `cap` selected points in position order, one
// block; rows are written in the padded 24-column layout + z, un-weighted by the localization weight
__global__ void rows_kernel(uint32_t N, ParamConst prm, int ext_en, const uint8_t* __restrict__ sel,
                            const uint8_t* __restrict__ lid8, const double* __restrict__ rows12,
                            const float* __restrict__ pd2v, const double* __restrict__ ucov,
                            const double* __restrict__ tau, const unsigned long long* __restrict__ d_mm, uint32_t cap,
                            double* __restrict__ rows /* cap x 25 */, uint32_t* __restrict__ n_rows) {
  __shared__ uint32_t s_base;
  __shared__ uint32_t s_wcnt[32];
  if (threadIdx.x == 0) s_base = 0;
  const double umin = dkey_inv(d_mm[0]), umax = -dkey_inv(d_mm[1]), tmin = dkey_inv(d_mm[2]), tmax = -dkey_inv(d_mm[3]);
  __syncthreads();
  for (uint32_t start = 0; start < N; start += blockDim.x) {
    const uint32_t p = start + threadIdx.x;
    const bool ok = (p < N) && sel[p];
    const uint32_t bal = __ballot_sync(0xffffffffu, ok);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) s_wcnt[w] = __popc(bal);
    __syncthreads();
    uint32_t off = s_base;
    for (int k = 0; k < w; ++k) off += s_wcnt[k];
    off += __popc(bal & ((1u << lane) - 1u));
    if (ok && off < cap) {
      double a, rho;
      point_weights(prm, ucov[p], ext_en ? tau[p] : 0.0, ext_en, umin, umax, tmin, tmax, a, rho);
      const int l = lid8[p];
      double* o = rows + (size_t)off * 25;
      for (int k = 0; k < 24; ++k) o[k] = 0.0;
      const double* j = rows12 + (size_t)p * 12;
      for (int k = 0; k < 6; ++k) o[k] = j[k] * a;
      for (int k = 0; k < 3; ++k) { o[6 + 3 * l + k] = j[6 + k] * a; o[15 + 3 * l + k] = j[9 + k] * a; }
      o[24] = ((-1) * (double)pd2v[p]) * a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t tot = 0;
      for (int k = 0; k < (int)(blockDim.x >> 5); ++k) tot += s_wcnt[k];
      s_base += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *n_rows = s_base;
    rows[(size_t)MALIO_MAX_DOF * 25] = (double)(s_base < cap ? s_base : cap);   // count travels with the rows (multi-rank gather)
  }
}

// per-scan state back to "nothing searched yet": point_selected_surf = 0, normal_y = 0, Nearest_Points empty, k-NN list
// counters 0 — one launch instead of four memsets (this sits at the head of every scan)
__global__ void reset_scan_kernel(uint32_t cap, uint8_t* __restrict__ sel, float* __restrict__ normal_y,
                                  uint32_t* __restrict__ nn_idx, uint32_t* __restrict__ gstats) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 4) gstats[2 + i] = 0;
  if (i < cap) {
    sel[i] = 0;
    normal_y[i] = 0.f;
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) nn_idx[(size_t)j * cap + i] = 0xFFFFFFFFu;
  }
}
// ------------------------------------------------------------------ next to the path: map_incremental's decision
// laserMapping.cpp:398-446 per point, from device-resident data: normal_y and Nearest_Points (indices into the snapshot)
// of the last pass, the scan point and the state after the update.  pointBodyToWorld (:134-147) has its own operation
// order (no detour through the LiDAR-0 frame), restated exactly by body_to_world (malio_device.cuh).  Outputs in caller order.
__global__ void map_incr_kernel(const malio_scan_pt* __restrict__ pts, const uint32_t* __restrict__ perm, uint32_t N,
                                PassConst pc, const float4* __restrict__ mpts, const uint32_t* __restrict__ nn_idx,
                                const float* __restrict__ normal_y, double cov_threshold, double fs, int ekf_inited,
                                uint8_t* __restrict__ cls_out, float* __restrict__ world_out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const uint32_t i = perm ? perm[p] : p;
  uint8_t cls = MALIO_MAP_SKIP;
  float w[3] = {0.f, 0.f, 0.f};
  if (!((double)normal_y[p] > cov_threshold)) {                                                 // :406
    const malio_scan_pt pt = pts[p];
    body_to_world(pc, pt.lidar, pt.x, pt.y, pt.z, w);                                           // :134-147
    uint32_t id[MALIO_K];
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) { id[j] = nn_idx[(size_t)j * N + p]; cnt += id[j] != 0xFFFFFFFFu; }
    if (cnt > 0 && ekf_inited) {                                                                // :411
      float mid[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) mid[k] = (float)(floor((double)w[k] / fs) * fs + 0.5 * fs);   // :417-419
      const float dist = (w[0] - mid[0]) * (w[0] - mid[0]) + (w[1] - mid[1]) * (w[1] - mid[1]) + (w[2] - mid[2]) * (w[2] - mid[2]);
      const float4 n0 = __ldg(mpts + id[0]);
      if ((double)fabsf(n0.x - mid[0]) > 0.5 * fs && (double)fabsf(n0.y - mid[1]) > 0.5 * fs && (double)fabsf(n0.z - mid[2]) > 0.5 * fs) {
        cls = MALIO_MAP_ADD_NO_DOWNSAMPLE;                                                      // :421-425
      } else {
        bool need_add = true;
        if (cnt >= MALIO_K) {                                                                   // :428-429
#pragma unroll
          for (int j = 0; j < MALIO_K; ++j) {
            const float4 q = __ldg(mpts + id[j]);
            const float dj = (q.x - mid[0]) * (q.x - mid[0]) + (q.y - mid[1]) * (q.y - mid[1]) + (q.z - mid[2]) * (q.z - mid[2]);
            if (need_add && dj < dist) need_add = false;                                        // :430-434
          }
        }
        cls = need_add ? MALIO_MAP_ADD : MALIO_MAP_DROP;
      }
    } else {
      cls = MALIO_MAP_ADD;                                                                      // :439-440
    }
  }
  cls_out[i] = cls;
  if (world_out) { world_out[3 * (size_t)i] = w[0]; world_out[3 * (size_t)i + 1] = w[1]; world_out[3 * (size_t)i + 2] = w[2]; }
}

// position space -> caller order
__global__ void scatter_aux_kernel(const uint32_t* __restrict__ perm, uint32_t N, const float* __restrict__ normal_y,
                                   const uint32_t* __restrict__ nn_idx, const float* __restrict__ nn_d2,
                                   const uint8_t* __restrict__ sel, const float4* __restrict__ world,
                                   float* __restrict__ o_ny, uint32_t* __restrict__ o_idx, float* __restrict__ o_d2,
                                   uint8_t* __restrict__ o_sel, float* __restrict__ o_world) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const uint32_t i = perm ? perm[p] : p;
  if (o_ny) o_ny[i] = normal_y[p];
  if (o_sel) o_sel[i] = sel[p];
  if (o_world) { const float4 w = world[p]; o_world[3 * (size_t)i] = w.x; o_world[3 * (size_t)i + 1] = w.y; o_world[3 * (size_t)i + 2] = w.z; }
  if (o_idx) {
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) o_idx[(size_t)i * MALIO_K + j] = nn_idx[(size_t)j * N + p];
  }
  if (o_d2) {
#pragma unroll
    for (int j = 0; j < MALIO_K; ++j) o_d2[(size_t)i * MALIO_K + j] = nn_d2[(size_t)j * N + p];
  }
}

// ------------------------------------------------------------------ NCCL through dlopen (no link-time dependency)
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool load(std::string& err) {
    if (lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
    if (!lib) { err = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return false; }
    GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
    AllReduce = (decltype(AllReduce))dlsym(lib, "ncclAllReduce");
    AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
    CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
    GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllReduce || !CommDestroy) { err = "NCCL symbols missing"; return false; }
    return true;
  }
};
NcclApi g_nccl;

PassConst make_pass_const(const malio_handle* h, const DeviceState* D, const malio_pass_state* s) {
  PassConst pc{};
  std::memcpy(pc.rot, s->rot, sizeof(pc.rot));
  std::memcpy(pc.pos, s->pos, sizeof(pc.pos));
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
    std::memcpy(pc.eq[l], s->ext[l].q, sizeof(pc.eq[l]));
    std::memcpy(pc.et[l], s->ext[l].t, sizeof(pc.et[l]));
    std::memcpy(pc.cq[l], D->tcomp[l].q, sizeof(pc.cq[l]));
    std::memcpy(pc.ct[l], D->tcomp[l].t, sizeof(pc.ct[l]));
  }
  for (int l = 0; l <= MALIO_MAX_LIDAR; ++l) pc.table_off[l] = D->table_off[l];
  auto conj_R = [](const double q[4], double R[9]) {   // Eigen's toRotationMatrix of the conjugate, row-major
    const double w = q[0], x = -q[1], y = -q[2], z = -q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
  };
  conj_R(pc.rot, pc.RsT);
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) { conj_R(pc.eq[l], pc.ReT[l]); conj_R(pc.cq[l], pc.RcT[l]); }
  pc.L = h->cfg.params.n_lidar;
  pc.ext_en = h->cfg.params.extrinsic_est_en;
  return pc;
}
ParamConst make_param_const(const malio_params& p) {
  ParamConst c{};
  c.plane_th = p.plane_th; c.knn_max_sqdist = p.knn_max_sqdist;
  c.cov_threshold = p.cov_threshold; c.point_cov_max = p.point_cov_max; c.point_cov_min = p.point_cov_min;
  c.plane_cov_max = p.plane_cov_max; c.plane_cov_min = p.plane_cov_min; c.range_min = p.range_min; c.range_max = p.range_max;
  return c;
}

// queries per warp for knn_kernel: halve the logical warp width while fewer than ~8 warps per SM would be resident
int pick_lanes(uint32_t n, int sm_count) {
  const uint64_t target = (uint64_t)sm_count * 8;
  int lanes = 32;
  while (lanes > 4 && (n + lanes - 1) / lanes < target) lanes >>= 1;
  return lanes;
}
uint32_t knn_blocks(uint32_t n, int lanes) {
  const uint32_t warps = (n + lanes - 1) / lanes;
  return (warps + KNN_THREADS / 32 - 1) / (KNN_THREADS / 32);
}

// blocks in one wave of the fused pass's FAST variant: its co-resident blocks, capped at the slots for the per-block
// systems (red_grid).  measure() and the sort's LiDAR-major switch derive the launch from it.
static uint32_t fast_wave(const DeviceState* D) {
  return (D->pass_max_blocks > 0 && (uint32_t)D->pass_max_blocks < D->red_grid) ? (uint32_t)D->pass_max_blocks : D->red_grid;
}

// keys + counting sort of n queries into D->d_perm (MODE 0: scan points through pc, MODE 1: D->d_queries)
template <int MODE>
int sort_queries(malio_handle* h, DeviceState* D, uint32_t n, const PassConst& pc) {
  cudaStream_t st = D->stream;
  CUDA_TRY(cudaMemsetAsync(D->d_hist, 0, SORT_BINS * sizeof(uint32_t), st));
  // LiDAR-major keys exactly where the fused pass leaves its FAST variant (more than PASS_FAST_TILES tiles per block)
  const int lid_major = (MODE == 0 && (uint64_t)n > (uint64_t)PASS_FAST_TILES * RED_THREADS * (uint64_t)fast_wave(D)) ? 1 : 0;
  count_kernel<MODE><<<(n + 255) / 256, 256, 0, st>>>(D->d_pts, D->d_queries, n, pc, lid_major, D->d_keys16, D->d_hist);
  scan_kernel<<<SCAN_BLOCKS, SCAN_THREADS, 0, st>>>(D->d_hist, D->d_offs, D->d_cursor, D->d_btot);
  // d_fb_list (the k-NN hand-over list, filled only later in the pass) doubles as the arrival-slot array of the sort
  scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(D->d_keys16, n, D->d_offs, D->d_btot, D->d_cursor, D->d_tmp_ids, D->d_fb_list);
  rank_kernel<<<(n + 255) / 256, 256, 0, st>>>(D->d_keys16, n, D->d_offs, D->d_btot, D->d_hist, D->d_tmp_ids, D->d_fb_list, D->d_perm,
                                               MODE == 0 ? D->d_pts : nullptr, MODE == 0 ? D->d_pts_sorted : nullptr);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 4;
  return MALIO_OK;
}


// ---- cell-list index: geometry from the snapshot root (its point + both children's boxes bound every live point)
constexpr uint32_t GRID_MAX_CELLS = 1u << 25;
bool grid_geometry(const malio_map_node* nodes, uint32_t n, float hcell, GridConst& G) {
  if (n == 0 || !(hcell > 0.f)) return false;
  const malio_map_node& r = nodes[0];
  float lo[3] = {r.x, r.y, r.z}, hi[3] = {r.x, r.y, r.z};
  auto grow = [&](const float* b) {
    for (int a = 0; a < 3; ++a) { lo[a] = std::fmin(lo[a], b[2 * a]); hi[a] = std::fmax(hi[a], b[2 * a + 1]); }
  };
  if (r.link & MALIO_LINK_HAS_LEFT) grow(r.lbox);
  if (r.link & MALIO_LINK_HAS_RIGHT) grow(r.rbox);
  for (int a = 0; a < 3; ++a) if (!std::isfinite(lo[a]) || !std::isfinite(hi[a])) return false;
  for (int it = 0; it < 64; ++it) {
    const float inv = 1.0f / hcell;
    double dims[3];
    for (int a = 0; a < 3; ++a) dims[a] = std::floor((double)((hi[a] - lo[a]) * inv)) + 1.0;
    const double cells = (dims[0] + 2 * GRID_PAD) * (dims[1] + 2 * GRID_PAD) * (dims[2] + 2 * GRID_PAD);
    if (cells + 1 <= (double)GRID_MAX_CELLS && dims[0] < 4000 && dims[1] < 4000 && dims[2] < 4000) {
      G.ox = lo[0]; G.oy = lo[1]; G.oz = lo[2]; G.inv_h = inv; G.h = hcell;
      G.nx = (int)dims[0]; G.ny = (int)dims[1]; G.nz = (int)dims[2];
      G.px = G.nx + 2 * GRID_PAD; G.py = G.ny + 2 * GRID_PAD;
      G.ncell = (uint32_t)cells;
      return true;
    }
    hcell *= 1.26f;
  }
  return false;
}

// (re)build the index for the snapshot resident in D->d_nodes; leaves {occupied cells, live points} in D->h_gstats
int grid_build(malio_handle* h, DeviceState* D, const GridConst& G) {
  cudaStream_t st = D->stream;
  const uint32_t n = D->n_nodes;
  const uint32_t ncell_pad = ((G.ncell + 1 + GRID_CHUNK - 1) / GRID_CHUNK) * GRID_CHUNK, nchunk = ncell_pad / GRID_CHUNK;
  if (ncell_pad > D->cap_cells) {
    if (int rc = ensure(h, D->d_cell_start, (size_t)ncell_pad)) return rc;
    if (int rc = ensure(h, D->d_cell_cnt, (size_t)ncell_pad)) return rc;
    if (!D->d_ctot) { if (int rc = ensure(h, D->d_ctot, 8192)) return rc; if (int rc = ensure(h, D->d_cbase, 8192)) return rc; }
    D->cap_cells = ncell_pad;
  }
  if (D->cap_nodes > D->cap_cell_pts) {
    if (int rc = ensure(h, D->d_cell_of, (size_t)D->cap_nodes)) return rc;
    if (int rc = ensure(h, D->d_cell_pts, (size_t)D->cap_nodes)) return rc;
    D->cap_cell_pts = D->cap_nodes;
  }
  CUDA_TRY(cudaMemsetAsync(D->d_cell_cnt, 0, (size_t)ncell_pad * sizeof(uint32_t), st));
  CUDA_TRY(cudaMemsetAsync(D->d_gstats, 0, 2 * sizeof(uint32_t), st));
  grid_count_kernel<<<(n + 255) / 256, 256, 0, st>>>(D->d_mpts, n, G, D->d_cell_cnt, D->d_cell_of);
  grid_scan_local_kernel<<<nchunk, 1024, 0, st>>>(D->d_cell_cnt, D->d_cell_start, D->d_ctot, D->d_gstats);
  grid_scan_tot_kernel<<<1, 1024, 0, st>>>(D->d_ctot, nchunk, D->d_cbase, D->d_gstats);
  grid_scan_add_kernel<<<nchunk, 1024, 0, st>>>(D->d_cell_start, D->d_cbase);
  grid_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(D->d_mpts, n, D->d_cell_of, D->d_cell_start, D->d_cell_cnt, D->d_cell_pts);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(D->h_gstats, D->d_gstats, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  D->ctr.kernel_launches += 5;
  D->grid = G;
  return MALIO_OK;
}

// lanes per query of the cell-list scan: small searches are latency-bound (one warp's chain), large ones issue-bound (the merge and
// the replicated preamble are pure overhead there).
static int pick_group(uint32_t n, int sm_count) {
  const uint64_t per_sm = (uint64_t)n / (uint64_t)(sm_count > 0 ? sm_count : 1);
  if (per_sm <= 256) return 4;        // <= ~34k queries on 132 SMs
  if (per_sm <= 1280) return 2;       // <= ~169k
  return 1;                           // knn_direct_kernel
}

// the k-NN of one search pass: cell-list fast path + exact ikd-Tree-order traversal for what it leaves, or the
// traversal alone when the index is off
template <int MODE>
int run_knn(malio_handle* h, DeviceState* D, uint32_t n, const malio_scan_pt* pts_in, const uint32_t* perm,
            const PassConst& pc, float max_sqdist) {
  cudaStream_t st = D->stream;
  const bool smem_stack = D->depth + KNN_POP_WIDTH <= (uint32_t)KNN_SMEM_DEPTH;
  const malio_scan_pt* pts = MODE == 0 ? pts_in : nullptr;
  const float* qs = MODE == 0 ? nullptr : D->d_queries;
  float4* world = MODE == 0 ? D->d_world : nullptr;
  uint8_t* sel = MODE == 0 ? D->d_sel : nullptr;
  auto need_boxes = [&]() -> int {   // the exact traversal reads the 64-byte records: wait for a rebuild still in flight
    if (D->refit_pending) { CUDA_TRY(cudaStreamWaitEvent(st, D->ev_refit, 0)); D->refit_pending = false; }
    return MALIO_OK;
  };
  if (D->grid_on) {
    // d_gstats: [2] traversal-list length, [4] ring-2 list length (both zeroed by the previous pass / the re-arm)
    const int grp = pick_group(n, D->sm_count);
    if (grp > 1) {
#define MALIO_LAUNCH_KEYS(GG, PP)                                                                                                \
  do {                                                                                                                         \
    const uint32_t qpb = GD_THREADS / GG;                                                                                      \
    knn_keys_kernel<MODE, GG, PP><<<(n + qpb - 1) / qpb, GD_THREADS, 0, st>>>(                                                 \
        D->d_cell_pts, D->d_cell_start, D->grid, pts, perm, qs, n, pc, max_sqdist, world, D->d_nn_idx, D->d_nn_d2, sel,        \
        D->d_gstats + 4, D->d_fb_list, D->d_gstats + 2, D->timing ? D->d_cand : nullptr);                                      \
  } while (0)
      // measured (ncu kernel time, C2 sub-sampled): 12.5k queries 31 -> 12 us with 4 lanes + row preload; 100k 29.5 -> 24 us with
      // 2 lanes; from ~200k queries on (C4, C5) the thread-per-query kernel is as fast or faster and stays
      if (grp == 2) MALIO_LAUNCH_KEYS(2, false);
      else MALIO_LAUNCH_KEYS(4, true);
#undef MALIO_LAUNCH_KEYS
    } else {
      knn_direct_kernel<MODE><<<(n + GD_THREADS - 1) / GD_THREADS, GD_THREADS, 0, st>>>(
          D->d_cell_pts, D->d_cell_start, D->grid, pts, perm, qs, n, pc, max_sqdist, world, D->d_nn_idx, D->d_nn_d2, sel,
          D->d_gstats + 4, D->d_fb_list, D->d_gstats + 2, D->timing ? D->d_cand : nullptr);
    }
    // 8 queries per warp and iteration; at most one resident wave of 64-thread blocks
    uint32_t fb_blocks = (n + 15) / 16;
    const uint32_t wave = (uint32_t)D->sm_count * 2;   // the list is usually (near) empty: a small grid walks it by stride
    if (fb_blocks > wave) fb_blocks = wave;
    if (D->tree_free) {   // device-resident map: no tree to walk, the open queries are settled on the cell list itself
      knn_ring_kernel<MODE><<<fb_blocks, KNN_THREADS, 0, st>>>(D->d_cell_pts, D->d_cell_start, D->grid, pts, perm, qs, n, pc, max_sqdist,
                                                             D->d_fb_list, D->d_gstats + 2, D->d_nn_idx, D->d_nn_d2, sel, D->d_gstats + 3,
                                                             D->d_gstats + 7);
      D->ctr.kernel_launches += 2;
      CUDA_TRY(cudaGetLastError());
      return MALIO_OK;
    }
    if (int rc = need_boxes()) return rc;
    if (smem_stack)
      knn_list_kernel<MODE, true><<<fb_blocks, KNN_THREADS, 0, st>>>(D->d_nodes, D->n_nodes, pts, perm, qs, n, pc, max_sqdist,
                                                                    D->d_fb_list, D->d_gstats + 2, D->d_nn_idx, D->d_nn_d2, sel, D->d_gstats + 3);
    else
      knn_list_kernel<MODE, false><<<fb_blocks, KNN_THREADS, 0, st>>>(D->d_nodes, D->n_nodes, pts, perm, qs, n, pc, max_sqdist,
                                                                     D->d_fb_list, D->d_gstats + 2, D->d_nn_idx, D->d_nn_d2, sel, D->d_gstats + 3);
    D->ctr.kernel_launches += 2;
  } else {
    // device-resident map without a live point: n_nodes = 0, the traversal below answers with empty lists as for an empty snapshot
    if (D->tree_free && D->n_nodes > 0) { h->err = "device-resident map: the cell-list index is required (map extent too large for it?)"; return MALIO_ERR_STATE; }
    if (int rc = need_boxes()) return rc;
    const int lanes = pick_lanes(n, D->sm_count);
    if (smem_stack)
      knn_kernel<MODE, true><<<knn_blocks(n, lanes), KNN_THREADS, 0, st>>>(D->d_nodes, D->n_nodes, pts, perm, qs, n, lanes, pc,
                                                                          max_sqdist, world, D->d_nn_idx, D->d_nn_d2, sel);
    else
      knn_kernel<MODE, false><<<knn_blocks(n, lanes), KNN_THREADS, 0, st>>>(D->d_nodes, D->n_nodes, pts, perm, qs, n, lanes, pc,
                                                                           max_sqdist, world, D->d_nn_idx, D->d_nn_d2, sel);
    D->ctr.kernel_launches += 1;
  }
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}

}  // namespace

// =================================================================== host-facing entry points
namespace malio_dev {

int create(malio_handle* h) {
  DeviceState* D = new DeviceState;
  h->dev = D;
  D->device = h->cfg.device;
  int ndev = 0;
  CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (ndev <= 0 || D->device >= ndev) { h->err = "no such CUDA device"; return MALIO_ERR_CUDA; }
  CUDA_TRY(cudaSetDevice(D->device));
  cudaDeviceProp prop{};
  CUDA_TRY(cudaGetDeviceProperties(&prop, D->device));
  D->sm_count = prop.multiProcessorCount;
  CUDA_TRY(cudaStreamCreateWithFlags(&D->stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&D->stream2, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&D->stream3, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_h2d, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_refit, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_cov, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_sorted, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&D->ev_tau, cudaEventDisableTiming));
  for (auto& e : D->ev) CUDA_TRY(cudaEventCreate(&e));
  CUDA_TRY(cudaMalloc((void**)&D->d_counters, 8 * sizeof(uint32_t)));
  CUDA_TRY(cudaMemset(D->d_counters, 0, 8 * sizeof(uint32_t)));
  CUDA_TRY(cudaMalloc((void**)&D->d_mmkey, 8 * sizeof(unsigned long long)));
  {
    const unsigned long long init[8] = {dkey(1000.0), dkey(-0.0), dkey(9999.0), dkey(-0.0), dkey(1000.0), dkey(-0.0), dkey(9999.0), dkey(-0.0)};
    CUDA_TRY(cudaMemcpy(D->d_mmkey, init, sizeof(init), cudaMemcpyHostToDevice));
  }
  CUDA_TRY(cudaMalloc((void**)&D->d_res, MALIO_RED_DOUBLES * sizeof(double)));
  CUDA_TRY(cudaMalloc((void**)&D->d_cand, 4 * sizeof(unsigned long long)));   // [0] candidates, [1..3] multi-GPU exchange waits (ns, ns, passes)
  CUDA_TRY(cudaMemset(D->d_cand, 0, 4 * sizeof(unsigned long long)));
  CUDA_TRY(cudaMalloc((void**)&D->d_gstats, 8 * sizeof(uint32_t)));
  CUDA_TRY(cudaMemset(D->d_gstats, 0, 8 * sizeof(uint32_t)));
  CUDA_TRY(cudaMalloc((void**)&D->d_hist, SORT_BINS * sizeof(uint32_t)));
  CUDA_TRY(cudaMalloc((void**)&D->d_offs, SORT_BINS * sizeof(uint32_t)));
  CUDA_TRY(cudaMalloc((void**)&D->d_cursor, SORT_BINS * sizeof(uint32_t)));
  CUDA_TRY(cudaMalloc((void**)&D->d_btot, SCAN_BLOCKS * sizeof(uint32_t)));
  CUDA_TRY(cudaMemset(D->d_hist, 0, SORT_BINS * sizeof(uint32_t)));
  CUDA_TRY(cudaMalloc((void**)&D->d_rows, (size_t)ROWS_DOUBLES * (1 + MAIL_MAX_WORLD) * sizeof(double)));   // own rows | gathered rows of all ranks
  D->red_grid = (uint32_t)D->sm_count * (PASS_MIN_BLOCKS > 4 ? PASS_MIN_BLOCKS : 4);   // slots for the per-block partial systems
  CUDA_TRY(cudaMalloc((void**)&D->d_block_red, (size_t)D->red_grid * MALIO_RED_DOUBLES * sizeof(double)));
  // pinned + mapped: [0, RED) result | +0..3 min/max keys | +4..7 k-NN list statistics | +8 pass sequence flag | +16.. rows
  CUDA_TRY(cudaHostAlloc((void**)&D->h_res, (MALIO_RED_DOUBLES + 16 + MALIO_MAX_DOF * 25) * sizeof(double), cudaHostAllocMapped));
  std::memset(D->h_res, 0, (MALIO_RED_DOUBLES + 16) * sizeof(double));
  CUDA_TRY(cudaHostGetDevicePointer((void**)&D->h_res_dev, D->h_res, 0));
  CUDA_TRY(cudaMalloc((void**)&D->d_bar, 4 * sizeof(uint32_t)));
  CUDA_TRY(cudaMemset(D->d_bar, 0, 4 * sizeof(uint32_t)));
  CUDA_TRY(cudaFuncSetAttribute(pass_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RED_SMEM_DOUBLES * (int)sizeof(double)));
  CUDA_TRY(cudaFuncSetAttribute(pass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, RED_SMEM_DOUBLES * (int)sizeof(double)));
  {
    int per_sm = 0, per_sm2 = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pass_kernel<true>, RED_THREADS, PASS_FAST_SMEM_DOUBLES * sizeof(double)));
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, pass_kernel<false>, RED_THREADS, RED_SMEM_DOUBLES * sizeof(double)));
    D->pass_max_blocks_generic = per_sm2 * D->sm_count;
    int coop = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, D->device));
    D->pass_max_blocks = per_sm * D->sm_count;
    D->fused = coop && per_sm > 0;
    if (const char* e = getenv("MALIO_FUSED_PASS")) D->fused = D->fused && atoi(e) != 0;
    if (const char* e = getenv("MALIO_PASS_TRACE")) D->trace_passes = atoi(e);
    if (const char* e = getenv("MALIO_KNN_CELL")) { D->env_knn_cell = (float)atof(e); D->env_knn_cell_set = true; }
    D->host_prof = getenv("MALIO_HOST_PROF") != nullptr;
  }
  D->h_gstats = reinterpret_cast<uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 4);
  std::memset(D->h_gstats, 0, 8 * sizeof(uint32_t));
  CUDA_TRY(cudaFuncSetAttribute(reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                RED_SMEM_DOUBLES * (int)sizeof(double)));
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) { D->tcomp[l] = malio_rigid{{1, 0, 0, 0}, {0, 0, 0}}; }
  return MALIO_OK;
}

void destroy(malio_handle* h) {
  DeviceState* D = (DeviceState*)h->dev;
  if (!D) return;
  malio_pre::destroy(h);
  malio_map::destroy(h);
  if (D->d_ids) cudaFree(D->d_ids);
  if (D->host_prof && D->host_passes)
    fprintf(stderr, "[malio] passes %llu: host launch %.1f us/pass, host wait-for-device %.1f us/pass\n",
            (unsigned long long)D->host_passes, D->host_launch_us / D->host_passes, D->host_wait_us / D->host_passes);
  cudaSetDevice(D->device);
  if (D->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(D->comm);
  void* ptrs[] = {D->d_nodes, D->d_cov, D->d_mpts, D->d_parent, D->d_arrived, D->d_pts, D->d_pts_sorted, D->d_perm, D->d_keys16, D->d_hist, D->d_offs, D->d_cursor, D->d_btot, D->d_tmp_ids,
                  D->d_table, D->d_nn_idx, D->d_nn_d2, D->d_sel, D->d_world, D->d_plane, D->d_ucov, D->d_tau, D->d_tau2, D->d_pd2, D->d_rows12, D->d_lid8,
                  D->d_normal_y, D->d_o_ny, D->d_o_idx, D->d_o_d2, D->d_o_sel, D->d_o_world, D->d_block_mm,
                  D->d_block_cnt, D->d_counters, D->d_mmkey, D->d_block_red, D->d_res, D->d_rows, D->d_queries,
                  D->d_cell_start, D->d_cell_cnt, D->d_cell_of, D->d_ctot, D->d_cbase, D->d_cell_pts, D->d_fb_list, D->d_gstats, D->d_bar, D->d_cand};
  for (void* p : ptrs) if (p) cudaFree(p);
  if (D->h_res) cudaFreeHost(D->h_res);
  for (auto& e : D->ev) if (e) cudaEventDestroy(e);
  if (D->stream2) { cudaStreamSynchronize(D->stream2); cudaStreamDestroy(D->stream2); }
  if (D->stream3) { cudaStreamSynchronize(D->stream3); cudaStreamDestroy(D->stream3); }
  if (D->ev_h2d) cudaEventDestroy(D->ev_h2d);
  if (D->ev_refit) cudaEventDestroy(D->ev_refit);
  if (D->ev_cov) cudaEventDestroy(D->ev_cov);
  if (D->ev_sorted) cudaEventDestroy(D->ev_sorted);
  if (D->ev_tau) cudaEventDestroy(D->ev_tau);
  if (D->stream) cudaStreamDestroy(D->stream);
  delete D;
  h->dev = nullptr;
}

static int ensure_map_buffers(malio_handle* h, DeviceState* D, uint32_t n) {
  if (n <= D->cap_nodes && D->d_nodes) return MALIO_OK;   // (slot mode grows d_mpts / d_cov only: no tree records there)
  uint32_t cap = n + n / 8 + 1024;
  if (cap < h->cfg.max_map_nodes) cap = h->cfg.max_map_nodes;
  if (int rc = ensure(h, D->d_nodes, (size_t)cap * 4)) return rc;
  if (int rc = ensure(h, D->d_mpts, (size_t)cap)) return rc;
  if (int rc = ensure(h, D->d_cov, (size_t)cap)) return rc;
  if (int rc = ensure(h, D->d_parent, (size_t)cap)) return rc;
  if (int rc = ensure(h, D->d_arrived, (size_t)cap)) return rc;
  D->cap_nodes = cap;
  D->cap_slots = 0;        // d_mpts / d_cov now hold the snapshot: the next malio_map_build re-creates the slot storage (grow_slots)
  return MALIO_OK;
}

// after the snapshot is resident (d_nodes, d_mpts, d_cov): cell-list index for the k-NN fast path.
// Cell edge: cfg.knn_cell_size (> 0 fixed, < 0 index off, 0 automatic: start at 1 m = twice the reference's map voxel,
// filter_size_map 0.5, and keep 2..9 live points per occupied cell).  root = host copy of node 0 (bounds every live point).
static int finish_map_upload(malio_handle* h, DeviceState* D, const malio_map_node* root, uint32_t n, uint32_t depth) {
  D->n_nodes = n; D->depth = depth;
  {
    const uint32_t zero = 0;
    CUDA_TRY(cudaMemcpyToSymbolAsync(g_fault_word, &zero, sizeof(zero), 0, cudaMemcpyHostToDevice, D->stream));
    D->h_gstats[6] = 0;
  }
  float hcfg = h->cfg.knn_cell_size;
  if (D->env_knn_cell_set) hcfg = D->env_knn_cell;
  D->grid_on = false;
  if (hcfg >= 0.f && n > 0) {
    const bool automatic = hcfg == 0.f;
    float hc = automatic ? (D->grid_h > 0.f ? D->grid_h : 1.0f) : hcfg;
    // A tuned edge from an earlier upload is re-used as is: one build, no host round trip in the middle of the upload;
    // its occupancy statistics arrive with the final synchronisation and steer the NEXT upload (maps change slowly).
    const int attempts = (automatic && D->grid_h == 0.f) ? 6 : 1;
    for (int attempt = 0; attempt < attempts; ++attempt) {
      GridConst G{};
      if (!grid_geometry(root, n, hc, G)) break;
      if (int rc = grid_build(h, D, G)) return rc;
      D->grid_on = true;
      D->grid_h = G.h;
      if (attempts == 1) break;
      CUDA_TRY(cudaStreamSynchronize(D->stream));
      if (D->h_gstats[0] == 0) break;
      const double mean = (double)D->h_gstats[1] / (double)D->h_gstats[0];
      if (mean < 2.0) hc = G.h * 1.5f;
      else if (mean > 9.0 && G.h > 0.05f) hc = G.h / 1.5f;
      else break;
    }
  }
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  if (D->grid_on && hcfg == 0.f && D->h_gstats[0] != 0) {   // steer the next upload
    const double mean = (double)D->h_gstats[1] / (double)D->h_gstats[0];
    if (mean < 2.0) D->grid_h *= 1.5f;
    else if (mean > 9.0 && D->grid_h > 0.05f) D->grid_h /= 1.5f;
  }
  D->map_ready = true;
  return MALIO_OK;
}

int upload_map(malio_handle* h, const malio_map_node* nodes, const float* cov, uint32_t n, uint32_t depth) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (depth > MALIO_MAX_TREE_DEPTH) { h->err = "snapshot deeper than MALIO_MAX_TREE_DEPTH"; return MALIO_ERR_TREE_TOO_DEEP; }
  if (D->refit_pending) { CUDA_TRY(cudaStreamSynchronize(D->stream2)); D->refit_pending = false; }
  if (int rc = ensure_map_buffers(h, D, n)) return rc;
  D->tree_free = false;
  malio_map::leave(h);
  CUDA_TRY(cudaMemcpyAsync(D->d_nodes, nodes, (size_t)n * sizeof(malio_map_node), cudaMemcpyHostToDevice, D->stream));
  CUDA_TRY(cudaMemcpyAsync(D->d_cov, cov, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, D->stream));
  if (n) {
    tree_extract_kernel<<<(n + 255) / 256, 256, 0, D->stream>>>(D->d_nodes, n, D->d_mpts);
    D->ctr.kernel_launches += 1;
  }
  D->ctr.h2d_bytes += (uint64_t)n * (sizeof(malio_map_node) + sizeof(float));
  return finish_map_upload(h, D, nodes, n, depth);
}

int upload_map_compact(malio_handle* h, const malio_map_point* pts, const float* cov, uint32_t n, uint32_t depth,
                       const float* root_box) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (depth > MALIO_MAX_TREE_DEPTH) { h->err = "snapshot deeper than MALIO_MAX_TREE_DEPTH"; return MALIO_ERR_TREE_TOO_DEEP; }
  if (D->refit_pending) { CUDA_TRY(cudaStreamSynchronize(D->stream2)); D->refit_pending = false; }
  if (int rc = ensure_map_buffers(h, D, n)) return rc;
  D->tree_free = false;
  malio_map::leave(h);
  static_assert(sizeof(malio_map_point) == sizeof(float4), "compact record is one float4");
  CUDA_TRY(cudaMemcpyAsync(D->d_mpts, pts, (size_t)n * sizeof(malio_map_point), cudaMemcpyHostToDevice, D->stream));
  CUDA_TRY(cudaEventRecord(D->ev_h2d, D->stream));
  // the map-side weights (only the plane fit reads them) follow on a copy stream of their own: their copy overlaps the cell-list
  // build that starts on the first stream as soon as the points are there
  CUDA_TRY(cudaStreamWaitEvent(D->stream3, D->ev_h2d, 0));
  CUDA_TRY(cudaMemcpyAsync(D->d_cov, cov, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, D->stream3));
  CUDA_TRY(cudaEventRecord(D->ev_cov, D->stream3));
  D->ctr.h2d_bytes += (uint64_t)n * (sizeof(malio_map_point) + sizeof(float));
  malio_map_node root{};
  if (n) {
    // Rebuild the 64-byte records (children's boxes) on the device.  Only the exact traversal reads them (tie / outlier
    // queries, index-off mode), so the rebuild runs on a second stream beside the cell-list build and the scan's first
    // kernels; whoever needs the records waits on ev_refit (run_knn, download_map_nodes).
    CUDA_TRY(cudaStreamWaitEvent(D->stream2, D->ev_h2d, 0));
    CUDA_TRY(cudaMemsetAsync(D->d_arrived, 0, (size_t)n * sizeof(uint32_t), D->stream2));
    tree_init_kernel<<<(n + 255) / 256, 256, 0, D->stream2>>>(D->d_mpts, n, D->d_nodes, D->d_parent);
    tree_refit_kernel<<<(n + 255) / 256, 256, 0, D->stream2>>>(D->d_mpts, n, D->d_nodes, D->d_parent, D->d_arrived);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(D->ev_refit, D->stream2));
    D->refit_pending = true;
    D->ctr.kernel_launches += 2;
    if (root_box) {   // the caller knows the map's bounding box (the ikd-Tree root's node_range_*): no read-back needed
      root.x = root_box[0]; root.y = root_box[2]; root.z = root_box[4];
      root.link = MALIO_LINK_HAS_LEFT;
      for (int k = 0; k < 6; ++k) root.lbox[k] = root_box[k];
    } else {   // node 0 of the rebuilt records: its point + its two boxes bound the map
      CUDA_TRY(cudaMemcpyAsync(D->h_res + MALIO_RED_DOUBLES + 16, D->d_nodes, sizeof(malio_map_node), cudaMemcpyDeviceToHost, D->stream2));
      CUDA_TRY(cudaStreamSynchronize(D->stream2));
      D->refit_pending = false;
      std::memcpy(&root, D->h_res + MALIO_RED_DOUBLES + 16, sizeof(root));
    }
  }
  const int rc = finish_map_upload(h, D, &root, n, depth);
  CUDA_TRY(cudaEventSynchronize(D->ev_cov));   // host buffer consumed; every later launch is issued after this point
  return rc;
}

// ---- device-resident map (malio_mapops.cu): slot storage and the index over it
// grow d_mpts / d_cov / d_ids to hold n slots, keeping the first `keep` of them
int grow_slots(malio_handle* h, uint32_t n, uint32_t keep) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (n <= D->cap_slots && D->d_ids) return MALIO_OK;
  uint32_t cap = n + n / 2 + 4096;
  if (cap < h->cfg.max_map_nodes) cap = h->cfg.max_map_nodes;
  float4* nm = nullptr; float* nc = nullptr; int32_t* ni = nullptr;
  CUDA_TRY(cudaMalloc((void**)&nm, (size_t)cap * sizeof(float4)));
  CUDA_TRY(cudaMalloc((void**)&nc, (size_t)cap * sizeof(float)));
  CUDA_TRY(cudaMalloc((void**)&ni, (size_t)cap * sizeof(int32_t)));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  if (keep && D->tree_free) {
    CUDA_TRY(cudaMemcpy(nm, D->d_mpts, (size_t)keep * sizeof(float4), cudaMemcpyDeviceToDevice));
    CUDA_TRY(cudaMemcpy(nc, D->d_cov, (size_t)keep * sizeof(float), cudaMemcpyDeviceToDevice));
    if (D->d_ids) CUDA_TRY(cudaMemcpy(ni, D->d_ids, (size_t)keep * sizeof(int32_t), cudaMemcpyDeviceToDevice));
  }
  if (D->d_mpts) cudaFree(D->d_mpts);
  if (D->d_cov) cudaFree(D->d_cov);
  if (D->d_ids) cudaFree(D->d_ids);
  // the tree records belong to the snapshot mode; they are re-created by the next malio_upload_map* call
  if (D->d_nodes) { cudaFree(D->d_nodes); D->d_nodes = nullptr; }
  if (D->d_parent) { cudaFree(D->d_parent); D->d_parent = nullptr; }
  if (D->d_arrived) { cudaFree(D->d_arrived); D->d_arrived = nullptr; }
  D->d_mpts = nm; D->d_cov = nc; D->d_ids = ni;
  D->cap_slots = cap;
  D->cap_nodes = cap;      // sizes the cell-list arrays (grid_build)
  return MALIO_OK;
}
// (re)build the cell-list index over the n_slots slots; box = {x_min,x_max,y_min,y_max,z_min,z_max} of the live points
int index_from_slots(malio_handle* h, uint32_t n_slots, const float box[6]) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (D->refit_pending) { CUDA_TRY(cudaStreamSynchronize(D->stream2)); D->refit_pending = false; }
  D->tree_free = true;
  malio_map_node root{};
  root.x = box[0]; root.y = box[2]; root.z = box[4];
  root.link = MALIO_LINK_HAS_LEFT;
  for (int k = 0; k < 6; ++k) root.lbox[k] = box[k];
  const int rc = finish_map_upload(h, D, &root, n_slots, 0);
  if (rc == MALIO_OK && n_slots > 0 && !D->grid_on) { h->err = "device-resident map: extent too large for the cell-list index"; return MALIO_ERR_CAPACITY; }
  return rc;
}

int download_map_nodes(malio_handle* h, malio_map_node* out, uint32_t cap) {
  DeviceState* D = (DeviceState*)h->dev;
  if (!D->map_ready || D->tree_free) { h->err = "download_map_nodes needs a snapshot uploaded with malio_upload_map*"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t n = D->n_nodes < cap ? D->n_nodes : cap;
  if (D->refit_pending) { CUDA_TRY(cudaStreamSynchronize(D->stream2)); D->refit_pending = false; }
  CUDA_TRY(cudaMemcpy(out, D->d_nodes, (size_t)n * sizeof(malio_map_node), cudaMemcpyDeviceToHost));
  return MALIO_OK;
}

static int ensure_point_buffers(malio_handle* h, DeviceState* D, uint32_t n) {
  if (n <= D->capN) return MALIO_OK;
  uint32_t cap = n + n / 8 + 1024;
  if (cap < h->cfg.max_points) cap = h->cfg.max_points;
  int rc = 0;
  if ((rc = ensure(h, D->d_pts, cap))) return rc;
  if ((rc = ensure(h, D->d_pts_sorted, cap))) return rc;
  if ((rc = ensure(h, D->d_perm, cap))) return rc;
  if ((rc = ensure(h, D->d_keys16, cap))) return rc;
  if ((rc = ensure(h, D->d_tmp_ids, cap))) return rc;
  if ((rc = ensure(h, D->d_nn_idx, (size_t)cap * MALIO_K))) return rc;
  if ((rc = ensure(h, D->d_nn_d2, (size_t)cap * MALIO_K))) return rc;
  if ((rc = ensure(h, D->d_sel, cap))) return rc;
  if ((rc = ensure(h, D->d_world, cap))) return rc;
  if ((rc = ensure(h, D->d_plane, cap))) return rc;
  if ((rc = ensure(h, D->d_ucov, cap))) return rc;
  if ((rc = ensure(h, D->d_tau, cap))) return rc;
  if ((rc = ensure(h, D->d_tau2, cap))) return rc;
  if ((rc = ensure(h, D->d_pd2, cap))) return rc;
  if ((rc = ensure(h, D->d_rows12, (size_t)cap * 12))) return rc;
  if ((rc = ensure(h, D->d_lid8, cap))) return rc;
  if ((rc = ensure(h, D->d_normal_y, cap))) return rc;
  if ((rc = ensure(h, D->d_o_ny, cap))) return rc;
  if ((rc = ensure(h, D->d_o_idx, (size_t)cap * MALIO_K))) return rc;
  if ((rc = ensure(h, D->d_o_d2, (size_t)cap * MALIO_K))) return rc;
  if ((rc = ensure(h, D->d_o_sel, cap))) return rc;
  if ((rc = ensure(h, D->d_o_world, (size_t)cap * 3))) return rc;
  if ((rc = ensure(h, D->d_fb_list, cap))) return rc;
  const uint32_t blocks = (cap + PLANE_THREADS - 1) / PLANE_THREADS;
  if ((rc = ensure(h, D->d_block_mm, (size_t)blocks * 4))) return rc;
  if ((rc = ensure(h, D->d_block_cnt, blocks))) return rc;
  D->cap_blocks = blocks;
  D->capN = cap;
  return MALIO_OK;
}

int upload_scan(malio_handle* h, const malio_scan_pt* pts, uint32_t n, const malio_pose_entry* table,
                const uint32_t* table_off, const malio_rigid* tcomp) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  const int L = h->cfg.params.n_lidar;
  for (int l = 0; l < L; ++l)
    if (table_off[l + 1] < table_off[l] + 2) { h->err = "pose table of each LiDAR needs >= 2 entries"; return MALIO_ERR_INVALID_ARG; }
  {   // pt.lidar indexes per-LiDAR tables on the device: reject ids outside [0, L) here (one vectorisable sweep)
    uint32_t bad = 0;
    for (uint32_t i = 0; i < n; ++i) bad |= (uint32_t)(pts[i].lidar >= (uint16_t)L);
    if (bad) { h->err = "scan point with lidar id >= n_lidar"; return MALIO_ERR_INVALID_ARG; }
  }
  if (int rc = ensure_point_buffers(h, D, n > 0 ? n : 1)) return rc;
  const uint32_t n_tab = table_off[L];
  if (n_tab > D->cap_table) {
    if (int rc = ensure(h, D->d_table, (size_t)(n_tab + 64) * TABLE_DOUBLES)) return rc;
    D->cap_table = n_tab + 64;
  }
  if (n) CUDA_TRY(cudaMemcpyAsync(D->d_pts, pts, (size_t)n * sizeof(malio_scan_pt), cudaMemcpyHostToDevice, D->stream));
  CUDA_TRY(cudaMemcpyAsync(D->d_table, table, (size_t)n_tab * sizeof(malio_pose_entry), cudaMemcpyHostToDevice, D->stream));
  reset_scan_kernel<<<(D->capN + 255) / 256, 256, 0, D->stream>>>(D->capN, D->d_sel, D->d_normal_y, D->d_nn_idx, D->d_gstats);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  for (int l = 0; l <= MALIO_MAX_LIDAR; ++l) D->table_off[l] = (l <= L) ? table_off[l] : table_off[L];
  for (int l = 1; l < L; ++l) D->tcomp[l] = tcomp[l - 1];
  D->N = n; D->scan_ready = true; D->perm_valid = false; D->tau_valid = false; D->pass_done = false; D->searched_once = false;
  D->ctr.h2d_bytes += (uint64_t)n * sizeof(malio_scan_pt) + (uint64_t)n_tab * sizeof(malio_pose_entry);
  return MALIO_OK;
}

// grow the per-point buffers to hold n points of a scan that is assembled on the device (malio_upload_scan_device);
// called right after upload_scan(.., 0 points, tables): the per-scan state is already reset, a re-allocation resets it again
int reserve_scan(malio_handle* h, uint32_t n) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (n > D->capN) {
    if (int rc = ensure_point_buffers(h, D, n)) return rc;
    reset_scan_kernel<<<(D->capN + 255) / 256, 256, 0, D->stream>>>(D->capN, D->d_sel, D->d_normal_y, D->d_nn_idx, D->d_gstats);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(D->stream));
  }
  return MALIO_OK;
}

int rearm_scan(malio_handle* h) {
  DeviceState* D = (DeviceState*)h->dev;
  if (!D->scan_ready) { h->err = "rearm_scan before upload_scan"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  reset_scan_kernel<<<(D->capN + 255) / 256, 256, 0, D->stream>>>(D->capN, D->d_sel, D->d_normal_y, D->d_nn_idx, D->d_gstats);
  CUDA_TRY(cudaGetLastError());
  D->perm_valid = false; D->tau_valid = false; D->pass_done = false; D->searched_once = false;
  return MALIO_OK;
}

int set_timing(malio_handle* h, int enable) {
  ((DeviceState*)h->dev)->timing = enable != 0;
  return MALIO_OK;
}

int get_counters(malio_handle* h, malio_counters* out) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  unsigned long long c[4] = {0, 0, 0, 0};
  CUDA_TRY(cudaMemcpy(c, D->d_cand, sizeof(c), cudaMemcpyDeviceToHost));
  D->ctr.knn_candidates = c[0];
  D->ctr.exchange_min_wait_ms = (double)c[1] * 1e-6;
  D->ctr.exchange_sum_wait_ms = (double)c[2] * 1e-6;
  D->ctr.exchange_passes = c[3];
  D->ctr.knn_tie_queries = D->h_gstats[7];
  *out = D->ctr;
  return MALIO_OK;
}

int measure(malio_handle* h, const malio_pass_state* s, int redo_knn, double* HtRinvH, double* HtRinvh,
            malio_pass_stats* st) {
  DeviceState* D = (DeviceState*)h->dev;
  if (h->mapst) { if (int rc = malio_map::commit(h)) return rc; }   // device-resident map: pending deltas -> index
  if (!D->map_ready || !D->scan_ready) { h->err = "measure before upload_map/upload_scan"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const malio_params& P = h->cfg.params;
  const int L = P.n_lidar, c = 6 * (L + 1);
  const uint32_t N = D->N;
  const auto hp0 = std::chrono::steady_clock::now();
  const PassConst pc = make_pass_const(h, D, s);
  const ParamConst prm = make_param_const(P);
  D->last_pc = pc;
  cudaStream_t st_ = D->stream;
  const uint32_t* perm = nullptr;
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[0], st_));
  bool sorted_now = false, knn_now = false, tau_async_outer = false;
  // the per-pass kernels read the scan in position order: the sorted copy when the scan was sorted, else the upload itself
  const malio_scan_pt* pts_k = (h->cfg.sort_queries && N > 0) ? D->d_pts_sorted : D->d_pts;
  const uint32_t* perm_k = nullptr;
  if (N > 0) {
    if (h->cfg.sort_queries) {
      if (!D->perm_valid) {
        if (int rc = sort_queries<0>(h, D, N, pc)) return rc;
        D->perm_valid = true;
        sorted_now = true;
      }
      perm = D->d_perm;
    }
    if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[5], st_));
    // once per scan: evalPointUncertainty's trace depends on the point and its table entry only.  On the first pass of
    // a scan that is a search pass it runs on the second stream beside the k-NN kernels (which leave most of the SMs'
    // warp slots empty) instead of inside the pass kernel.
    bool tau_async = false;
    if (!D->tau_valid && redo_knn && D->fused) {
      CUDA_TRY(cudaEventRecord(D->ev_sorted, st_));
      CUDA_TRY(cudaStreamWaitEvent(D->stream2, D->ev_sorted, 0));
      tau_kernel<<<(N + PLANE_THREADS - 1) / PLANE_THREADS, PLANE_THREADS, 0, D->stream2>>>(pts_k, perm_k, N, pc, D->d_table, D->d_tau2);
      CUDA_TRY(cudaEventRecord(D->ev_tau, D->stream2));
      D->tau_valid = true;
      D->ctr.kernel_launches += 1;
      tau_async = true;
    }
    tau_async_outer = tau_async;
    if (redo_knn) {
      knn_now = true;
      if (int rc = run_knn<0>(h, D, N, pts_k, perm_k, pc, P.knn_max_sqdist)) return rc;
      D->searched_once = true;
      if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[6], st_));
      // list statistics of this search: the fused pass kernel ships them with its result; the separate-kernel path copies
      if (!(D->fused && (!D->comm || D->p2p))) {
        if (D->grid_on) CUDA_TRY(cudaMemcpyAsync(D->h_gstats + 2, D->d_gstats + 2, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st_));
        CUDA_TRY(cudaMemcpyFromSymbolAsync(D->h_gstats + 6, g_fault_word, sizeof(uint32_t), 0, cudaMemcpyDeviceToHost, st_));
        CUDA_TRY(cudaMemcpyAsync(D->h_gstats + 7, D->d_gstats + 7, sizeof(uint32_t), cudaMemcpyDeviceToHost, st_));
      }
    }
  }
  if (tau_async_outer) CUDA_TRY(cudaStreamWaitEvent(st_, D->ev_tau, 0));
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[1], st_));
  unsigned long long* mmkey = D->d_mmkey + 4 * D->parity;
  unsigned long long* mmkey_next = D->d_mmkey + 4 * (1 - D->parity);
  uint32_t* cnt_cell = D->d_counters + 4 + D->parity;
  uint32_t* cnt_next = D->d_counters + 4 + (1 - D->parity);
  const uint32_t n_tiles = (N + RED_THREADS - 1) / RED_THREADS;
  // one resident wave, every block the same number of tiles (+-1): no straggler blocks
  const bool fused_now = D->fused && (!D->comm || D->p2p);
  uint32_t wave = fused_now ? fast_wave(D) : D->red_grid;
  uint32_t per_block = n_tiles ? (n_tiles + wave - 1) / wave : 1;
  if (fused_now && per_block > (uint32_t)PASS_FAST_TILES) {   // rows through global memory: that variant's own co-residency limit
    wave = (uint32_t)D->pass_max_blocks_generic < D->red_grid ? (uint32_t)D->pass_max_blocks_generic : D->red_grid;
    per_block = (n_tiles + wave - 1) / wave;
  }
  const uint32_t grid = n_tiles ? (n_tiles + per_block - 1) / per_block : 1;
  std::chrono::steady_clock::time_point hp1, hp2;
  if (D->fused && (!D->comm || D->p2p)) {
    // ---- the whole pass in one cooperative launch; the result arrives in mapped host memory.  With several GPUs the two
    // exchanges of the pass happen inside the kernel through the peers' mailboxes (CUDA IPC over NVLink)
    PassArgs a{};
    a.pts = pts_k; a.perm = perm_k; a.N = N; a.table = D->d_table; a.nodes = D->d_mpts; a.node_cov = D->d_cov;
    a.nn_idx = D->d_nn_idx; a.sel = D->d_sel; a.world = D->d_world; a.plane = D->d_plane; a.ucov = D->d_ucov;
    a.tau2 = D->d_tau2; a.pd2 = D->d_pd2; a.tau = D->d_tau; a.normal_y = D->d_normal_y; a.rows12 = D->d_rows12; a.lid8 = D->d_lid8;
    a.do_tau = (N > 0 && !D->tau_valid) ? 1 : 0;
    a.do_fit = (N > 0 && redo_knn) ? 1 : 0;
    a.mmkey = mmkey; a.mmkey_next = mmkey_next; a.cnt_cell = cnt_cell; a.cnt_next = cnt_next; a.gstats = D->d_gstats;
    a.bar = D->d_bar;
    for (int k = 0; k < 3; ++k) a.bar_base[k] = D->bar_base[k];
    D->bar_base[0] += grid; D->bar_base[1] += grid; D->bar_base[2] += MALIO_RED_DOUBLES;
    a.n_tiles = n_tiles; a.block_red = D->d_block_red; a.d_res = D->d_res; a.h_res = D->h_res_dev;
    a.seq = ++D->seq;
    a.peer.rank = D->rank; a.peer.world = D->p2p ? D->world : 1;
    for (int r = 0; r < MAIL_MAX_WORLD; ++r) a.peer.mail[r] = D->mail_peer[r];
    *reinterpret_cast<volatile uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 9) = 0u;
    a.dbg = nullptr;
    a.xwait = D->d_cand + 1;
    if (D->trace_passes > 0) {
      if (!D->d_dbg) { CUDA_TRY(cudaMalloc((void**)&D->d_dbg, (size_t)4096 * 8 * sizeof(unsigned long long))); D->trace_left = D->trace_passes; }
      if (D->trace_left > 0 && grid <= 4096) a.dbg = D->d_dbg;
    }
    PassConst pc_arg = pc;
    ParamConst prm_arg = prm;
    void* kargs[] = {&a, &pc_arg, &prm_arg};
    const bool fast = per_block <= (uint32_t)PASS_FAST_TILES;
    const size_t pass_smem = (fast ? PASS_FAST_SMEM_DOUBLES : RED_SMEM_DOUBLES) * sizeof(double);
    CUDA_TRY(cudaLaunchCooperativeKernel(fast ? (const void*)pass_kernel<true> : (const void*)pass_kernel<false>, dim3(grid),
                                         dim3(RED_THREADS), kargs, pass_smem, st_));
    D->ctr.kernel_launches += 1;
    D->tau_valid = D->tau_valid || N > 0;
    if (D->timing) { CUDA_TRY(cudaEventRecord(D->ev[2], st_)); CUDA_TRY(cudaEventRecord(D->ev[3], st_)); CUDA_TRY(cudaEventRecord(D->ev[4], st_)); }
    D->last_parity = D->parity;
    D->parity = 1 - D->parity;
    hp1 = std::chrono::steady_clock::now();
    // the host needs the 3.5 KB system to take the IESKF step: spin on the sequence flag the kernel writes last
    volatile uint32_t* flag = reinterpret_cast<volatile uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 8);
    for (uint64_t spins = 1; *flag != D->seq; ++spins) {
      __builtin_ia32_pause();
      if ((spins & 0x3FFF) == 0) {
        const cudaError_t q = cudaStreamQuery(st_);
        if (q == cudaErrorNotReady) {
          if (std::chrono::duration<double>(std::chrono::steady_clock::now() - hp1).count() > 20.0) {
            h->err = "pass_kernel: no result after 20 s";
            return MALIO_ERR_CUDA;
          }
          continue;
        }
        if (q != cudaSuccess) { h->err = std::string("pass_kernel: ") + cudaGetErrorString(q); return MALIO_ERR_CUDA; }
        if (*flag != D->seq) { h->err = "pass_kernel finished without publishing its result"; return MALIO_ERR_CUDA; }
      }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    if (const uint32_t fault = *reinterpret_cast<volatile uint32_t*>(D->h_res + MALIO_RED_DOUBLES + 9)) {
      if (fault == 2u) { h->err = "pass_kernel: a grid barrier did not complete within 2 s (blocks not co-resident)"; return MALIO_ERR_CUDA; }
      h->err = "pass_kernel: a peer GPU did not answer the in-kernel exchange within 2 s";
      return MALIO_ERR_NCCL;
    }
    if (a.dbg) {
      CUDA_TRY(cudaStreamSynchronize(st_));
      std::vector<unsigned long long> t((size_t)grid * 8);
      CUDA_TRY(cudaMemcpy(t.data(), D->d_dbg, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      unsigned long long t00 = ~0ull;
      for (uint32_t b = 0; b < grid; ++b) if (t[b * 8] < t00) t00 = t[b * 8];
      const char* nm[6] = {"start", "phase1 done", "barrier1 passed", "phase2 done", "barrier2 passed", "end"};
      fprintf(stderr, "[malio] pass trace: grid %u fast %d fit %d tau %d (us from first block start: min / mean / max over blocks)\n",
              grid, per_block <= (uint32_t)PASS_FAST_TILES, a.do_fit, a.do_tau);
      for (int k = 0; k < 6; ++k) {
        double mn = 1e30, mx = 0, sm = 0;
        for (uint32_t b = 0; b < grid; ++b) { const double v = (double)(t[b * 8 + k] - t00) * 1e-3; mn = v < mn ? v : mn; mx = v > mx ? v : mx; sm += v; }
        fprintf(stderr, "[malio]   %-16s %8.2f %8.2f %8.2f\n", nm[k], mn, sm / grid, mx);
      }
      D->trace_left--;
    }
    if (D->timing) CUDA_TRY(cudaEventSynchronize(D->ev[4]));
    hp2 = std::chrono::steady_clock::now();
  } else {
  const uint32_t pblocks = N > 0 ? (N + PLANE_THREADS - 1) / PLANE_THREADS : 1;
  if (N > 0 && !D->tau_valid) {   // once per scan
    tau_kernel<<<pblocks, PLANE_THREADS, 0, st_>>>(pts_k, perm_k, N, pc, D->d_table, D->d_tau2);
    D->tau_valid = true;
    D->ctr.kernel_launches += 1;
  }
  if (N > 0 && redo_knn) {         // once per search
    fit_kernel<<<pblocks, PLANE_THREADS, 0, st_>>>(D->d_mpts, D->d_cov, N, prm, D->d_nn_idx, D->d_sel, D->d_plane, D->d_ucov);
    D->ctr.kernel_launches += 1;
  }
  D->ctr.kernel_launches += 3;     // gate, reduce, fold
  const uint32_t gblocks = N > 0 ? (N + GATE_THREADS - 1) / GATE_THREADS : 1;
  gate_kernel<<<gblocks, GATE_THREADS, 0, st_>>>(pts_k, perm_k, N, pc, D->d_plane, D->d_ucov, D->d_tau2, D->d_sel,
                                                   D->d_world, D->d_pd2, D->d_tau, D->d_normal_y, D->d_rows12, D->d_lid8, mmkey, cnt_cell);
  if (D->comm)   // keys of {min_u, -max_u, min_tau, -max_tau}: one MIN all-reduce (laserMapping.cpp:615-628, 700-703)
    if (g_nccl.AllReduce(mmkey, mmkey, 4, ncclUint64, ncclMin, D->comm, st_) != ncclSuccess) { h->err = "ncclAllReduce(min) failed"; return MALIO_ERR_NCCL; }
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[2], st_));
  reduce_kernel<<<grid, RED_THREADS, RED_SMEM_DOUBLES * sizeof(double), st_>>>(
      N, prm, pc.ext_en, D->d_sel, D->d_lid8, D->d_rows12, D->d_pd2, D->d_ucov, D->d_tau, mmkey, n_tiles, D->d_block_red);
  fold_kernel<<<(MALIO_RED_DOUBLES * 32 + 255) / 256, 256, 0, st_>>>(D->d_block_red, grid, D->d_res, mmkey_next, cnt_next, D->d_gstats);
  if (D->comm)   // the reduced system + n_eff: one SUM all-reduce
    if (g_nccl.AllReduce(D->d_res, D->d_res, MALIO_RED_DOUBLES, ncclDouble, ncclSum, D->comm, st_) != ncclSuccess) { h->err = "ncclAllReduce(sum) failed"; return MALIO_ERR_NCCL; }
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[3], st_));
  CUDA_TRY(cudaMemcpyAsync(D->h_res, D->d_res, MALIO_RED_DOUBLES * sizeof(double), cudaMemcpyDeviceToHost, st_));
  CUDA_TRY(cudaMemcpyAsync(D->h_res + MALIO_RED_DOUBLES, mmkey, 4 * sizeof(double), cudaMemcpyDeviceToHost, st_));
  D->last_parity = D->parity;
  D->parity = 1 - D->parity;
  if (D->timing) CUDA_TRY(cudaEventRecord(D->ev[4], st_));
  hp1 = std::chrono::steady_clock::now();
  CUDA_TRY(cudaStreamSynchronize(st_));
  hp2 = std::chrono::steady_clock::now();
  CUDA_TRY(cudaGetLastError());
  }
  D->pass_done = true;
  if (D->h_gstats[6] & FAULT_STACK_OVERFLOW) {
    h->err = "k-NN traversal stack overflow: the snapshot is deeper than the max_depth declared at upload";
    return MALIO_ERR_TREE_TOO_DEEP;
  }
  D->host_launch_us += std::chrono::duration<double, std::micro>(hp1 - hp0).count();
  D->host_wait_us += std::chrono::duration<double, std::micro>(hp2 - hp1).count();
  D->host_passes += 1;

  // ---- host epilogue: un-block, localization weight (laserMapping.cpp:745-759), compact to c x c
  const double* res = D->h_res;
  double mm[4];
  for (int k = 0; k < 4; ++k) { unsigned long long key; std::memcpy(&key, D->h_res + MALIO_RED_DOUBLES + k, 8); mm[k] = dkey_inv(key); }
  // res holds, per LiDAR l, the 9 upper-triangular 4x4 blocks of the compact 12 x 16 system Gc_l; scatter into the
  // padded 24 x 28 one (columns at their L=3 positions: 0-5 | 6+3l | 15+3l ; 24 = residual ; 25-27 = normal scatter)
  double G[MALIO_RED_ROWS][MALIO_RED_COLS];
  std::memset(G, 0, sizeof(G));
  for (int l = 0; l < MALIO_MAX_LIDAR; ++l) {
    double Gc[12][16];
    std::memset(Gc, 0, sizeof(Gc));
    int t = 0;
    for (int gi = 0; gi < 3; ++gi)
      for (int gj = gi; gj < 4; ++gj, ++t)
        for (int a = 0; a < 4; ++a)
          for (int b = 0; b < 4; ++b) Gc[4 * gi + a][4 * gj + b] = res[(l * 9 + t) * 16 + a * 4 + b];
    for (int a = 0; a < 12; ++a) for (int b = 0; b < a; ++b) Gc[a][b] = Gc[b][a];
    int col[16];
    for (int k = 0; k < 6; ++k) col[k] = k;
    for (int k = 0; k < 3; ++k) { col[6 + k] = 6 + 3 * l + k; col[9 + k] = 15 + 3 * l + k; }
    col[12] = 24; col[13] = 25; col[14] = 26; col[15] = 27;
    for (int a = 0; a < 12; ++a)
      for (int b = 0; b < 16; ++b) G[col[a]][col[b]] += Gc[a][b];
  }
  const uint32_t n_eff = (uint32_t)(res[MALIO_RED_BLOCKS * 16] + 0.5);
  malio_pass_stats S{};
  S.n_points = N; S.n_eff = n_eff; S.searched = redo_knn ? 1 : 0;
  S.u_min = mm[0]; S.u_max = -mm[1]; S.tau_min = mm[2]; S.tau_max = -mm[3];
  float ms = 0.f;
  if (knn_now && D->grid_on) { D->ctr.knn_fallback_queries += D->h_gstats[3]; D->ctr.knn_ring2_queries += D->h_gstats[5]; }
  if (D->timing) {
  if (N > 0 && sorted_now) { cudaEventElapsedTime(&ms, D->ev[0], D->ev[5]); S.ms_sort = ms; }
  if (knn_now) {
    cudaEventElapsedTime(&ms, D->ev[5], D->ev[6]); S.ms_knn = ms;
    D->ctr.knn_launches += 1; D->ctr.knn_queries += N; D->ctr.knn_ms += ms;
  }
  D->ctr.d2h_bytes += (MALIO_RED_DOUBLES + 4) * sizeof(double);
  cudaEventElapsedTime(&ms, D->ev[1], D->ev[2]); S.ms_plane = ms;
  cudaEventElapsedTime(&ms, D->ev[2], D->ev[3]); S.ms_reduce = ms;
  cudaEventElapsedTime(&ms, D->ev[0], D->ev[4]); S.ms_total = ms;
  cudaEventElapsedTime(&ms, D->ev[1], D->ev[4]);
  D->ctr.pass_launches += 1; D->ctr.pass_points += N; D->ctr.pass_ms += ms; D->ctr.pass_fit_launches += redo_knn ? 1 : 0;
  }
  if (n_eff < 1) {
    S.valid = 0;
    if (st) *st = S;
    return MALIO_ERR_NO_EFFECTIVE_POINTS;
  }
  S.valid = 1;
  const double Ssym[6] = {G[0][25], G[0][26], G[0][27], G[1][26], G[1][27], G[2][27]};
  malio_host::sym3_singular_values(Ssym, S.sigma);
  double weight = S.sigma[2] / S.sigma[0];
  if (weight > P.localize_thresh_max) weight = P.localize_cov_max;
  else if (weight < P.localize_thresh_min) weight = P.localize_cov_min;
  else weight = (P.localize_cov_max - P.localize_cov_min) * (weight - P.localize_thresh_min) / (P.localize_thresh_max - P.localize_thresh_min) + P.localize_cov_min;
  S.loc_weight = weight;
  const double w2 = weight * weight;
  // padded (L=3 positions) -> compact c columns: 0-5 | 6+3l | 6+3L+3l
  int map[MALIO_MAX_COLS];
  for (int k = 0; k < 6; ++k) map[k] = k;
  for (int l = 0; l < L; ++l)
    for (int k = 0; k < 3; ++k) { map[6 + 3 * l + k] = 6 + 3 * l + k; map[6 + 3 * L + 3 * l + k] = 15 + 3 * l + k; }
  for (int a = 0; a < c; ++a) {
    for (int b = 0; b < c; ++b) HtRinvH[a * c + b] = w2 * G[map[a]][map[b]];
    HtRinvh[a] = w2 * G[map[a]][24];
  }
  if (st) *st = S;
  return MALIO_OK;
}

int download_rows(malio_handle* h, double* h_x, double* hvec, uint32_t cap, uint32_t* n_rows) {
  DeviceState* D = (DeviceState*)h->dev;
  if (!D->pass_done) { h->err = "download_rows before measure"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const malio_params& P = h->cfg.params;
  const int L = P.n_lidar, c = 6 * (L + 1);
  if (cap > MALIO_MAX_DOF) cap = MALIO_MAX_DOF;
  rows_kernel<<<1, 256, 0, D->stream>>>(D->N, make_param_const(P), D->last_pc.ext_en, D->d_sel, D->d_lid8, D->d_rows12,
                                          D->d_pd2, D->d_ucov, D->d_tau, D->d_mmkey + 4 * D->last_parity, cap, D->d_rows,
                                          D->d_counters + 3);
  double* hr = D->h_res + MALIO_RED_DOUBLES + 16;
  uint32_t nr = 0;
  std::vector<double> gathered;
  if (D->comm && D->world > 1) {
    // stats->n_eff is summed over the ranks, the rows are not: gather every rank's (at most cap) rows and concatenate them in
    // rank order, so that every rank forms the same H and takes the same step (esekfom.hpp:574-582 needs all N_eff rows)
    if (!g_nccl.AllGather) { h->err = "ncclAllGather unavailable: cannot gather the rows of the degenerate branch"; return MALIO_ERR_NCCL; }
    double* d_all = D->d_rows + ROWS_DOUBLES;
    if (g_nccl.AllGather(D->d_rows, d_all, ROWS_DOUBLES, ncclDouble, D->comm, D->stream) != ncclSuccess) { h->err = "ncclAllGather(rows) failed"; return MALIO_ERR_NCCL; }
    gathered.resize((size_t)ROWS_DOUBLES * D->world);
    CUDA_TRY(cudaMemcpyAsync(gathered.data(), d_all, gathered.size() * sizeof(double), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    D->ctr.kernel_launches += 1;
    for (int r = 0; r < D->world && nr < cap; ++r) {
      const double* src = gathered.data() + (size_t)r * ROWS_DOUBLES;
      const uint32_t cnt = (uint32_t)(src[(size_t)MALIO_MAX_DOF * 25] + 0.5);
      for (uint32_t k = 0; k < cnt && nr < cap; ++k, ++nr) std::memcpy(hr + (size_t)nr * 25, src + (size_t)k * 25, 25 * sizeof(double));
    }
  } else {
    CUDA_TRY(cudaMemcpyAsync(hr, D->d_rows, (size_t)cap * 25 * sizeof(double), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaMemcpyAsync(&nr, D->d_counters + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    if (nr > cap) nr = cap;
  }
  int map[MALIO_MAX_COLS];
  for (int k = 0; k < 6; ++k) map[k] = k;
  for (int l = 0; l < L; ++l)
    for (int k = 0; k < 3; ++k) { map[6 + 3 * l + k] = 6 + 3 * l + k; map[6 + 3 * L + 3 * l + k] = 15 + 3 * l + k; }
  for (uint32_t r = 0; r < nr; ++r) {
    for (int k = 0; k < c; ++k) h_x[(size_t)r * c + k] = hr[(size_t)r * 25 + map[k]];
    hvec[r] = hr[(size_t)r * 25 + 24];
  }
  *n_rows = nr;
  return MALIO_OK;
}

int download_aux(malio_handle* h, float* normal_y, uint32_t* nn_idx, float* nn_d2, uint8_t* sel, float* world) {
  DeviceState* D = (DeviceState*)h->dev;
  if (!D->pass_done) { h->err = "download_aux before measure"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t N = D->N;
  if (N == 0) return MALIO_OK;
  const uint32_t* perm = (h->cfg.sort_queries && D->perm_valid) ? D->d_perm : nullptr;
  scatter_aux_kernel<<<(N + 255) / 256, 256, 0, D->stream>>>(
      perm, N, D->d_normal_y, D->d_nn_idx, D->d_nn_d2, D->d_sel, D->d_world, normal_y ? D->d_o_ny : nullptr,
      nn_idx ? D->d_o_idx : nullptr, nn_d2 ? D->d_o_d2 : nullptr, sel ? D->d_o_sel : nullptr,
      world ? D->d_o_world : nullptr);
  if (normal_y) CUDA_TRY(cudaMemcpyAsync(normal_y, D->d_o_ny, (size_t)N * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  if (nn_idx) CUDA_TRY(cudaMemcpyAsync(nn_idx, D->d_o_idx, (size_t)N * MALIO_K * sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
  if (nn_d2) CUDA_TRY(cudaMemcpyAsync(nn_d2, D->d_o_d2, (size_t)N * MALIO_K * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  if (sel) CUDA_TRY(cudaMemcpyAsync(sel, D->d_o_sel, (size_t)N, cudaMemcpyDeviceToHost, D->stream));
  if (world) CUDA_TRY(cudaMemcpyAsync(world, D->d_o_world, (size_t)N * 3 * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  D->ctr.kernel_launches += 1;
  D->ctr.d2h_bytes += (uint64_t)N * ((normal_y ? 4 : 0) + (nn_idx ? 20 : 0) + (nn_d2 ? 20 : 0) + (sel ? 1 : 0) + (world ? 12 : 0));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}

int knn(malio_handle* h, const float* q, uint32_t nq, uint32_t* idx, float* d2, float* ms_out) {
  DeviceState* D = (DeviceState*)h->dev;
  if (h->mapst) { if (int rc = malio_map::commit(h)) return rc; }
  if (!D->map_ready) { h->err = "knn before upload_map"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  if (nq == 0) return MALIO_OK;
  if (int rc = ensure_point_buffers(h, D, nq)) return rc;
  if (nq > D->capQ) {
    if (int rc = ensure(h, D->d_queries, (size_t)(nq + 1024) * 3)) return rc;
    D->capQ = nq + 1024;
  }
  D->scan_ready = false;   // point buffers are shared with the scan path
  D->pass_done = false;
  CUDA_TRY(cudaMemcpyAsync(D->d_queries, q, (size_t)nq * 3 * sizeof(float), cudaMemcpyHostToDevice, D->stream));
  PassConst pc{};
  const uint32_t* perm = nullptr;
  if (h->cfg.sort_queries) {
    if (int rc = sort_queries<1>(h, D, nq, pc)) return rc;
    perm = D->d_perm;
  }
  CUDA_TRY(cudaMemsetAsync(D->d_gstats + 2, 0, 4 * sizeof(uint32_t), D->stream));
  CUDA_TRY(cudaEventRecord(D->ev[0], D->stream));
  if (int rc = run_knn<1>(h, D, nq, nullptr, perm, pc, 0.f)) return rc;
  CUDA_TRY(cudaEventRecord(D->ev[1], D->stream));
  scatter_aux_kernel<<<(nq + 255) / 256, 256, 0, D->stream>>>(perm, nq, nullptr, D->d_nn_idx, D->d_nn_d2, nullptr,
                                                               nullptr, nullptr, idx ? D->d_o_idx : nullptr,
                                                               d2 ? D->d_o_d2 : nullptr, nullptr, nullptr);
  if (idx) CUDA_TRY(cudaMemcpyAsync(idx, D->d_o_idx, (size_t)nq * MALIO_K * sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
  if (d2) CUDA_TRY(cudaMemcpyAsync(d2, D->d_o_d2, (size_t)nq * MALIO_K * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  if (D->grid_on) CUDA_TRY(cudaMemcpyAsync(D->h_gstats + 2, D->d_gstats + 2, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
  CUDA_TRY(cudaMemcpyFromSymbolAsync(D->h_gstats + 6, g_fault_word, sizeof(uint32_t), 0, cudaMemcpyDeviceToHost, D->stream));
  CUDA_TRY(cudaMemcpyAsync(D->h_gstats + 7, D->d_gstats + 7, sizeof(uint32_t), cudaMemcpyDeviceToHost, D->stream));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  CUDA_TRY(cudaGetLastError());
  if (D->h_gstats[6] & FAULT_STACK_OVERFLOW) {
    h->err = "k-NN traversal stack overflow: the snapshot is deeper than the max_depth declared at upload";
    return MALIO_ERR_TREE_TOO_DEEP;
  }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, D->ev[0], D->ev[1]);
  if (ms_out) *ms_out = ms;
  D->ctr.kernel_launches += 1;   // scatter (the sort and the k-NN count their own)
  if (D->grid_on) { D->ctr.knn_fallback_queries += D->h_gstats[3]; D->ctr.knn_ring2_queries += D->h_gstats[5]; }
  D->ctr.knn_launches += 1; D->ctr.knn_queries += nq; D->ctr.knn_ms += ms;
  D->ctr.h2d_bytes += (uint64_t)nq * 12;
  D->ctr.d2h_bytes += (uint64_t)nq * ((idx ? 20 : 0) + (d2 ? 20 : 0));
  return MALIO_OK;
}

int map_incremental(malio_handle* h, const malio_pass_state* s, double fs, int ekf_inited, uint8_t* cls, float* world) {
  DeviceState* D = (DeviceState*)h->dev;
  if (!D->pass_done) { h->err = "map_incremental before measure"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t N = D->N;
  if (N == 0) return MALIO_OK;
  const bool sorted = h->cfg.sort_queries && D->perm_valid;
  const PassConst pc = make_pass_const(h, D, s);
  // d_o_sel / d_o_world: the caller-order staging buffers of download_aux
  map_incr_kernel<<<(N + 255) / 256, 256, 0, D->stream>>>(sorted ? D->d_pts_sorted : D->d_pts, sorted ? D->d_perm : nullptr, N, pc,
                                                           D->d_mpts, D->d_nn_idx, D->d_normal_y, h->cfg.params.cov_threshold, fs,
                                                           ekf_inited, D->d_o_sel, world ? D->d_o_world : nullptr);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(cls, D->d_o_sel, (size_t)N, cudaMemcpyDeviceToHost, D->stream));
  if (world) CUDA_TRY(cudaMemcpyAsync(world, D->d_o_world, (size_t)N * 3 * sizeof(float), cudaMemcpyDeviceToHost, D->stream));
  CUDA_TRY(cudaStreamSynchronize(D->stream));
  D->ctr.kernel_launches += 1;
  D->ctr.d2h_bytes += (uint64_t)N * (1 + (world ? 12 : 0));
  return MALIO_OK;
}

int get_unique_id(uint8_t* id) {
  std::string err;
  if (!g_nccl.load(err)) return MALIO_ERR_NCCL;
  ncclUniqueId uid;
  if (g_nccl.GetUniqueId(&uid) != ncclSuccess) return MALIO_ERR_NCCL;
  static_assert(sizeof(ncclUniqueId) == MALIO_NCCL_UNIQUE_ID_BYTES, "ncclUniqueId size");
  std::memcpy(id, &uid, sizeof(uid));
  return MALIO_OK;
}

int comm_init(malio_handle* h, const uint8_t* id, int rank, int world) {
  DeviceState* D = (DeviceState*)h->dev;
  CUDA_TRY(cudaSetDevice(D->device));
  if (!g_nccl.load(h->err)) return MALIO_ERR_NCCL;
  ncclUniqueId uid;
  std::memcpy(&uid, id, sizeof(uid));
  ncclResult_t r = g_nccl.CommInitRank(&D->comm, world, uid, rank);
  if (r != ncclSuccess) {
    h->err = std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    D->comm = nullptr;
    return MALIO_ERR_NCCL;
  }
  D->rank = rank; D->world = world;
  // ---- peer mailboxes for the in-kernel exchanges (CUDA IPC; NCCL only carries the 64-byte handles).  Falls back to the
  // NCCL all-reduce path between separate kernels unless EVERY rank succeeded.
  D->p2p = false;
  const char* env = getenv("MALIO_P2P");
  int ok = (world > 1 && world <= MAIL_MAX_WORLD && D->fused && g_nccl.AllGather && !(env && atoi(env) == 0)) ? 1 : 0;
  cudaIpcMemHandle_t mine{};
  unsigned char* d_h = nullptr;
  std::vector<cudaIpcMemHandle_t> all((size_t)world);
  if (ok) {
    if (cudaMalloc((void**)&D->d_mail, MAIL_BYTES) != cudaSuccess || cudaMemset(D->d_mail, 0, MAIL_BYTES) != cudaSuccess ||
        cudaIpcGetMemHandle(&mine, D->d_mail) != cudaSuccess) { ok = 0; cudaGetLastError(); }
  }
  // every rank takes part in the two collectives below whatever its own outcome
  if (world > 1 && g_nccl.AllGather) {
    CUDA_TRY(cudaMalloc((void**)&d_h, (size_t)(world + 1) * sizeof(mine) + 2 * sizeof(int)));
    CUDA_TRY(cudaMemcpy(d_h + (size_t)world * sizeof(mine), &mine, sizeof(mine), cudaMemcpyHostToDevice));
    if (g_nccl.AllGather(d_h + (size_t)world * sizeof(mine), d_h, sizeof(mine), ncclChar, D->comm, D->stream) != ncclSuccess) ok = 0;
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    CUDA_TRY(cudaMemcpy(all.data(), d_h, (size_t)world * sizeof(mine), cudaMemcpyDeviceToHost));
    if (ok) {
      for (int r = 0; r < world && ok; ++r) {
        if (r == rank) { D->mail_peer[r] = D->d_mail; continue; }
        void* ptr = nullptr;
        if (cudaIpcOpenMemHandle(&ptr, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); }
        D->mail_peer[r] = (unsigned char*)ptr;
      }
    }
    int* d_ok = reinterpret_cast<int*>(d_h + (size_t)(world + 1) * sizeof(mine));
    CUDA_TRY(cudaMemcpy(d_ok, &ok, sizeof(int), cudaMemcpyHostToDevice));
    if (g_nccl.AllReduce(d_ok, d_ok + 1, 1, ncclInt, ncclMin, D->comm, D->stream) != ncclSuccess) ok = 0;
    CUDA_TRY(cudaStreamSynchronize(D->stream));
    int all_ok = 0;
    CUDA_TRY(cudaMemcpy(&all_ok, d_ok + 1, sizeof(int), cudaMemcpyDeviceToHost));
    cudaFree(d_h);
    D->p2p = ok && all_ok;
  }
  if (D->host_prof) fprintf(stderr, "[malio] rank %d/%d: in-kernel peer exchange %s\n", rank, world, D->p2p ? "ON" : "off (NCCL path)");
  return MALIO_OK;
}

}  // namespace malio_dev
