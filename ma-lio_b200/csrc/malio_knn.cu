// malio_knn.cu — the k-NN search of libmalio_b200.so and the map it searches, sm_90a:
//   K1 knn_kernel      KD_TREE::Nearest_Search / Search   (ikd_Tree.cpp:426-461, 1073-1255)
// with its cell-list fast path, the tree-free ring search of the device-resident map, the snapshot uploads (and the box
// rebuild of the compact one), the cell-list index build and the query sort.  DESIGN.md has the data layout.
// Compiled with -fmad=false: every float/double expression below is evaluated with the same IEEE operations, in the same
// order, as the reference's x86-64 build (no FMA, CMakeLists.txt:8), so that k-NN index sets are bit-exact.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>

#include "malio_internal.h"
#include "malio_device.cuh"

using namespace malio_devstate;
namespace {

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
                                             uint32_t oi[MALIO_K], float od[MALIO_K], int& found_out, uint32_t* fault) {
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
      else atomicOr(fault, FAULT_STACK_OVERFLOW);
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
                                              unsigned wmask, uint32_t oi[MALIO_K], float od[MALIO_K], int& found,
                                              uint32_t* fault) {
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
        else atomicOr(fault, FAULT_STACK_OVERFLOW);   // deeper than declared: the result is not trusted, the call fails
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
    knn_exact_query(nodes, qx, qy, qz, oi, od, found, fault);
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
           float* __restrict__ nn_d2, uint8_t* __restrict__ sel, uint32_t* fault) {
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
    knn_tree_lane<SMEM_STACK>(nodes, qx, qy, qz, true, wmask, oi, od, found, fault);
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
                uint32_t* __restrict__ count_out, uint32_t* fault) {
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
      knn_tree_lane<SMEM_STACK>(nodes, qx, qy, qz, valid, 0xffffffffu, oi, od, found, fault);
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
constexpr int SCAN_THREADS = 256;
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
  if (ncell_pad > D->d_cell_start.size()) {
    if (int rc = malio_buf::allocate_group(h, st, {{D->d_cell_start, ncell_pad}, {D->d_cell_cnt, ncell_pad}})) return rc;
    if (!D->d_ctot) { if (int rc = malio_buf::allocate_group(h, st, {{D->d_ctot, 8192}, {D->d_cbase, 8192}})) return rc; }
  }
  if (D->d_mpts.size() > D->d_cell_of.size()) {
    if (int rc = malio_buf::allocate_group(h, st, {{D->d_cell_of, D->d_mpts.size()}, {D->d_cell_pts, D->d_mpts.size()}})) return rc;
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

}  // namespace

namespace malio_devstate {

template <int MODE>
int sort_queries(malio_handle* h, DeviceState* D, uint32_t n, const PassConst& pc, int lid_major, const float* queries) {
  cudaStream_t st = D->stream;
  CUDA_TRY(cudaMemsetAsync(D->d_hist, 0, SORT_BINS * sizeof(uint32_t), st));
  count_kernel<MODE><<<(n + 255) / 256, 256, 0, st>>>(D->d_pts, queries ? queries : D->d_queries, n, pc, lid_major, D->d_keys16, D->d_hist);
  scan_kernel<<<SCAN_BLOCKS, SCAN_THREADS, 0, st>>>(D->d_hist, D->d_offs, D->d_cursor, D->d_btot);
  // d_fb_list (the k-NN hand-over list, filled only later in the pass) doubles as the arrival-slot array of the sort
  scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(D->d_keys16, n, D->d_offs, D->d_btot, D->d_cursor, D->d_tmp_ids, D->d_fb_list);
  rank_kernel<<<(n + 255) / 256, 256, 0, st>>>(D->d_keys16, n, D->d_offs, D->d_btot, D->d_hist, D->d_tmp_ids, D->d_fb_list, D->d_perm,
                                               MODE == 0 ? D->d_pts.data() : nullptr, MODE == 0 ? D->d_pts_sorted.data() : nullptr);
  CUDA_TRY(cudaGetLastError());
  D->ctr.kernel_launches += 4;
  return MALIO_OK;
}

// the k-NN of one search pass: cell-list fast path + exact ikd-Tree-order traversal for what it leaves, or the
// traversal alone when the index is off
template <int MODE>
int run_knn(malio_handle* h, DeviceState* D, uint32_t n, const malio_scan_pt* pts_in, const uint32_t* perm,
            const PassConst& pc, float max_sqdist, const float* queries) {
  cudaStream_t st = D->stream;
  const bool smem_stack = D->depth + KNN_POP_WIDTH <= (uint32_t)KNN_SMEM_DEPTH;
  const malio_scan_pt* pts = MODE == 0 ? pts_in : nullptr;
  const float* qs = MODE == 0 ? nullptr : (queries ? queries : D->d_queries);
  float4* world = MODE == 0 ? D->d_world.data() : nullptr;
  uint8_t* sel = MODE == 0 ? D->d_sel.data() : nullptr;
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
        D->d_gstats + 4, D->d_fb_list, D->d_gstats + 2, D->timing ? D->d_cand.data() : nullptr);                                      \
  } while (0)
      // measured (ncu kernel time, C2 sub-sampled): 12.5k queries 31 -> 12 us with 4 lanes + row preload; 100k 29.5 -> 24 us with
      // 2 lanes; from ~200k queries on (C4, C5) the thread-per-query kernel is as fast or faster and stays
      if (grp == 2) MALIO_LAUNCH_KEYS(2, false);
      else MALIO_LAUNCH_KEYS(4, true);
#undef MALIO_LAUNCH_KEYS
    } else {
      knn_direct_kernel<MODE><<<(n + GD_THREADS - 1) / GD_THREADS, GD_THREADS, 0, st>>>(
          D->d_cell_pts, D->d_cell_start, D->grid, pts, perm, qs, n, pc, max_sqdist, world, D->d_nn_idx, D->d_nn_d2, sel,
          D->d_gstats + 4, D->d_fb_list, D->d_gstats + 2, D->timing ? D->d_cand.data() : nullptr);
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
                                                                    D->d_fb_list, D->d_gstats + 2, D->d_nn_idx, D->d_nn_d2, sel, D->d_gstats + 3,
                                                                    D->d_gstats + 6);
    else
      knn_list_kernel<MODE, false><<<fb_blocks, KNN_THREADS, 0, st>>>(D->d_nodes, D->n_nodes, pts, perm, qs, n, pc, max_sqdist,
                                                                     D->d_fb_list, D->d_gstats + 2, D->d_nn_idx, D->d_nn_d2, sel, D->d_gstats + 3,
                                                                     D->d_gstats + 6);
    D->ctr.kernel_launches += 2;
  } else {
    // device-resident map without a live point: n_nodes = 0, the traversal below answers with empty lists as for an empty snapshot
    if (D->tree_free && D->n_nodes > 0) { h->err = "device-resident map: the cell-list index is required (map extent too large for it?)"; return MALIO_ERR_STATE; }
    if (int rc = need_boxes()) return rc;
    const int lanes = pick_lanes(n, D->sm_count);
    if (smem_stack)
      knn_kernel<MODE, true><<<knn_blocks(n, lanes), KNN_THREADS, 0, st>>>(D->d_nodes, D->n_nodes, pts, perm, qs, n, lanes, pc,
                                                                          max_sqdist, world, D->d_nn_idx, D->d_nn_d2, sel, D->d_gstats + 6);
    else
      knn_kernel<MODE, false><<<knn_blocks(n, lanes), KNN_THREADS, 0, st>>>(D->d_nodes, D->n_nodes, pts, perm, qs, n, lanes, pc,
                                                                           max_sqdist, world, D->d_nn_idx, D->d_nn_d2, sel, D->d_gstats + 6);
    D->ctr.kernel_launches += 1;
  }
  CUDA_TRY(cudaGetLastError());
  return MALIO_OK;
}
template int sort_queries<0>(malio_handle*, DeviceState*, uint32_t, const PassConst&, int, const float*);
template int sort_queries<1>(malio_handle*, DeviceState*, uint32_t, const PassConst&, int, const float*);
template int run_knn<0>(malio_handle*, DeviceState*, uint32_t, const malio_scan_pt*, const uint32_t*, const PassConst&, float, const float*);
template int run_knn<1>(malio_handle*, DeviceState*, uint32_t, const malio_scan_pt*, const uint32_t*, const PassConst&, float, const float*);

int fetch_knn_stats(malio_handle* h, DeviceState* D, cudaStream_t st) {
  CUDA_TRY(cudaMemcpyAsync(D->h_gstats + 2, D->d_gstats + 2, 6 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  return MALIO_OK;
}

int knn_fault(malio_handle* h, const DeviceState* D) {
  if (D->h_gstats[6] & FAULT_STACK_OVERFLOW) {
    h->err = "k-NN traversal stack overflow: the snapshot is deeper than the max_depth declared at upload";
    return MALIO_ERR_TREE_TOO_DEEP;
  }
  return MALIO_OK;
}

}  // namespace malio_devstate

namespace malio_dev {

static int ensure_map_buffers(malio_handle* h, DeviceState* D, uint32_t n) {
  if (n <= D->d_nodes.size() / 4 && D->d_nodes) return MALIO_OK;   // (slot mode grows d_mpts / d_cov only: no tree records there)
  uint32_t cap = n + n / 8 + 1024;
  if (cap < h->cfg.max_map_nodes) cap = h->cfg.max_map_nodes;
  if (int rc = malio_buf::allocate_group(h, D->stream, {{D->d_nodes, (size_t)cap * 4}, {D->d_mpts, cap}, {D->d_cov, cap}, {D->d_parent, cap},
                                                        {D->d_arrived, cap}}))
    return rc;
  D->slot_store = false;   // d_mpts / d_cov now hold the snapshot: the next malio_map_build re-creates the slot storage (grow_slots)
  return MALIO_OK;
}

// after the snapshot is resident (d_nodes, d_mpts, d_cov): cell-list index for the k-NN fast path.
// Cell edge: cfg.knn_cell_size (> 0 fixed, < 0 index off, 0 automatic: start at 1 m = twice the reference's map voxel,
// filter_size_map 0.5, and keep 2..9 live points per occupied cell).  root = host copy of node 0 (bounds every live point).
static int finish_map_upload(malio_handle* h, DeviceState* D, const malio_map_node* root, uint32_t n, uint32_t depth) {
  D->n_nodes = n; D->depth = depth;
  CUDA_TRY(cudaMemsetAsync(D->d_gstats + 6, 0, sizeof(uint32_t), D->stream));   // a new map: no traversal has faulted on it
  D->h_gstats[6] = 0;
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
  DeviceState* D = h->dev.get();
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
  DeviceState* D = h->dev.get();
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
  DeviceState* D = h->dev.get();
  CUDA_TRY(cudaSetDevice(D->device));
  if (D->slot_store && n <= D->d_ids.size()) return MALIO_OK;
  uint32_t cap = n + n / 2 + 4096;
  if (cap < h->cfg.max_map_nodes) cap = h->cfg.max_map_nodes;
  if (!D->tree_free) keep = 0;   // d_mpts / d_cov hold a snapshot, not slots
  CUDA_TRY(malio_buf::grow_keep(D->stream, {{D->d_mpts, cap, keep}, {D->d_cov, cap, keep}, {D->d_ids, cap, keep}}));
  // the tree records belong to the snapshot mode; they are re-created by the next malio_upload_map* call
  D->d_nodes.release(); D->d_parent.release(); D->d_arrived.release();
  D->slot_store = true;
  return MALIO_OK;
}
// (re)build the cell-list index over the n_slots slots; box = {x_min,x_max,y_min,y_max,z_min,z_max} of the live points
int index_from_slots(malio_handle* h, uint32_t n_slots, const float box[6]) {
  DeviceState* D = h->dev.get();
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
  DeviceState* D = h->dev.get();
  if (!D->map_ready || D->tree_free) { h->err = "download_map_nodes needs a snapshot uploaded with malio_upload_map*"; return MALIO_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(D->device));
  const uint32_t n = D->n_nodes < cap ? D->n_nodes : cap;
  if (D->refit_pending) { CUDA_TRY(cudaStreamSynchronize(D->stream2)); D->refit_pending = false; }
  CUDA_TRY(cudaMemcpy(out, D->d_nodes, (size_t)n * sizeof(malio_map_node), cudaMemcpyDeviceToHost));
  return MALIO_OK;
}

}  // namespace malio_dev
