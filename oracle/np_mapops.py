"""numpy mirror of the device-resident map's delta protocol (include/malio_mapsync.hpp).  TEST INFRASTRUCTURE ONLY.

A flat table of (xyz, normal_y, id, live) that receives exactly the calls the device receives:
  build / add_points (plain append) / delete_boxes (half-open boxes) / sync_voxels (replace the content of each box).
tests/test_mapops_cpu.py drives the REAL ikd_Tree.cpp (oracle/_ref) and this mirror with the same call stream and checks
after every scan that the mirror's live set equals KD_TREE::flatten() — i.e. the protocol is exact whatever the tree's
topology; the GPU tests then check the device against the same stream."""
import numpy as np

F = np.float32
NONE = np.uint32(0xFFFFFFFF)
TIE_WINDOW = F(1e-10)       # PointType_CMP's window; (double)v < 1e-10 <=> v < 1e-10f for a float v
KD_MARGIN = 1e-5            # relative: float32 calc_dist is within 5 * 2^-24 of the exact distance (three positive terms)


def in_box(xyz, box):
    """Delete_by_range's / Search_by_range's point test (ikd_Tree.cpp:807, :1270): half-open per axis, min <= p < max, in
    float32.  -0.0 and +0.0 compare equal; a degenerate box (min == max) holds nothing."""
    b = np.asarray(box, F).reshape(6)
    p = np.asarray(xyz, F).reshape(-1, 3)
    return np.all((b[:3] <= p) & (p < b[3:]), axis=1)


def calc_dist(q, p):
    """calc_dist's float32 expression, left to right: ((dx*dx + dy*dy) + dz*dz).  q [m,3] against p [n,3] -> [m,n]."""
    q = np.asarray(q, F); p = np.asarray(p, F)
    dx = q[:, None, 0] - p[None, :, 0]; dy = q[:, None, 1] - p[None, :, 1]; dz = q[:, None, 2] - p[None, :, 2]
    return (dx * dx + dy * dy) + dz * dz


def _six_best(d, slots):
    """Six smallest by (distance, slot) of every row of d [m,n] float32 (n >= 6); slots [n] or [m,n]."""
    s = slots.astype(np.uint64)
    key = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | (s if s.ndim == 2 else s[None, :])   # d >= 0: bits order like values
    part = np.argpartition(key, 5, axis=1)[:, :6]
    kp = np.take_along_axis(key, part, 1)
    o = np.argsort(kp, axis=1)
    return np.take_along_axis(part, o, 1)


def _brute(xyz, slots, q, out_i, out_d, rows):
    n = xyz.shape[0]
    step = max(1, 4_000_000 // max(n, 1))
    for a in range(0, len(rows), step):
        r = rows[a:a + step]
        d = calc_dist(q[r], xyz)
        if n < 6:
            d = np.concatenate([d, np.full((len(r), 6 - n), np.inf, F)], 1)
            s = np.concatenate([slots, np.full(6 - n, NONE, np.uint32)])
        else:
            s = slots
        j = _six_best(np.where(np.isfinite(d), d, F(np.inf)), s)
        out_d[r] = np.take_along_axis(d, j, 1)
        out_i[r] = np.where(np.isfinite(out_d[r]), s[j], NONE)


def knn_bruteforce(xyz_live, slots, queries, k=5, kd_from=4096, kd_k=24, stats=None):
    """Exact k nearest of every query among the live points (xyz_live [n,3] float32 at slot indices `slots`), ordered by
    (calc_dist in float32, slot): the device-resident map's tie rule (Top6T::lt).  Missing entries are 0xFFFFFFFF / +inf.
    Returns (idx uint32 [m,k], d2 float32 [m,k], ties) with ties = the number of queries whose six best hold two adjacent
    finite distances within 1e-10f (what malio_counters.knn_tie_queries counts).
    Maps of kd_from points or more take candidates from a float64 cKDTree (kd_k per query); a query is settled by its
    candidates only if the float64 distance of the last one exceeds the float32 6th best by the relative KD_MARGIN, which
    no float32 rounding of a point outside the candidates can bridge.  Every other query is searched by brute force.
    stats (dict, optional) receives the number of such fallbacks."""
    xyz = np.ascontiguousarray(xyz_live, F).reshape(-1, 3)
    slots = np.ascontiguousarray(slots, np.uint32).reshape(-1)
    q = np.ascontiguousarray(queries, F).reshape(-1, 3)
    m, n = q.shape[0], xyz.shape[0]
    oi = np.full((m, 6), NONE, np.uint32); od = np.full((m, 6), np.inf, F)
    fallback = np.zeros(0, np.int64)
    if n == 0:
        pass
    elif n < kd_from or n <= kd_k:
        _brute(xyz, slots, q, oi, od, np.arange(m))
    else:
        from scipy.spatial import cKDTree
        dd, jj = cKDTree(xyz.astype(np.float64)).query(q.astype(np.float64), k=kd_k)
        d32 = (lambda dx, dy, dz: (dx * dx + dy * dy) + dz * dz)(*(q[:, None, a] - xyz[jj][:, :, a] for a in range(3)))
        s32 = slots[jj]
        j = _six_best(d32, s32)
        od[:] = np.take_along_axis(d32, j, 1); oi[:] = np.take_along_axis(s32, j, 1)
        complete = dd[:, -1] ** 2 > od[:, 5].astype(np.float64) * (1.0 + KD_MARGIN)
        fallback = np.flatnonzero(~complete)
        if len(fallback):
            _brute(xyz, slots, q, oi, od, fallback)
    if stats is not None:
        stats["fallback"] = int(len(fallback))
    fin = np.isfinite(od)
    with np.errstate(invalid="ignore"):
        close = fin[:, 1:] & (np.abs(od[:, 1:] - od[:, :-1]) < TIE_WINDOW)
    ties = int(np.any(close, axis=1).sum())
    return oi[:, :k].copy(), od[:, :k].copy(), ties


class MirrorMap:
    def __init__(self):
        self.xyz = np.zeros((0, 3), F); self.ny = np.zeros(0, F); self.ids = np.zeros(0, np.int64); self.live = np.zeros(0, bool)

    def build(self, xyz, normal_y, ids):
        self.xyz = np.array(xyz, F).reshape(-1, 3).copy(); self.ny = np.array(normal_y, F).copy()
        self.ids = np.array(ids, np.int64).copy(); self.live = np.ones(len(self.ids), bool)

    def add_points(self, xyz, normal_y, ids):
        self.xyz = np.concatenate([self.xyz, np.array(xyz, F).reshape(-1, 3)]); self.ny = np.concatenate([self.ny, np.array(normal_y, F)])
        self.ids = np.concatenate([self.ids, np.array(ids, np.int64)]); self.live = np.concatenate([self.live, np.ones(len(ids), bool)])

    def _inside(self, b):
        return self.live & in_box(self.xyz, b)

    def delete_boxes(self, boxes):
        n = 0
        for b in np.array(boxes, F).reshape(-1, 6):
            m = self._inside(b); n += int(m.sum()); self.live[m] = False
        return n

    def sync_voxels(self, sync):
        kill = np.zeros(len(self.live), bool)
        for b in sync["boxes"]:
            kill |= self._inside(b)
        self.live[kill] = False
        self.add_points(sync["xyz"], sync["normal_y"], sync["ids"])

    def live_points(self):
        return self.xyz[self.live], self.ny[self.live], self.ids[self.live]
