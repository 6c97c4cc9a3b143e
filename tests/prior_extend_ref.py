"""numpy float32 restatement of the session layer (malio_prior_map_extend, include/malio_b200.h) and of the window over
prior ∪ session, built on prior_map_ref.py (cube, slabs, half-open boxes) and map_incr_ref.py (calc_dist):
  - box: per axis lo = floor(x / ds) * ds, hi = lo + ds in float32 (Add_Points(.., true), ikd_Tree.cpp:491-497); a candidate is
    eligible when it lies in its own box and in neither neighbour's;
  - admission: eligible candidates (MAP_ADD / MAP_ADD_NO_DOWNSAMPLE) whose box holds no live point at the call's start;
  - fold: the admitted MAP_ADD candidates of one box in caller order, by the down-sample rule of ikd_Tree.cpp:498-534;
  - order: fold winners by ascending caller index, then admitted no-downsample points by caller index; ids -1 - k.
`variant` switches in one deliberate deviation, so that a test can show it sees the difference: "le_fold" (<= for the fold's
strict <), "session_only" (admission against the session's live points only), "sequential" (admission after the call's own
earlier inserts) and "double_box" (the box in float64)."""
import numpy as np

import map_incr_ref as MI
import prior_map_ref as R
from malio_b200 import capi

F = np.float32
SESSION_NY = F(0.001)
VARIANTS = ("le_fold", "session_only", "sequential", "double_box")
TILE = F(25.0)


def vox(v, ds, variant=None):
    """Per-coordinate box of v (float32 array): (f, lo, hi, sole) with sole = inside its own box and neither neighbour's."""
    v = np.asarray(v, F)
    if variant == "double_box":
        d = np.float64(F(ds))
        vd = v.astype(np.float64)
        f = np.floor(vd / d)
        lo = f * d
        hi = lo + d
        return f, lo, hi, (lo <= vd) & (vd < hi)
    d = F(ds)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(v / d).astype(F)
        lo = (f * d).astype(F)
        hi = (lo + d).astype(F)
        lm = ((f - F(1)) * d).astype(F)
        lp = ((f + F(1)) * d).astype(F)
        sole = (lo <= v) & (v < hi) & ~((lm <= v) & (v < (lm + d).astype(F))) & ~((lp <= v) & (v < (lp + d).astype(F)))
    return f, lo, hi, sole


def boxes(world, ds, variant=None):
    """(f [N,3], lo [N,3], hi [N,3], eligible [N]) of every point."""
    f, lo, hi, sole = vox(np.asarray(world, F).reshape(-1, 3), ds, variant)
    return f, lo, hi, np.all(sole, axis=1)


def _count_in_boxes(lo, hi, pts):
    """Points of pts (float32 [M,3]) inside each half-open box [lo, hi) (in the boxes' type), through a hash of pts' cells."""
    n = lo.shape[0]
    out = np.zeros(n, np.int64)
    if n == 0 or len(pts) == 0:
        return out
    pts = np.asarray(pts, F)
    size = np.float64(np.max(hi - lo)) if n else 1.0
    cell = np.floor(pts.astype(np.float64) / size).astype(np.int64)
    table = {}
    for i, c in enumerate(map(tuple, cell)):
        table.setdefault(c, []).append(i)
    pc = pts.astype(lo.dtype)
    for k in range(n):
        base = np.floor(lo[k].astype(np.float64) / size).astype(np.int64)
        cand = []
        for dz in (-1, 0, 1, 2):
            for dy in (-1, 0, 1, 2):
                for dx in (-1, 0, 1, 2):
                    cand += table.get((base[0] + dx, base[1] + dy, base[2] + dz), [])
        if cand:
            q = pc[cand]
            out[k] = int(np.sum(np.all((lo[k] <= q) & (q < hi[k]), axis=1)))
    return out


def fold(idx, world, ds, variant=None):
    """Add_Points(world[idx], true) into a box that was empty, idx in caller order, all candidates with normal_y SESSION_NY.
    Returns the winner's caller index."""
    w = np.asarray(world, F)
    _, lo, hi, _ = vox(w[idx[0]], ds)
    mid = (lo.astype(np.float64) + (hi - lo).astype(np.float64) / 2.0).astype(F)                     # :497-499
    ds8 = F(F(ds) / F(8))
    lt = (lambda a, b: a <= b) if variant == "le_fold" else (lambda a, b: a < b)
    win = idx[0]
    dw = MI.calc_dist(w[win], mid)
    for p in idx[1:]:
        dp = MI.calc_dist(w[p], mid)
        if lt(dw, ds8) and lt(dp, ds8):
            keep_w = lt(SESSION_NY, SESSION_NY)                                                     # :511, equal normal_y
        else:
            keep_w = lt(dw, dp)                                                                     # :517
        if not keep_w:
            win, dw = p, dp
    return win


def extend(cls, world, ds, live_xyz, live_ids, variant=None):
    """One extend call on the classes and world points of a scan.  live_xyz / live_ids: the window's live points at the call's
    start.  Returns dict(inserted = caller indices in session order, n_candidates, n_admitted, add_mask, nods_mask)."""
    cls = np.asarray(cls).reshape(-1)
    w = np.asarray(world, F).reshape(-1, 3)
    cand = (cls == capi.MAP_ADD) | (cls == capi.MAP_ADD_NO_DOWNSAMPLE)
    f, lo, hi, ok = boxes(w, ds, variant)
    elig = cand & ok
    live_xyz = np.asarray(live_xyz, F).reshape(-1, 3)
    ref = live_xyz[np.asarray(live_ids) < 0] if variant == "session_only" else live_xyz
    ci = np.flatnonzero(elig)
    adm = np.zeros(len(cls), bool)
    if variant == "sequential":
        placed = ref
        for i in ci:
            if _count_in_boxes(lo[i:i + 1], hi[i:i + 1], placed)[0] == 0:
                adm[i] = True
                placed = np.concatenate([placed, w[i:i + 1]])
    else:
        adm[ci] = _count_in_boxes(lo[ci], hi[ci], ref) == 0
    add = np.flatnonzero(adm & (cls == capi.MAP_ADD))
    runs = {}
    for i in add:
        runs.setdefault(tuple(f[i].tolist()), []).append(i)
    winners = sorted(fold(np.array(r), w, ds, variant) for r in runs.values())
    nods = np.flatnonzero(adm & (cls == capi.MAP_ADD_NO_DOWNSAMPLE))
    return dict(inserted=np.array(list(winners) + list(nods), np.int64), n_candidates=int(cand.sum()), n_admitted=int(adm.sum()),
                add_mask=adm & (cls == capi.MAP_ADD), nods_mask=adm & (cls == capi.MAP_ADD_NO_DOWNSAMPLE))


def tile_order(xyz):
    """The prior's slot order: tile keys (z, y, x) of floor(x / 25) in float, input order within a tile."""
    t = np.floor(np.asarray(xyz, F) / TILE).astype(np.int64)
    return np.lexsort((np.arange(len(t)), t[:, 0], t[:, 1], t[:, 2]))


class SessionWindow:
    """The window over prior ∪ session: cube, live points in slot order (xyz, normal_y, ids) and the session."""

    def __init__(self, xyz, normal_y, ids, cube_len, det_range):
        order = tile_order(xyz)
        self.pxyz = np.asarray(xyz, F)[order]
        self.pny = np.asarray(normal_y, F)[order]
        self.pids = np.asarray(ids, np.int32)[order]
        self.cube_len, self.det_range = float(cube_len), float(det_range)
        self.cube = None
        self.sxyz = np.zeros((0, 3), F)
        self.xyz, self.ny, self.ids = np.zeros((0, 3), F), np.zeros(0, F), np.zeros(0, np.int32)

    def session_ids(self):
        return (-1 - np.arange(len(self.sxyz))).astype(np.int32)

    def _enter(self, m_prior, m_sess):
        self.xyz = np.concatenate([self.xyz, self.pxyz[m_prior], self.sxyz[m_sess]])
        self.ny = np.concatenate([self.ny, self.pny[m_prior], np.full(int(m_sess.sum()), SESSION_NY, F)])
        self.ids = np.concatenate([self.ids, self.pids[m_prior], self.session_ids()[m_sess]])
        return int(m_prior.sum() + m_sess.sum())

    def end(self):
        """malio_map_build* ended the window: the next step builds it afresh."""
        self.cube = None

    def step(self, pos):
        """One window call.  Returns (initialized, moved, slabs, n_entered)."""
        if self.cube is None:
            self.cube = R.init_cube(pos, self.cube_len)
            self.xyz, self.ny, self.ids = np.zeros((0, 3), F), np.zeros(0, F), np.zeros(0, np.int32)
            return True, False, np.zeros((0, 6), F), self._enter(R.in_box(self.pxyz, self.cube), R.in_box(self.sxyz, self.cube))
        old = self.cube
        moved, self.cube, slabs = R.segment(old, pos, self.cube_len, self.det_range)
        if not moved:
            return False, False, slabs, 0
        keep = ~R.in_any(self.xyz, slabs)
        self.xyz, self.ny, self.ids = self.xyz[keep], self.ny[keep], self.ids[keep]
        n = self._enter(R.in_box(self.pxyz, self.cube) & ~R.in_box(self.pxyz, old),
                        R.in_box(self.sxyz, self.cube) & ~R.in_box(self.sxyz, old))
        return False, True, slabs, n

    def extend(self, cls, world, ds, variant=None):
        """One extend call: the restated report and the session / window after it."""
        r = extend(cls, world, ds, self.xyz, self.ids, variant)
        pts = np.asarray(world, F).reshape(-1, 3)[r["inserted"]]
        k0 = len(self.sxyz)
        self.sxyz = np.concatenate([self.sxyz, pts])
        inc = R.in_box(pts, self.cube)
        self.xyz = np.concatenate([self.xyz, pts[inc]])
        self.ny = np.concatenate([self.ny, np.full(int(inc.sum()), SESSION_NY, F)])
        self.ids = np.concatenate([self.ids, (-1 - (k0 + np.flatnonzero(inc))).astype(np.int32)])
        return dict(n_candidates=r["n_candidates"], n_admitted=r["n_admitted"], n_inserted=len(pts), n_session=len(self.sxyz))
