"""Test infrastructure for map_incremental's per-point decision (laserMapping.cpp:398-446): a plain numpy restatement in the
reference's types, and planted scenes whose scan points sit exactly on the decision's comparisons.

The restatement takes the neighbour lists as given (the device's own, from aux()), together with the point array their
indices refer to (snapshot nodes, or the device-resident map's slots), so that it judges the decision alone; the lists are
pinned separately (pyoracle.knn_snapshot, np_mapops.knn_bruteforce).  No oracle import."""
import numpy as np

import world_ref
from malio_b200 import capi

F = np.float32
NONE = 0xFFFFFFFF
MUTANTS = ("le_for_lt", "or_for_and", "mid_float64", "no_cnt_guard", "ge_at_406")


def voxel_mid(w, fs, dtype=F):
    """floor(w / fs) * fs + 0.5 * fs in float64 (:417-419), rounded to dtype."""
    return (np.floor(np.asarray(w, np.float64) / fs) * fs + 0.5 * fs).astype(dtype)


def calc_dist(a, b):
    """calc_dist (:109-115) elementwise over the last axis, in a's and b's type, ((dx*dx + dy*dy) + dz*dz), no FMA."""
    d = a - b
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def decide(world, normal_y, nn_idx, map_xyz, cov_threshold, fs, ekf_inited, mutant=None):
    """The decision on given world points (float32 [N,3]), normal_y [N], neighbour lists [N,5] (uint32, 0xFFFFFFFF = none;
    -1 from int32 arrays is the same) and the point array they index.  mutant: one of MUTANTS (a deliberately wrong variant,
    to show that a planted set reaches each comparison) or None.  Returns (cls uint8[N] with capi.MAP_*, world float32[N,3]
    zero on skipped points)."""
    w = np.asarray(world, F).reshape(-1, 3)
    n = w.shape[0]
    ny = np.asarray(normal_y, F).reshape(n).astype(np.float64)
    keep = ~(ny >= cov_threshold) if mutant == "ge_at_406" else ~(ny > cov_threshold)              # :406
    idx = np.asarray(nn_idx).reshape(n, capi.K).astype(np.int64) & NONE
    valid = idx != NONE
    cnt = valid.sum(axis=1)                                                                        # Nearest_Points[i].size()
    mpts = np.asarray(map_xyz, F).reshape(-1, 3)
    T = np.float64 if mutant == "mid_float64" else F
    mid = voxel_mid(w, fs, T)
    wt = w.astype(T)
    dist = calc_dist(wt, mid)
    q = mpts[np.where(valid, idx, 0)] if mpts.shape[0] else np.zeros((n, capi.K, 3), F)
    q = q.astype(T)
    far = np.abs(q[:, 0] - mid).astype(np.float64) > 0.5 * fs                                     # :421 per axis
    nods = np.any(far, axis=1) if mutant == "or_for_and" else np.all(far, axis=1)
    dj = calc_dist(q, mid[:, None, :])
    closer = (dj <= dist[:, None]) if mutant == "le_for_lt" else (dj < dist[:, None])              # :430
    closer &= valid
    guard = np.ones(n, bool) if mutant == "no_cnt_guard" else cnt >= capi.K                        # :428
    drop = guard & np.any(closer, axis=1)
    cls = np.where(nods, capi.MAP_ADD_NO_DOWNSAMPLE, np.where(drop, capi.MAP_DROP, capi.MAP_ADD))
    cls = np.where((cnt > 0) & bool(ekf_inited), cls, capi.MAP_ADD)                                # :411, :439-440
    cls = np.where(keep, cls, capi.MAP_SKIP).astype(np.uint8)
    return cls, np.where(keep[:, None], w, F(0)).astype(F)


def map_incremental_ref(state, temporal_comp, body_xyz, lidar, normal_y, nn_idx, map_xyz, cov_threshold, fs, ekf_inited,
                        mutant=None):
    """map_incremental on a scan (body xyz, lidar ids): world points from world_ref.register_world for the updated state,
    then decide()."""
    w = world_ref.register_world(state, temporal_comp, body_xyz, lidar, 0.0)[:, :3]
    return decide(w, normal_y, nn_idx, map_xyz, cov_threshold, fs, ekf_inited, mutant)


def slot_points(m):
    """map_download() -> float32[max slot + 1, 3] indexed by slot (dead slots zero; no list refers to them)."""
    out = np.zeros((int(m["slots"].max()) + 1 if len(m["slots"]) else 1, 3), F)
    out[m["slots"]] = m["xyz"]
    return out


# ------------------------------------------------------------------ planted scenes
# Each planted scan point gets its own cluster of map points, at least SITE metres from every other cluster, so that its five
# nearest map points are the ones planted for it.  `expect` holds the class a point was built for; NOT_NODS means "ADD or
# DROP, not ADD_NO_DOWNSAMPLE".
SITE = 8.0
NOT_NODS = 255


def _nextafter(x, toward):
    return np.nextafter(F(x), F(toward)).astype(F)


class Scene:
    def __init__(self, origin=(0.0, 0.0, 0.0)):
        self.origin = np.asarray(origin, np.float64)
        self.w, self.map, self.expect, self.group, self.fs = [], [], [], [], []
        self.n_sites = 0
        self.n_zero = 0

    def site(self):
        """Centre of the next free site: an 8 x 8 x n lattice of SITE-metre cells from the origin."""
        i = self.n_sites
        self.n_sites += 1
        return self.origin + SITE * np.array([i % 8, (i // 8) % 8, i // 64], np.float64)

    def add(self, w, pts, expect, group, fs):
        self.w.append(np.asarray(w, F)); self.map.extend(np.asarray(pts, F)); self.expect.append(expect)
        self.group.append(group); self.fs.append(fs)

    def arrays(self):
        return (np.array(self.w, F).reshape(-1, 3), np.array(self.map, F).reshape(-1, 3), np.array(self.expect, np.int64),
                np.array(self.group), np.array(self.fs, np.float64))

    # -- voxel faces: w on a voxel corner k*fs (and one float32 ulp below / above on each axis); n0 0.25 fs below w on every
    # axis.  In the upper voxel on all three axes |n0 - mid| > 0.5 fs everywhere: ADD_NO_DOWNSAMPLE; below it on any axis: not.
    def voxel_faces(self, fs, group="face", zero_x=False):
        """zero_x: the corners sit on x = 0 (between two lattice planes, half a site up), the middle variant at x = -0.0 and
        the others at the smallest subnormals; y and z one ulp above their corner (upper voxel)."""
        step = next(s for s in range(1, 11) if abs(s * fs - round(s * fs)) < 1e-9)   # k*fs on x is a whole metre: for an
        uyz = (1,) if zero_x else (-1, 0, 1)                                         # inexact fs, w/fs rounds onto k
        for ux in (-1, 0, 1):
            for uy in uyz:
                for uz in uyz:
                    if zero_x:
                        j = self.n_zero
                        self.n_zero += 1
                        c = self.origin + SITE * np.array([0.0, j % 8, j // 8 + 0.5])
                    else:
                        c = self.site()
                    k = np.round(c / fs) + np.array([0.0, 3.0, 1.0])   # y, z: k*fs not a float32 in general
                    k[0] = 0.0 if zero_x else np.round(c[0] / (fs * step)) * step
                    corner = (k * fs).astype(F)
                    if zero_x:
                        corner[0] = F(-0.0)
                    w = corner.copy()
                    for a, u in enumerate((ux, uy, uz)):
                        if u:
                            w[a] = _nextafter(w[a], np.inf if u > 0 else -np.inf)
                    upper = np.floor(w.astype(np.float64) / fs) == k
                    n0 = (w.astype(np.float64) - 0.25 * fs).astype(F)
                    fill = [corner.astype(np.float64) + fs * r * np.asarray(v) for r, v in
                            ((2.2, (1, 0, 0)), (2.4, (0, 1, 0)), (2.6, (0, 0, 1)), (2.8, (-0.577, -0.577, -0.577)))]
                    self.add(w, [n0] + fill, capi.MAP_ADD_NO_DOWNSAMPLE if upper.all() else NOT_NODS, group, fs)

    # -- the no-downsample test (:421): w 0.45 fs from mid towards a corner, n0 across the faces: exactly 0.5 fs from mid on
    # the axes in `axes` (or one ulp further), 0.6 fs on the others.  Exact: not all three > 0.5 fs, and every neighbour is
    # farther from mid than w: ADD.  One ulp further: ADD_NO_DOWNSAMPLE.
    def no_downsample(self, fs, axes, above, group="nods"):
        c = self.site()
        m = voxel_mid(c, fs)
        s = np.array([1.0, -1.0, 1.0])
        w = (m + 0.45 * fs * s).astype(F)
        n0 = (m + 0.6 * fs * s).astype(F)
        for a in axes:
            n0[a] = F(m[a] + 0.5 * fs * s[a])
            assert np.float64(abs(n0[a] - m[a])) == 0.5 * fs
            if above:
                n0[a] = _nextafter(n0[a], n0[a] + s[a])
        r = float(np.linalg.norm(n0.astype(np.float64) - w))
        fill = [w + t * r * s / np.sqrt(3.0) for t in (1.5, 2.0, 2.5, 3.0)]
        self.add(w, [n0] + fill, capi.MAP_ADD_NO_DOWNSAMPLE if above else capi.MAP_ADD, group, fs)

    # -- distance ties (:430): the neighbour at position j has dj == dist exactly (a mirror image of w through mid on its
    # farthest axis, or w itself for j = 0): kept, ADD; or one ulp closer to mid: DROP.  The other four lie on the ray from mid
    # through w, farther from mid than w, at distances from w below / above the tie's.
    def tie(self, w, fs, j, exact, group="tie"):
        w = np.asarray(w, F)
        m = voxel_mid(w, fs)
        d = (w - m).astype(F)
        a = int(np.argmax(np.abs(d)))
        t = w.copy()
        if j:
            t[a] = F(2.0 * np.float64(m[a]) - np.float64(w[a]))
            assert t[a] - m[a] == -d[a]
        assert calc_dist(t, m) == calc_dist(w, m)
        if not exact:
            while not calc_dist(t, m) < calc_dist(w, m):
                t[a] = _nextafter(t[a], m[a])
        d64 = d.astype(np.float64)
        u = d64 / np.linalg.norm(d64)
        rt = 2.0 * abs(d64[a]) if j else 0.0
        scale = rt if j else np.linalg.norm(d64)
        ts = [scale * (i + 1) / (j + 1) for i in range(j)] + [scale * (1.3 + 0.25 * i) if j else scale * (0.3 + 0.2 * i)
                                                             for i in range(4 - j)]
        fill = [w + ti * u for ti in ts]
        self.add(w, fill[:j] + [t] + fill[j:], capi.MAP_ADD if exact else capi.MAP_DROP, group, fs)

    def tie_site(self, fs):
        """A w well inside its voxel (|w - mid| between 0.08 and 0.22 fs on each axis) at the next site."""
        m = voxel_mid(self.site(), fs)
        return (m + fs * np.array([0.21, -0.16, 0.09])).astype(F)

    # -- mid rounded to float32 (:417-419): n0 placed where |n0 - mid| > 0.5 fs on the x axis holds for the float32 mid but not
    # for the float64 one (or the other way round); w and n0 as in no_downsample otherwise.
    def mid_rounding(self, fs, group="midround"):
        for tries in range(64 * 8):
            if tries % 8 == 0:
                c0 = self.site()
            c = c0 + np.array([fs * (tries % 8), 0.0, 0.0])   # neighbouring voxels of one site
            m32 = voxel_mid(c, fs)
            m64 = voxel_mid(c, fs, np.float64)
            base = F(m64[0] - 0.5 * fs)
            for step in range(-3, 4):
                x = base
                for _ in range(abs(step)):
                    x = _nextafter(x, np.inf if step > 0 else -np.inf)
                f32 = np.float64(abs(x - m32[0])) > 0.5 * fs
                f64 = abs(np.float64(x) - m64[0]) > 0.5 * fs
                if f32 != f64:
                    s = np.array([-1.0, 1.0, 1.0])
                    w = (m32 + 0.45 * fs * s).astype(F)
                    n0 = (m32 + 0.6 * fs * s).astype(F)
                    n0[0] = x
                    r = float(np.linalg.norm(n0.astype(np.float64) - w))
                    fill = [w + t * r * s / np.sqrt(3.0) for t in (1.5, 2.0, 2.5, 3.0)]
                    self.add(w, [n0] + fill, capi.MAP_ADD_NO_DOWNSAMPLE if f32 else capi.MAP_ADD, group, fs)
                    return
        raise AssertionError(f"no float32 / float64 mid disagreement found for fs={fs}")


def planted_scene(origin=(0.0, 0.0, 0.0), face_fs=(0.5, 0.2, 0.1, 0.3), zero_x=True):
    """Every planted edge on one scan (identity state: the world points are the planted points): voxel faces for each fs in
    face_fs (zero_x: also on x = -0.0 and the subnormals), the no-downsample test on each axis alone and all three, exact and
    one ulp above, distance ties at j = 0..4 exact and one ulp closer, and a float32-mid rounding case for fs 0.2, 0.1, 0.3.
    Returns a Scene."""
    sc = Scene(origin)
    for fs in face_fs:
        sc.voxel_faces(fs, group=f"face fs={fs}")
        if zero_x:
            sc.voxel_faces(fs, group=f"face x=-0.0 fs={fs}", zero_x=True)
    for axes in ((0,), (1,), (2,), (0, 1, 2)):
        for above in (False, True):
            sc.no_downsample(0.5, axes, above, group=f"nods axes={axes} {'+1ulp' if above else 'exact'}")
    for j in range(capi.K):
        for exact in (True, False):
            sc.tie(sc.tie_site(0.5), 0.5, j, exact, group=f"tie j={j} {'exact' if exact else '-1ulp'}")
    for fs in (0.2, 0.1, 0.3):
        sc.mid_rounding(fs, group=f"midround fs={fs}")
    return sc


def short_list_scene(n_map, fs=0.5, origin=(0.0, 0.0, 0.0)):
    """A map of n_map points, all closer to mid than the scan point w is, so that Nearest_Points holds min(n_map, 5) points:
    with the cnt >= 5 guard (:428) the point is DROPped only when the list is full, and ADDed otherwise (n_map = 0: cnt = 0,
    :439-440).  Three copies of w.  Returns (w float32[3,3], map float32[n_map,3], expected class)."""
    m = voxel_mid(np.asarray(origin, np.float64) + 0.1, fs).astype(np.float64)
    w = np.tile((m + 0.2 * fs).astype(F), (3, 1))
    pts = np.array([m + fs * np.array([0.02 * (i + 1), 0.011 * i, -0.013 * i]) for i in range(n_map)], F).reshape(-1, 3)
    return w, pts, (capi.MAP_DROP if n_map >= capi.K else capi.MAP_ADD)


def scan_records(body_xyz, L=1, lidar=None):
    """capi.SCAN_PT records of body points, LiDARs round-robin (or `lidar`), pose-table index 0."""
    n = body_xyz.shape[0]
    pts = np.zeros(n, capi.SCAN_PT)
    pts["xyz"] = np.asarray(body_xyz, F)
    pts["lidar"] = (np.arange(n) % L if lidar is None else np.asarray(lidar)).astype(np.uint16)
    pts["table_idx"] = 0
    return pts


def check_expect(cls, expect):
    """Every planted point reached the class it was built for."""
    cls = np.asarray(cls).astype(np.int64)
    ok = np.where(expect == NOT_NODS, (cls == capi.MAP_ADD) | (cls == capi.MAP_DROP), cls == expect)
    return np.flatnonzero(~ok)
