"""GPU edges of the device-resident map (malio_mapops.cu), without the reference checkout: every scenario drives one handle in
device-map mode and a flat numpy mirror (np_mapops.in_box, the stable compaction rule) with the same calls, and checks
  - malio_map_download = the mirror's live set in the mirror's slot order, ids included (the compaction is stable),
  - the kill counts of malio_map_delete_boxes / malio_map_sync_voxels,
  - malio_knn = np_mapops.knn_bruteforce over the downloaded (xyz, slot), bit for bit, ties in (distance, slot) order, and
    the knn_tie_queries delta = the reference's tie count.
Scenarios: switches between snapshot and device-map mode on one handle, empty and tiny maps, points on box faces through both
kill kernels, bulk deltas past the bounce buffers and the slot capacity, and compaction at its threshold and past 1024 blocks."""
import numpy as np
import pytest

import helpers as H
import np_mapops as nm
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
NONE = 0xFFFFFFFF


class Pair:
    """A device-map handle and its mirror.  The mirror keeps every slot (dead ones too) and applies the library's commit
    rule: a commit runs when something changed; it compacts when slots > 65536 and 2 * live < slots."""

    def __init__(self, dev=None, n_lidar=1, params=None):
        self.dev = dev if dev is not None else plugin.MeasurementModel(n_lidar, params=params)
        self.compactions = 0
        self._reset()

    def _reset(self):
        self.xyz = np.zeros((0, 3), F); self.ny = np.zeros(0, F); self.ids = np.zeros(0, np.int64); self.live = np.zeros(0, bool)
        self.dirty = self.appended = False
        self.indexed = False          # the last commit saw a live point (the voxel-box kill walks that index)

    def _append(self, xyz, ny, ids):
        xyz = np.asarray(xyz, F).reshape(-1, 3)
        n = len(xyz)
        if n == 0:
            return
        ids = np.arange(len(self.live), len(self.live) + n) if ids is None else np.asarray(ids, np.int64)   # slot at append time
        self.xyz = np.concatenate([self.xyz, xyz]); self.ny = np.concatenate([self.ny, np.asarray(ny, F)])
        self.ids = np.concatenate([self.ids, ids]); self.live = np.concatenate([self.live, np.ones(n, bool)])
        self.dirty = self.appended = True

    def _commit(self):
        if not self.dirty:
            return
        n, live = len(self.live), int(self.live.sum())
        if n > 65536 and 2 * live < n:
            k = self.live
            self.xyz, self.ny, self.ids, self.live = self.xyz[k], self.ny[k], self.ids[k], self.live[k]
            self.compactions += 1
        self.dirty = self.appended = False
        self.indexed = live > 0

    def build(self, xyz, ny, ids=None):
        self.dev.map_build(xyz, ny, ids)
        self._reset()
        self._append(xyz, ny, ids if ids is not None else np.arange(len(np.asarray(xyz).reshape(-1, 3))))
        self.dirty = True
        self._commit()

    def add(self, xyz, ny, ids=None, clobber=False):
        keep = [None if a is None else np.array(a) for a in (xyz, ny, ids)]
        self.dev.map_add_points(xyz, ny, ids)
        if clobber:                      # the caller's arrays are consumed when the call returns
            for a in (xyz, ny, ids):
                if a is not None:
                    a[...] = 0
        self._append(*keep)

    def delete(self, boxes):
        n = self.dev.map_delete_boxes(boxes)
        kill = np.zeros(len(self.live), bool)
        for b in np.asarray(boxes, F).reshape(-1, 6):
            kill |= self.live & nm.in_box(self.xyz, b)
        self.live[kill] = False
        assert n == int(kill.sum())
        if n:
            self.dirty = True
        return n

    def sync(self, boxes, xyz, ny, ids=None, want_count=True, clobber=False):
        boxes = np.ascontiguousarray(boxes, F).reshape(-1, 6)
        xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3); ny = np.ascontiguousarray(ny, F)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        keep = [None if a is None else a.copy() for a in (boxes, xyz, ny, ids)]
        if self.appended:
            self._commit()
        n = self.dev.map_sync_voxels(dict(boxes=boxes, xyz=xyz, normal_y=ny, ids=ids), want_count=want_count)
        if clobber:
            for a in (boxes, xyz, ny, ids):
                if a is not None:
                    a[...] = 0
        boxes, xyz, ny, ids = keep
        kill = self.live & _in_voxels(self.xyz, boxes)
        self.live[kill] = False
        if want_count:
            assert n == int(kill.sum())
        if len(boxes) and self.indexed and (kill.any() or not want_count):
            self.dirty = True
        self._append(xyz, ny, ids)
        return int(kill.sum())

    def commit(self):
        self.dev.map_commit()
        self._commit()

    def check(self, q=None):
        """Live set, slot numbers, compaction count and (with queries) the k-NN against the brute force."""
        self._commit()
        live, slots = self.dev.map_info()
        assert (live, slots) == (int(self.live.sum()), len(self.live))
        m = self.dev.map_download()
        k = self.live
        assert np.array_equal(m["slots"], np.flatnonzero(k).astype(np.uint32))
        assert np.array_equal(m["xyz"].view(np.uint32), self.xyz[k].view(np.uint32))
        assert np.array_equal(m["normal_y"], self.ny[k]) and np.array_equal(m["ids"].astype(np.int64), self.ids[k])
        assert self.dev.counters().map_compactions == self.compactions
        if q is not None:
            knn_check(self.dev, m, q)
        return m


def _in_voxels(xyz, boxes):
    """Union of nm.in_box over boxes.  Many 0.5 m voxel boxes on the 0.5 lattice take a hash lookup: for such a box,
    min <= p < min + 0.5 in float32 is exactly floor(2 p) == 2 min (both products are exact)."""
    b = np.asarray(boxes, F).reshape(-1, 6)
    lo2 = b[:, :3] * F(2)
    if len(b) > 64 and np.all(b[:, 3:] - b[:, :3] == F(0.5)) and np.all(lo2 == np.floor(lo2)) and np.all(np.abs(lo2) < 2 ** 20):
        key = lambda v: ((v[:, 0] + 2 ** 20) * 2 ** 21 + (v[:, 1] + 2 ** 20)) * 2 ** 21 + (v[:, 2] + 2 ** 20)
        with np.errstate(invalid="ignore"):
            v = np.floor(xyz * F(2))
        ok = np.all(np.isfinite(v) & (np.abs(v) < 2 ** 20), axis=1)
        return ok & np.isin(key(np.where(ok[:, None], v, 0).astype(np.int64)), key(lo2.astype(np.int64)))
    m = np.zeros(len(xyz), bool)
    for x in b:
        m |= nm.in_box(xyz, x)
    return m


def knn_check(dev, m, q):
    c0 = dev.counters().knn_tie_queries
    di, dd, _ = dev.Nearest_Search(q)
    ties = dev.counters().knn_tie_queries - c0
    ri, rd, rt = nm.knn_bruteforce(m["xyz"], m["slots"], q)
    bad = np.flatnonzero(np.any(di != ri, axis=1) | np.any(dd.view(np.uint32) != rd.view(np.uint32), axis=1))
    assert len(bad) == 0, (len(bad), q[bad[:3]], di[bad[:3]], ri[bad[:3]], dd[bad[:3]], rd[bad[:3]])
    assert ties == rt, (ties, rt)
    return rt


def queries(xyz, rng, n=4000, lattice=None):
    """Near the map, a sparse fringe, far outside (ring expansion up to the whole grid), and points on candidate cell faces."""
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    if len(xyz) == 0:
        return rng.uniform(-5, 5, (64, 3)).astype(F)
    c = xyz[rng.integers(0, len(xyz), n)].astype(np.float64)
    q = c + rng.normal(0, 0.4, c.shape)
    q[: n // 20] += 60.0
    q[n // 20: n // 10] *= 3.0
    lo = xyz.min(0).astype(np.float64)
    h = lattice if lattice is not None else rng.choice([0.5, 1.0, 1.5], (n // 10, 1))
    q[n // 10: n // 5] = lo + np.floor((q[n // 10: n // 5] - lo) / h) * h     # on faces of cells of edge 0.5, 1, 1.5 from the origin
    return q.astype(F)


def cloud(n, rng, ext=(40.0, 40.0, 4.0)):
    return (rng.uniform(0, 1, (n, 3)) * np.array(ext)).astype(F)


def empty_snapshot():
    return plugin.MapSnapshot(np.zeros(0, capi.MAP_NODE), np.zeros(0, F), np.zeros(0, np.int64), 0)


def _refuses_map_calls(h):
    z3 = np.zeros((1, 3), F); z1 = np.zeros(1, F)
    calls = (lambda: h.map_add_points(z3, z1), lambda: h.map_delete_boxes(np.zeros((1, 6), F)),
             lambda: h.map_sync_voxels(dict(boxes=np.zeros((1, 6), F), xyz=z3, normal_y=z1, ids=None)), h.map_info, h.map_download)
    for f in calls:
        with pytest.raises(capi.MalioError) as e:
            f()
        assert e.value.status == capi.ERR_STATE
    h.map_commit()        # a no-op, as before any build


def _to_ids(idx, table):
    if table is None:
        return idx
    t = np.asarray(table, np.int64) if len(table) else np.zeros(1, np.int64)
    return np.where(idx != NONE, t[np.where(idx != NONE, idx, 0)], -1)


def _same_answers(h, fresh, case, q, tables=(None, None)):
    """Nearest_Search, one measurement pass and a 3-pass update of h equal those of a handle that only saw this mode and data.
    tables: index -> id of each handle when their indices differ in kind (slots against snapshot nodes)."""
    i1, d1, _ = h.Nearest_Search(q); i2, d2, _ = fresh.Nearest_Search(q)
    assert np.array_equal(d1, d2) and np.array_equal(_to_ids(i1, tables[0]), _to_ids(i2, tables[1]))
    for m in (h, fresh):
        m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    ok1, H1, h1, s1 = h.h_share_model(case.x_prop, True)
    ok2, H2, h2, s2 = fresh.h_share_model(case.x_prop, True)
    a1, a2 = h.aux(), fresh.aux()
    assert ok1 == ok2
    for k in ("nn_sqdist", "world", "selected"):
        assert np.array_equal(a1[k], a2[k]), k
    assert np.array_equal(_to_ids(a1["nn_idx"], tables[0]), _to_ids(a2["nn_idx"], tables[1]))
    if ok1:
        assert s1.n_eff == s2.n_eff and H.rel_err(H1, H2) < 1e-11 and H.rel_err(h1, h2) < 1e-11
    x1, P1 = case.x_prop.copy(), case.P_prop.copy()
    x2, P2 = case.x_prop.copy(), case.P_prop.copy()
    h.rearm_scan(); fresh.rearm_scan()
    r1 = h.update_iterated_dyn_share_modified(x1, P1, 3)
    r2 = fresh.update_iterated_dyn_share_modified(x2, P2, 3)
    nd = 17 + 6 * case.n_lidar
    assert r1.passes == r2.passes and r1.last_status == r2.last_status
    assert np.abs(synth.state_to_vec(x1, case.n_lidar) - synth.state_to_vec(x2, case.n_lidar)).max() <= 1e-9
    assert np.abs(P1 - P2).max() <= 1e-9 * max(np.abs(P2).max(), 1e-300) and P1.shape == (nd, nd)
    return ok1


@pytest.fixture(scope="module")
def case():
    return synth.make_case("map edges", 6000, 120000, 1, 3)


@pytest.fixture(scope="module")
def scan_world(case):
    """feats_down_world of the case's scan at x_prop (where a tiny map must sit to be found)."""
    m = H.make_model(case, plugin.build_static_snapshot(case.map_xyz, case.map_normal_y))
    m.h_share_model(case.x_prop, True)
    w = m.aux()["world"].copy()
    m.close()
    return w


def test_mode_switches_on_one_handle_in_both_directions(case):
    rng = np.random.default_rng(1)
    X, NY = case.map_xyz, case.map_normal_y
    A = slice(0, 60000)
    extra = (X[rng.integers(0, len(X), 40000)] + rng.normal(0, 0.3, (40000, 3))).astype(F)
    Dx = np.concatenate([X, extra]).astype(F); Dny = np.concatenate([NY, np.full(40000, 0.002, F)])
    h = plugin.MeasurementModel(case.n_lidar, params=case.params)
    q = queries(X, rng, 3000)

    def fresh_build(xyz, ny):
        f = plugin.MeasurementModel(case.n_lidar, params=case.params); f.map_build(xyz, ny); return f

    def fresh_snap(snap, compact):
        f = plugin.MeasurementModel(case.n_lidar, params=case.params)
        (f.upload_map_compact if compact else f.upload_map)(snap); return f

    big = plugin.build_static_snapshot(X, NY)                  # 120k nodes: larger than the 60k-slot device map
    small = plugin.build_static_snapshot(X[:20000], NY[:20000])  # smaller than it
    steps = [("build", (X[A], NY[A])), ("snap", (big, False)), ("build", (X[A], NY[A])), ("snap", (small, True)),
             ("build", (X[A], NY[A])), ("snap", (small, False)), ("snap", (big, True)), ("build", (Dx, Dny))]
    for kind, arg in steps:
        if kind == "build":
            h.map_build(*arg)
            f = fresh_build(*arg)
            live, slots = h.map_info()
            assert live == slots == len(arg[0])
        else:
            (h.upload_map_compact if arg[1] else h.upload_map)(arg[0])
            f = fresh_snap(*arg)
            _refuses_map_calls(h)
        assert _same_answers(h, f, case, q)
        f.close()
    # the last build is larger than every earlier size: its slots are all there and the deltas keep working
    p = Pair(dev=h)
    p.build(Dx, Dny)
    p.add(extra[:5000] + F(0.01), np.full(5000, 0.003, F))
    p.delete([[0, 0, -100, 20, 20, 100]])
    p.check(q)
    h.close()


@pytest.mark.parametrize("n", [0, 1, 4, 5, 6])
def test_empty_and_tiny_maps(case, scan_world, n):
    rng = np.random.default_rng(10 + n)
    c = scan_world[1234]
    pts = (c + rng.uniform(-0.8, 0.8, (n, 3))).astype(F)
    ny = np.full(n, 0.001, F)
    p = Pair(n_lidar=case.n_lidar, params=case.params)
    p.build(pts, ny)
    q = np.concatenate([queries(case.map_xyz, rng, 400), (c + rng.normal(0, 1.0, (200, 3))).astype(F)]).astype(F)
    p.check(q)
    ref = plugin.MeasurementModel(case.n_lidar, params=case.params)
    snap = empty_snapshot() if n == 0 else plugin.build_static_snapshot(pts, ny)
    ref.upload_map(snap)
    m = p.dev.map_download()
    slot_id = np.zeros(max(n, 1), np.int64); slot_id[m["slots"]] = m["ids"]
    ok = _same_answers(p.dev, ref, case, q, tables=(slot_id, snap.node_ids))
    a = p.dev.aux()
    if n < 5:
        assert not ok and a["selected"].sum() == 0
        assert np.all(a["nn_idx"][:, n:] == NONE) and np.all(np.isinf(a["nn_sqdist"][:, n:]))
    else:
        gate = a["nn_sqdist"][:, 4] <= case.params.knn_max_sqdist
        assert np.all(a["selected"] <= gate) and gate.any()
    ref.close()
    p.dev.close()


def test_everything_deleted_with_and_without_compaction_then_refilled(case):
    rng = np.random.default_rng(2)
    empty = plugin.MeasurementModel(case.n_lidar, params=case.params)
    empty.upload_map(empty_snapshot())
    everything = [[-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf]]
    for n, compacts in ((1000, 0), (65536, 0), (70000, 1)):
        p = Pair(n_lidar=case.n_lidar, params=case.params)
        xyz = cloud(n, rng)
        p.build(xyz, np.full(n, 0.001, F))
        assert p.delete(everything) == n
        m = p.check()
        assert len(m["slots"]) == 0 and p.compactions == compacts
        assert p.dev.map_info() == (0, 0 if compacts else n)
        q = queries(xyz, rng, 500)
        di, dd, _ = p.dev.Nearest_Search(q)
        assert np.all(di == NONE) and np.all(np.isinf(dd))
        _same_answers(p.dev, empty, case, q)
        p.add(xyz[:7] + F(0.25), np.full(7, 0.002, F))
        p.check(q)
        p.sync([[0, 0, 0, 20, 20, 2]], xyz[7:40], np.full(33, 0.003, F), np.arange(10 ** 6, 10 ** 6 + 33))
        p.check(q)
        p.dev.close()
    # built empty, then filled
    p = Pair(n_lidar=case.n_lidar, params=case.params)
    p.build(np.zeros((0, 3), F), np.zeros(0, F))
    q = queries(case.map_xyz, rng, 500)
    _same_answers(p.dev, empty, case, q)
    assert p.sync([[0, 0, 0, 1, 1, 1]], np.zeros((0, 3), F), np.zeros(0, F)) == 0
    p.add(case.map_xyz[:3000], case.map_normal_y[:3000])
    p.check(q)
    p.dev.close(); empty.close()


def _lattice(rng):
    g = np.arange(-4.0, 4.01, 0.5, dtype=F)
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(F)
    up = np.nextafter(lat, F(np.inf)); dn = np.nextafter(lat, F(-np.inf))
    mix = np.where(rng.uniform(size=lat.shape) < 0.5, up, dn).astype(F)
    z = lat.copy(); z[z == 0] = F(-0.0)
    return np.concatenate([lat, mix, z, up[::3], dn[::5]]).astype(F)


def _lattice_boxes(rng, k):
    a = rng.integers(-10, 9, (k, 3)) * 0.5
    w = rng.integers(0, 6, (k, 3)) * 0.5                        # 0: degenerate on that axis
    b = np.concatenate([a, a + w], 1).astype(F)
    return b


@pytest.mark.parametrize("nb", [0, 1, 16, 17, 33])
def test_box_faces_through_the_sweep(nb):
    rng = np.random.default_rng(100 + nb)
    pts = _lattice(rng)
    p = Pair()
    p.build(pts, np.full(len(pts), 0.001, F))
    boxes = _lattice_boxes(rng, nb)
    if nb >= 16:
        boxes[3] = boxes[2]                                      # overlapping boxes count a point once
        boxes[5] = [-np.inf, -np.inf, 1.0, np.inf, -2.0, np.inf]  # +-inf faces
        boxes[7] = [0, 0, 0, 0, 0, 0]
        boxes[-1] = [1.0, -np.inf, -np.inf, 1.5, np.inf, np.inf]  # the last partial chunk kills points no other box does
    p.delete(boxes)
    q = np.concatenate([queries(pts, rng, 2000, lattice=0.5), _lattice(rng)[::7] + F(0.25)]).astype(F)
    p.check(q)
    p.dev.close()


def test_box_faces_through_the_voxel_index():
    rng = np.random.default_rng(7)
    pts = _lattice(rng)
    ny = np.full(len(pts), 0.001, F)
    p = Pair()
    p.build(pts, ny)
    # disjoint voxel boxes on the lattice, at the grid's first and last cell, partly and wholly outside the grid
    cells = rng.choice(16 ** 3, 300, replace=False)
    ijk = np.stack([cells % 16, cells // 16 % 16, cells // 256], 1) * 0.5 - 4.0
    boxes = np.concatenate([ijk, ijk + 0.5], 1).astype(F)
    extra = np.array([[-4.5, -4.5, -4.5, -4.0, -4.0, -4.0], [-4.25, 3.5, 0.25, -3.75, 4.25, 0.75], [4.0, 4.0, 4.0, 4.5, 4.5, 4.5],
                      [3.5, -4.5, 3.5, 4.5, -3.5, 4.5], [50, 50, 50, 51, 51, 51], [-60, 0, 0, -59, 1, 1]], F)
    overlap = np.all((boxes[:, None, :3] < extra[None, :, 3:]) & (boxes[:, None, 3:] > extra[None, :, :3]), axis=2).any(1)
    boxes = np.concatenate([extra, boxes[~overlap]]).astype(F)
    new = (boxes[:40, :3] + F(0.125)).astype(F)
    p.sync(boxes, new, np.full(len(new), 0.002, F), np.arange(10 ** 6, 10 ** 6 + len(new)))
    q = queries(pts, rng, 2000, lattice=0.5)
    p.check(q)
    # appends not yet committed, then a sync: the kill must see them
    app = (_lattice(rng)[::11] + F(0.0)).astype(F)
    p.add(app, np.full(len(app), 0.004, F))
    cells = rng.choice(16 ** 3, 200, replace=False)
    ijk = np.stack([cells % 16, cells // 16 % 16, cells // 256], 1) * 0.5 - 4.0
    p.sync(np.concatenate([ijk, ijk + 0.5], 1).astype(F), np.zeros((0, 3), F), np.zeros(0, F))
    p.check(q)
    # one box covering the whole grid
    p.sync([[-4.0, -4.0, -4.0, 4.5, 4.5, 4.5]], pts[:5], ny[:5], np.arange(5))
    p.check(q)
    p.dev.close()


def test_bulk_deltas_growth_and_bounce_limits():
    rng = np.random.default_rng(4)
    p = Pair()
    base = cloud(1000, rng)
    p.build(base, np.full(1000, 0.001, F), None)                 # ids = NULL: 0..n-1
    q = queries(base, rng, 2000)
    for k in (5000, 12000, 30000):                               # past the slot capacity each time: growth keeps the slots
        a = cloud(k, rng)
        p.add(a, rng.uniform(0.0005, 0.01, k).astype(F), None)  # ids = NULL: the slot index at append time
        p.check(q)
    for k in (70000, 65536):                                     # direct path, and the bounce buffer at its limit
        a = cloud(k, rng); ny = rng.uniform(0.0005, 0.01, k).astype(F); ids = (np.arange(k) + 5 * 10 ** 6).astype(np.int32)
        p.add(a, ny, ids, clobber=True)
        p.check(q)
    allv = np.stack(np.meshgrid(np.arange(80), np.arange(80), np.arange(8), indexing="ij"), -1).reshape(-1, 3) * 0.5
    for nbx, want in ((17000, True), (17000, False), (16384, True), (16384, False)):
        v = allv[rng.choice(len(allv), nbx, replace=False)]
        boxes = np.concatenate([v, v + 0.5], 1).astype(F)
        xyz = (v[:3000] + rng.uniform(0, 0.5, (3000, 3))).astype(F); ny = np.full(3000, 0.002, F)
        ids = np.arange(3000, dtype=np.int32) + 7 * 10 ** 6
        p.sync(boxes, xyz, ny, ids, want_count=want, clobber=True)
        p.check(q)
    p.dev.close()


def _dead_cloud(n, dead, rng, ext=(60.0, 60.0, 4.0)):
    """n points; those with dead[i] sit 50 m above the others, so one box deletes exactly them."""
    x = cloud(n, rng, ext)
    x[dead, 2] += F(50.0)
    return x


UP = [[-np.inf, -np.inf, 40.0, np.inf, np.inf, np.inf]]


@pytest.mark.parametrize("n,live,compacts", [(65536, 1000, 0), (65537, 1000, 1), (70000, 35000, 0), (70001, 35000, 1)])
def test_compaction_threshold(n, live, compacts):
    rng = np.random.default_rng(n)
    dead = np.ones(n, bool); dead[rng.choice(n, live, replace=False)] = False
    x = _dead_cloud(n, dead, rng)
    p = Pair()
    p.build(x, np.full(n, 0.001, F))
    assert p.delete(UP) == n - live
    p.commit()
    assert p.dev.counters().map_compactions == compacts == p.compactions
    p.check(queries(x[~dead], rng, 1000))
    p.dev.close()


def test_compaction_block_patterns_ties_and_two_compactions():
    rng = np.random.default_rng(5)
    n = 100000
    dead = np.zeros(n, bool)
    dead[1000:3100] = True                   # a dead run across two 1024-slot block boundaries
    dead[4096:6144] = True                   # two wholly dead blocks
    dead[20480:75000] = rng.uniform(size=75000 - 20480) < 0.9   # sparse survivors; [10240, 20480) stays wholly live
    x = _dead_cloud(n, dead, rng)
    p = Pair()
    p.build(x, np.full(n, 0.001, F))
    dup = x[~dead][rng.choice(int((~dead).sum()), 500, replace=False)]
    p.add(dup, np.full(500, 0.002, F))       # exact duplicates in later slots: ties in (distance, slot) order
    q = np.concatenate([queries(x[~dead], rng, 3000), dup[:300]]).astype(F)
    p.delete(UP)
    m = p.check(q)
    assert p.compactions == 1 and len(m["slots"]) == p.live.sum()
    # growth after the swap, then a second compaction
    more = _dead_cloud(150000, np.zeros(150000, bool), rng)
    p.add(more, np.full(150000, 0.003, F))
    p.check(q)
    p.delete([[0, 0, -1, 55, 60, 10]])
    m = p.check(q)
    assert p.compactions == 2
    t = knn_check(p.dev, m, np.concatenate([dup[:300], m["xyz"][:200]]).astype(F))
    assert t > 0
    p.dev.close()


def test_more_than_1024_blocks():
    rng = np.random.default_rng(6)
    n = 1_200_000
    dead = np.zeros(n, bool)
    dead[rng.choice(n, 300000, replace=False)] = True
    x = _dead_cloud(n, dead, rng, ext=(200.0, 200.0, 8.0))
    p = Pair()
    p.build(x, np.full(n, 0.001, F))
    p.delete(UP)                             # a quarter dead: no compaction, the download's scan carries over 1172 blocks
    q = queries(x[~dead], rng, 3000)
    p.check(q)
    assert p.compactions == 0
    p.delete([[0, 0, -1, 120, 200, 20]])     # now most are dead: the commit's scan carries over 1172 blocks
    p.check(q)
    assert p.compactions == 1
    p.dev.close()
