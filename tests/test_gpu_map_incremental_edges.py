"""map_incr_kernel (map_incremental, laserMapping.cpp:398-446) against the numpy restatement (tests/map_incr_ref.py) on the
device's own neighbour lists, at the edges random scans never reach: voxel faces (and -0.0, subnormals, offsets up to 1e5 m),
|n0 - mid| == 0.5 fs, distance ties at every neighbour position, short lists, normal_y == cov_threshold.  Both map modes
(snapshot; device-resident fresh, with dead slots, right after a compaction), both entry points (host arrays and CUDA
tensors, with and without the world output).  The lists themselves are pinned first: pyoracle.knn_snapshot in snapshot mode,
np_mapops.knn_bruteforce (slot tie rule) in device-resident mode.  Then a scan-to-map loop on the device-resident map against
the real ikd-Tree."""
import numpy as np
import pytest

import map_incr_ref as R
import np_mapops
import pyoracle as po
import world_ref
from malio_b200 import capi, plugin, synth
from test_mapops_cpu import same_set

pytestmark = pytest.mark.gpu
F = np.float32
NONE = 0xFFFFFFFF
MODES = ("snapshot", "device", "device_dead", "device_compacted")


def _identity(pos=(0.0, 0.0, 0.0)):
    return synth.make_state(pos, [1.0, 0.0, 0.0, 0.0], [], [])


def _model(L, mode, mp, sort=True, params=None, rng=None):
    """A handle holding the map mp in `mode`.  Returns (model, point array indexed by the lists, pin(world, idx, d2))."""
    m = plugin.MeasurementModel(L, sort_queries=sort, params=params)
    ny = np.full(len(mp), 0.001, F)
    if mode == "snapshot":
        snap = (plugin.build_static_snapshot(mp, ny) if len(mp) else
                plugin.MapSnapshot(np.zeros(0, capi.MAP_NODE), np.zeros(0, F), np.zeros(0, np.int64), 0))
        m.upload_map(snap)

        def pin(world, idx, d2):
            if len(snap.nodes) == 0:
                assert np.all(idx == NONE)
                return
            i, d, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, world)
            assert np.array_equal(i.view(np.uint32), idx) and np.array_equal(d, d2)
        return m, snap.nodes["xyz"], pin
    junk_n = {"device": 0, "device_dead": 3000, "device_compacted": 70000}[mode]
    rng = rng or np.random.default_rng(3)
    junk = (rng.uniform(-30, 30, (junk_n, 3)) + np.array([0.0, 0.0, 80.0])).astype(F)   # 80 m above the planted sites
    allp = np.concatenate([mp, junk]).astype(F)
    order = rng.permutation(len(allp))                                                     # dead slots between live ones
    m.map_build(allp[order], np.full(len(allp), 0.001, F), order.astype(np.int32))
    c0 = m.counters().map_compactions
    if junk_n:
        assert m.map_delete_boxes(np.array([[-40, -40, 40, 40, 40, 120]], F)) == junk_n
        m.map_commit()
        live, slots = m.map_info()
        assert live == len(mp)
        if mode == "device_dead":
            assert slots == len(allp) and m.counters().map_compactions == c0
        else:
            assert slots == live and m.counters().map_compactions == c0 + 1
    d = m.map_download()

    def pin(world, idx, d2):
        i, dd, _ = np_mapops.knn_bruteforce(d["xyz"], d["slots"], world)
        assert np.array_equal(i, idx) and np.array_equal(dd, d2)
    return m, (R.slot_points(d) if len(d["slots"]) else np.zeros((0, 3), F)), pin


def _lid(n, L, lidar):
    return np.arange(n) % L if lidar is None else np.asarray(lidar)


def _scan(m, body, L, tcomp=None, lidar=None):
    table, off = synth.make_tables(L, 2, np.random.default_rng(5))
    m.upload_scan(R.scan_records(body, L, _lid(len(body), L, lidar)), table, off, tcomp)


def _decide_everywhere(m, state, tcomp, body, L, mxyz, pin, fs_list, cov_threshold=0.5, lidar=None):
    """One searching pass, the lists pinned, then every entry point against the restatement for each fs, initialised or not.
    Returns {fs: classes of the initialised filter}."""
    import torch
    m.h_share_model(state, True)
    a = m.aux()
    pin(a["world"], a["nn_idx"], a["nn_sqdist"])
    lid = _lid(len(body), L, lidar)
    out = {}
    for fs in fs_list:
        for inited in (False, True):
            cls_r, w_r = R.map_incremental_ref(state, tcomp, body, lid, a["normal_y"], a["nn_idx"], mxyz, cov_threshold, fs, inited)
            for tensor in (False, True):
                for world in (True, False):
                    if tensor:
                        c, w = m.map_incremental_tensor(state, fs, inited, world=world)
                        torch.cuda.synchronize()
                        c, w = c.cpu().numpy(), (None if w is None else w.cpu().numpy())
                    else:
                        c, w = m.map_incremental(state, fs, inited, world=world)
                    assert np.array_equal(c, cls_r), (fs, inited, tensor, world, int((c != cls_r).sum()))
                    if world:
                        assert np.array_equal(w.view(np.uint32), w_r.view(np.uint32)), (fs, inited, tensor)
                    else:
                        assert w is None
            if not inited:
                assert np.all(cls_r[cls_r != capi.MAP_SKIP] == capi.MAP_ADD)
        out[fs] = cls_r
    return out


def _check_planted(cls_by_fs, exp, grp, fsa):
    for fs, cls in cls_by_fs.items():
        sel = fsa == fs
        bad = R.check_expect(cls[sel], exp[sel])
        assert len(bad) == 0, [(grp[sel][b], int(cls[sel][b]), int(exp[sel][b])) for b in bad]
        for g in np.unique(grp[sel]):          # every face group is hit from both sides
            if g.startswith("face"):
                e = exp[sel][grp[sel] == g]
                assert (e == capi.MAP_ADD_NO_DOWNSAMPLE).any() and (e == R.NOT_NODS).any(), g


@pytest.mark.parametrize("sort", [True, False])
@pytest.mark.parametrize("mode", MODES)
def test_planted_edges_identity_state(mode, sort):
    """World = body bit for bit on the identity state (checked first); then every planted edge reaches its class on the device
    exactly as in the restatement."""
    w, mp, exp, grp, fsa = R.planted_scene(origin=(-28.0, -28.0, -3.0)).arrays()
    m, mxyz, pin = _model(1, mode, mp, sort)
    _scan(m, w, 1)
    st = _identity()
    m.h_share_model(st, True)
    cls, wd = m.map_incremental(st, 0.5, True)
    assert np.array_equal(wd, w) and np.all(cls != capi.MAP_SKIP)
    res = _decide_everywhere(m, st, None, w, 1, mxyz, pin, np.unique(fsa))
    _check_planted(res, exp, grp, fsa)
    m.close()


@pytest.mark.parametrize("mode", ["snapshot", "device"])
@pytest.mark.parametrize("offset", [1.0e3, 1.0e4, 1.0e5, -1.0e4])
def test_planted_edges_far_from_the_origin(offset, mode):
    """The same scene moved to `offset` on every axis, seen from a state at that position (identity rotation): the body points
    are the planted world points minus the position, exactly."""
    pos = np.full(3, offset)
    w, mp, exp, grp, fsa = R.planted_scene(origin=pos + np.array([-28.0, -28.0, -3.0]), zero_x=False).arrays()
    body = (w.astype(np.float64) - pos).astype(F)
    assert np.array_equal(body.astype(np.float64) + pos, w.astype(np.float64))
    st = _identity(pos)
    assert np.array_equal(world_ref.register_world(st, None, body, 0, 0.0)[:, :3], w)
    m, mxyz, pin = _model(1, mode, mp)
    _scan(m, body, 1)
    res = _decide_everywhere(m, st, None, body, 1, mxyz, pin, np.unique(fsa))
    _check_planted(res, exp, grp, fsa)
    m.close()


@pytest.mark.parametrize("mode", ["snapshot", "device"])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_distance_ties_on_a_far_state(L, mode):
    """world_ref.far_state (1e4 m out, rotated, non-identity extrinsics, temporal compensation on LiDARs 1..): the world
    points come from register_world (checked against the device's), the tie clusters are planted around them."""
    st, tc = world_ref.far_state(L, seed=7 + L)
    rng = np.random.default_rng(L)
    body = rng.uniform(-40, 40, (6000, 3)).astype(F)
    lid = np.arange(len(body)) % L
    wall = world_ref.register_world(st, tc, body, lid, 0.0)[:, :3]
    fs = 0.5
    d = np.abs(wall - R.voxel_mid(wall, fs)) / fs
    sc = R.Scene()
    chosen = []
    for i in np.flatnonzero(np.all((d > 0.08) & (d < 0.22), axis=1)):   # one per SITE-metre cell
        if any(np.abs(wall[i] - wall[c]).max() <= R.SITE for c in chosen):
            continue
        n = len(chosen)
        j, exact = n % capi.K, (n // capi.K) % 2 == 0
        try:
            sc.tie(wall[i], fs, j, exact, group=f"tie j={j} {'exact' if exact else '-1ulp'}")
        except AssertionError:                 # the mirror image of w through mid is not a float32: not an exact tie
            continue
        chosen.append(i)
        if len(chosen) == 4 * 2 * capi.K:
            break
    assert len(chosen) == 4 * 2 * capi.K and set(lid[chosen].tolist()) == set(range(L))
    w, mp, exp, grp, fsa = sc.arrays()
    b = body[chosen]
    m, mxyz, pin = _model(L, mode, mp)
    _scan(m, b, L, tc, lidar=lid[chosen])
    res = _decide_everywhere(m, st, tc, b, L, mxyz, pin, [fs], lidar=lid[chosen])
    _check_planted(res, exp, grp, fsa)
    m.close()


@pytest.mark.parametrize("mode", ["snapshot", "device"])
@pytest.mark.parametrize("n_map", [0, 1, 4, 5, 6])
def test_short_neighbour_lists(n_map, mode):
    w, mp, expect = R.short_list_scene(n_map)
    m, mxyz, pin = _model(1, mode, mp)
    _scan(m, w, 1)
    res = _decide_everywhere(m, _identity(), None, w, 1, mxyz, pin, [0.5])
    assert np.all(res[0.5] == expect)
    assert np.all((m.aux()["nn_idx"] != NONE).sum(axis=1) == min(n_map, capi.K))
    m.close()


@pytest.mark.parametrize("mode", ["snapshot", "device"])
def test_normal_y_at_the_cov_threshold(mode):
    """A probe handle gives the float normal_y of a group of identical points; with cov_threshold equal to it they are kept,
    one float ulp below it they are skipped (world zero), one ulp above kept."""
    w = np.tile(np.array([3.25, -1.5, 0.75], F), (6, 1))
    mp = (w[0] + np.array([[0.01 * i, 0.3, -0.2] for i in range(6)])).astype(F)
    probe, _, _ = _model(1, mode, mp)
    _scan(probe, w, 1)
    probe.h_share_model(_identity(), True)
    ny = probe.aux()["normal_y"]
    probe.close()
    assert np.all(ny == ny[0]) and ny[0] > 0
    v = F(ny[0])
    for thr, kept in ((float(v), True), (float(np.nextafter(v, F(0))), False), (float(np.nextafter(v, F(1))), True)):
        prm = capi.default_params(1)
        prm.cov_threshold = thr
        m, mxyz, pin = _model(1, mode, mp, params=prm)
        _scan(m, w, 1)
        res = _decide_everywhere(m, _identity(), None, w, 1, mxyz, pin, [0.5], cov_threshold=thr)
        assert np.array_equal(m.aux()["normal_y"], ny)
        assert np.all((res[0.5] != capi.MAP_SKIP) == kept), thr
        m.close()


@pytest.mark.parametrize("mode", ["snapshot", "device"])
@pytest.mark.parametrize("N", [0, 1, 255, 256, 257, 100000])
def test_scan_sizes(N, mode):
    """A synthetic 3-LiDAR case cut to N points (100000: a C2-size scan) after a full update."""
    case = synth.make_case("mi-sizes", max(N, 300), 300000, 3, 3, varied_map_cov=True)
    pts = case.pts[:N]
    m, mxyz, pin = _model(3, mode, case.map_xyz)
    m.upload_scan(pts, case.table, case.table_off, case.temporal_comp)
    x, P = case.x_prop.copy(), case.P_prop.copy()
    m.update_iterated_dyn_share_modified(x, P, case.max_iter)
    if N == 0:
        c, w = m.map_incremental(x, 0.5, True)
        ct, wt = m.map_incremental_tensor(x, 0.5, True)
        assert c.shape == (0,) and w.shape == (0, 3) and tuple(ct.shape) == (0,)
        m.close()
        return
    a = m.aux()
    for fs in (0.5, 0.2):
        cls_r, w_r = R.map_incremental_ref(x, case.temporal_comp, pts["xyz"], pts["lidar"], a["normal_y"], a["nn_idx"], mxyz,
                                           case.params.cov_threshold, fs, True)
        c, w = m.map_incremental(x, fs, True)
        assert np.array_equal(c, cls_r) and np.array_equal(w.view(np.uint32), w_r.view(np.uint32)), (N, fs)
    m.close()


@pytest.mark.skipif(not po.ref_available(), reason="oracle/_ref (the real ikd_Tree.cpp) was not built")
def test_scan_to_map_loop_on_the_device_resident_map_against_the_real_tree():
    """20 scans: update, map_incremental (the tensor path every other scan) equal to the restatement on the device's lists,
    MAP_ADD into the tree with down-sampling and its re-synchronisation records into the device, MAP_ADD_NO_DOWNSAMPLE into
    both; the live sets stay equal.  Every fifth scan a snapshot-mode handle on the same live set and state decides too: where
    both modes list the same neighbours the classes agree, and every list that differs sits on a counted distance tie."""
    import torch
    base = synth.make_case("loop", 4000, 60000, 1, 3)
    tree = po.RefTree(box_length=0.5)
    dev = plugin.MeasurementModel(1, params=base.params)
    n0 = base.map_xyz.shape[0]
    ny0 = np.full(n0, 0.001, F)
    tree.build(base.map_xyz, ny0, np.arange(n0, dtype=np.int32)); dev.map_build(base.map_xyz, ny0, np.arange(n0, dtype=np.int32))
    nid = n0
    counts = np.zeros(4, np.int64)
    for s in range(20):
        case = synth.make_case("loop", 4000, 60000, 1, 3, map_xyz=base.map_xyz, seed_scan=100 + s, seed_state=200 + s)
        dev.upload_scan(case.pts, case.table, case.table_off, None)
        x, P = case.x_prop.copy(), case.P_prop.copy()
        dev.update_iterated_dyn_share_modified(x, P, case.max_iter)
        a = dev.aux()
        d = dev.map_download()
        mxyz = R.slot_points(d)
        cls_r, w_r = R.map_incremental_ref(x, None, case.pts["xyz"], case.pts["lidar"], a["normal_y"], a["nn_idx"], mxyz,
                                           case.params.cov_threshold, 0.5, True)
        if s % 2:
            ct, wt = dev.map_incremental_tensor(x, 0.5, True)
            torch.cuda.synchronize()
            cls, w = ct.cpu().numpy(), wt.cpu().numpy()
        else:
            cls, w = dev.map_incremental(x, 0.5, True)
        assert np.array_equal(cls, cls_r) and np.array_equal(w.view(np.uint32), w_r.view(np.uint32)), s
        counts += np.bincount(cls, minlength=4)
        if s % 5 == 4:
            nodes, cov, ids, depth, _ = tree.snapshot()
            snap = plugin.MapSnapshot(nodes, cov, ids, depth)
            ref = plugin.MeasurementModel(1, params=base.params)
            ref.upload_map(snap)
            ref.upload_scan(case.pts, case.table, case.table_off, None)
            dev.rearm_scan()
            t0 = dev.counters().knn_tie_queries
            dev.h_share_model(x, True); ref.h_share_model(x, True)
            ties = dev.counters().knn_tie_queries - t0
            ad, ar = dev.aux(), ref.aux()
            slot_id = np.full(len(mxyz), -1, np.int64); slot_id[d["slots"]] = d["ids"]
            di = np.where(ad["nn_idx"] != NONE, slot_id[np.where(ad["nn_idx"] != NONE, ad["nn_idx"], 0)], -1)
            ri = np.where(ar["nn_idx"] != NONE, snap.node_ids[np.where(ar["nn_idx"] != NONE, ar["nn_idx"], 0)].astype(np.int64), -1)
            cd, _ = dev.map_incremental(x, 0.5, True)
            cr, _ = ref.map_incremental(x, 0.5, True)
            same = np.all(di == ri, axis=1)
            assert np.array_equal(cd[same], cr[same]), s
            dd = ad["nn_sqdist"]
            for r in np.flatnonzero(~same):
                for j in np.flatnonzero(di[r] != ri[r]):
                    tied = (j > 0 and abs(dd[r, j] - dd[r, j - 1]) < 1e-10) or (j < 4 and abs(dd[r, j] - dd[r, j + 1]) < 1e-10) or j == 4
                    assert tied, (s, r, j, dd[r])
            assert int((~same).sum()) <= ties
            ref.close()
        add, nods = cls == capi.MAP_ADD, cls == capi.MAP_ADD_NO_DOWNSAMPLE
        k1, k2 = int(add.sum()), int(nods.sum())
        ids1 = np.arange(nid, nid + k1, dtype=np.int32); nid += k1
        _, sync = tree.add_points_synced(w[add], a["normal_y"][add], ids1, 0.5)
        dev.map_sync_voxels(sync)
        ids2 = np.arange(nid, nid + k2, dtype=np.int32); nid += k2
        tree.add_points(w[nods], a["normal_y"][nods], ids2, downsample=False)
        dev.map_add_points(w[nods], a["normal_y"][nods], ids2)
        tree.wait_rebuild()
        d = dev.map_download()
        assert same_set(tree, (d["xyz"], d["normal_y"], d["ids"])), s
        assert dev.map_info()[0] == tree.validnum()
    assert counts[capi.MAP_ADD] > 0 and counts[capi.MAP_DROP] > 0 and counts[capi.MAP_ADD_NO_DOWNSAMPLE] > 0, counts
    dev.close(); tree.close()
