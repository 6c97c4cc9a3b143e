"""map_incremental's decision (laserMapping.cpp:398-446): the numpy restatement (tests/map_incr_ref.py) against the oracle's
C++ one (orc_map_incremental) on a synthetic case and on the planted edges, and deliberately wrong variants of the
restatement against the planted set: each must change at least one planted point, or the set does not reach that comparison."""
import numpy as np
import pytest

import map_incr_ref as R
import np_mapops
import pyoracle as po
from malio_b200 import capi, synth

F = np.float32
IDENTITY = synth.make_state([0.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0], [], [])


def _table(L):
    return synth.make_tables(L, 2, np.random.default_rng(5))


def _oracle(w, map_xyz, params=None):
    """Oracle on the identity state (world = body) with a static snapshot of map_xyz, after one searching pass.  Returns
    (oracle, snapshot point array)."""
    prm = params if params is not None else capi.default_params(1)
    nodes, cov, _ = po.static_snapshot(map_xyz, 0.001)
    orc = po.Oracle(prm)
    orc.set_map_snapshot(nodes, cov)
    table, off = _table(1)
    orc.set_scan(R.scan_records(w), table, off, None)
    orc.h_share_model(IDENTITY, True)
    return orc, nodes["xyz"]


def _ref(orc, mxyz, w, fs, inited, cov_threshold=0.5, mutant=None):
    a = orc.aux()
    return R.map_incremental_ref(IDENTITY, None, w, 0, a["normal_y"], a["nn_idx"], mxyz, cov_threshold, fs, inited, mutant)


@pytest.fixture(scope="module")
def scene():
    return R.planted_scene(origin=(-28.0, -28.0, -3.0)).arrays()


def test_restatement_equals_oracle_on_a_synthetic_case():
    case = synth.make_case("mi-ref", 3000, 40000, 3, 3, varied_map_cov=True)
    nodes, cov, _ = po.static_snapshot(case.map_xyz, case.map_normal_y)
    orc = po.Oracle(case.params)
    orc.set_map_snapshot(nodes, cov)
    orc.set_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    x, P = case.x_prop.copy(), case.P_prop.copy()
    orc.update_iterated(x, P, case.max_iter)
    a = orc.aux()
    for fs in (0.5, 0.2, 0.1):
        for inited in (False, True):
            cls_o, w_o = orc.map_incremental(x, fs, inited)
            cls_r, w_r = R.map_incremental_ref(x, case.temporal_comp, case.pts["xyz"], case.pts["lidar"], a["normal_y"],
                                               a["nn_idx"], nodes["xyz"], case.params.cov_threshold, fs, inited)
            assert np.array_equal(cls_r, cls_o), (fs, inited, int((cls_r != cls_o).sum()))
            assert np.array_equal(w_r.view(np.uint32), w_o.view(np.uint32))
    assert len(set(cls_o.tolist())) >= 2


def test_restatement_equals_oracle_on_the_planted_edges(scene):
    w, mp, exp, grp, fsa = scene
    orc, mxyz = _oracle(w, mp)
    for fs in np.unique(fsa):
        for inited in (False, True):
            cls_o, w_o = orc.map_incremental(IDENTITY, fs, inited)
            cls_r, w_r = _ref(orc, mxyz, w, fs, inited)
            assert np.array_equal(cls_r, cls_o) and np.array_equal(w_r, w_o), (fs, inited)
            assert np.array_equal(w_r, w)
            if not inited:
                assert np.all(cls_o == capi.MAP_ADD)     # every point is added before the filter is initialised (:439-440)
        sel = fsa == fs
        bad = R.check_expect(cls_r[sel], exp[sel])
        assert len(bad) == 0, [(grp[sel][b], int(cls_r[sel][b]), int(exp[sel][b])) for b in bad]


@pytest.mark.parametrize("n_map", [0, 1, 4, 5, 6])
def test_restatement_equals_oracle_on_short_neighbour_lists(n_map):
    w, mp, expect = R.short_list_scene(n_map)
    orc, mxyz = _oracle(w, mp)
    assert np.all(orc.aux()["nn_cnt"] == min(n_map, capi.K))
    cls_o, w_o = orc.map_incremental(IDENTITY, 0.5, True)
    cls_r, w_r = _ref(orc, mxyz, w, 0.5, True)
    assert np.array_equal(cls_r, cls_o) and np.array_equal(w_r, w_o)
    assert np.all(cls_r == expect)


def test_restatement_equals_oracle_at_the_cov_threshold():
    """normal_y == cov_threshold is kept (:406 is a strict '>'); one float ulp below it as the threshold skips the points."""
    w = np.tile(np.array([3.25, -1.5, 0.75], F), (4, 1))
    mp = (w[0] + np.array([[0.01 * i, 0.3, -0.2] for i in range(6)])).astype(F)
    orc, _ = _oracle(w, mp)
    ny = orc.aux()["normal_y"]
    assert np.all(ny == ny[0]) and ny[0] > 0
    v = F(ny[0])
    for thr, kept in ((float(v), True), (float(np.nextafter(v, F(0))), False), (float(np.nextafter(v, F(1))), True)):
        prm = capi.default_params(1)
        prm.cov_threshold = thr
        o2, mxyz = _oracle(w, mp, prm)
        assert np.array_equal(o2.aux()["normal_y"], ny)
        cls_o, w_o = o2.map_incremental(IDENTITY, 0.5, True)
        cls_r, w_r = _ref(o2, mxyz, w, 0.5, True, cov_threshold=thr)
        assert np.array_equal(cls_r, cls_o) and np.array_equal(w_r, w_o)
        assert np.all((cls_r != capi.MAP_SKIP) == kept) and np.all((w_r == 0).all(axis=1) == (not kept))


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_every_wrong_variant_changes_a_planted_point(scene, mutant):
    w, mp, exp, grp, fsa = scene
    idx, d2, _ = np_mapops.knn_bruteforce(mp, np.arange(len(mp)), w)
    assert np.all(idx // 5 == np.arange(len(w))[:, None]) and np.all(np.diff(d2, axis=1) > 0)   # its own five, no tie
    changed = []
    for fs in np.unique(fsa):
        sel = fsa == fs
        ny = np.zeros(int(sel.sum()), F)
        ny[:3] = F(0.25)                           # three points with normal_y == cov_threshold
        good, _ = R.decide(w[sel], ny, idx[sel], mp, 0.25, fs, True)
        bad, _ = R.decide(w[sel], ny, idx[sel], mp, 0.25, fs, True, mutant=mutant)
        changed += list(grp[sel][good != bad])
    for n_map in (1, 4):
        sw, sp, _ = R.short_list_scene(n_map)
        si, _, _ = np_mapops.knn_bruteforce(sp, np.arange(len(sp)), sw)
        good, _ = R.decide(sw, np.zeros(3), si, sp, 0.5, 0.5, True)
        bad, _ = R.decide(sw, np.zeros(3), si, sp, 0.5, 0.5, True, mutant=mutant)
        changed += [f"short list {n_map}"] * int((good != bad).sum())
    assert changed, mutant
