"""CPU tier of the device-resident map's edge tests: the references the GPU tests (test_gpu_mapops_edges.py) hold the device
to.  np_mapops.knn_bruteforce against a plain float64 search, its tie count on hand-built ties, its cKDTree candidate guard,
and the half-open box rule of MirrorMap against the real ikd-Tree (where oracle/_ref was built) for points on box faces."""
import numpy as np
import pytest

import np_mapops as nm
import pyoracle as po

F = np.float32


def _plain64(xyz, slots, q):
    """O(N*M) float64 search ordered by (distance, slot)."""
    d = ((q[:, None, :].astype(np.float64) - xyz[None, :, :].astype(np.float64)) ** 2).sum(-1)
    o = np.argsort(slots, kind="stable")
    d, s = d[:, o], slots[o]
    o2 = np.argsort(d, axis=1, kind="stable")
    return np.take_along_axis(d, o2, 1), s[o2]


@pytest.mark.parametrize("n", [0, 1, 4, 5, 6, 7, 300, 5000])
def test_bruteforce_equals_a_float64_search_where_the_orders_agree(n):
    rng = np.random.default_rng(n)
    xyz = rng.uniform(-5, 5, (n, 3)).astype(F)
    slots = np.sort(rng.choice(10 * n + 10, n, replace=False)).astype(np.uint32)
    q = np.concatenate([rng.uniform(-6, 6, (300, 3)), rng.uniform(40, 60, (20, 3))]).astype(F)
    idx, d2, ties = nm.knn_bruteforce(xyz, slots, q)
    assert idx.shape == (320, 5) and d2.dtype == F and idx.dtype == np.uint32
    found = min(n, 5)
    assert np.all(idx[:, found:] == nm.NONE) and np.all(np.isinf(d2[:, found:]))
    if n == 0:
        assert ties == 0
        return
    d64, s64 = _plain64(xyz, slots, q)
    # float32 rounding cannot reorder two neighbours whose exact distances differ by more than the relative margin
    k7 = min(n, 6)
    gaps = np.diff(d64[:, :k7], axis=1) > d64[:, 1:k7] * 1e-5 if k7 > 1 else np.ones((len(q), 0), bool)
    agree = np.all(gaps, axis=1)
    assert agree.mean() > 0.95
    assert np.array_equal(idx[agree, :found], s64[agree, :found])
    np.testing.assert_allclose(d2[:, :found].astype(np.float64), d64[:, :found], rtol=1e-6, atol=1e-12)
    # the float32 distance is calc_dist's expression, bit for bit
    for r in range(0, len(q), 37):
        for j in range(found):
            p = xyz[np.flatnonzero(slots == idx[r, j])[0]]
            dx, dy, dz = q[r, 0] - p[0], q[r, 1] - p[1], q[r, 2] - p[2]
            assert d2[r, j] == (dx * dx + dy * dy) + dz * dz
    assert np.all(np.diff(d2[:, :found], axis=1) >= 0)


def test_tie_count_and_the_slot_rule_on_hand_built_ties():
    # a query with two duplicates: the smaller slot comes first
    xyz = np.array([[1, 0, 0], [1, 0, 0], [3, 0, 0], [4, 0, 0], [5, 0, 0], [6, 0, 0], [7, 0, 0]], F)
    slots = np.array([9, 2, 3, 4, 5, 6, 7], np.uint32)
    idx, d2, ties = nm.knn_bruteforce(xyz, slots, np.zeros((1, 3), F))
    assert idx[0].tolist() == [2, 9, 3, 4, 5] and ties == 1
    # points mirrored about the query: each pair ties, in slot order
    q = np.array([[10.25, -3.5, 2.0]], F)
    off = np.array([[0.5, 0, 0], [0, 1.0, 0], [0, 0, 1.5]], F)
    xyz = np.concatenate([q + off, q - off]).astype(F)
    slots = np.array([40, 11, 7, 3, 12, 8], np.uint32)
    idx, d2, ties = nm.knn_bruteforce(xyz, slots, q)
    assert idx[0].tolist() == [3, 40, 11, 12, 7] and ties == 1
    assert d2[0, 0] == d2[0, 1] and d2[0, 2] == d2[0, 3]
    # a tie between the 5th and the 6th counts; one between the 6th and the 7th does not
    x = np.arange(1, 9, dtype=F)[:, None] * np.array([[1, 0, 0]], F)
    x6 = np.concatenate([x[:5], x[4:5], x[5:]]).astype(F)            # 5th == 6th
    _, _, t = nm.knn_bruteforce(x6, np.arange(len(x6), dtype=np.uint32), np.zeros((1, 3), F))
    assert t == 1
    x7 = np.concatenate([x[:6], x[5:6], x[6:]]).astype(F)            # 6th == 7th
    _, _, t = nm.knn_bruteforce(x7, np.arange(len(x7), dtype=np.uint32), np.zeros((1, 3), F))
    assert t == 0
    # distances 1 ulp apart at 1.0 (1.2e-7) are no tie; a pair within 1e-10 is
    d = np.float32(1.0)
    x = np.array([[1, 0, 0], [np.nextafter(d, F(2)), 0, 0], [3, 0, 0], [4, 0, 0], [5, 0, 0], [6, 0, 0]], F)
    _, _, t = nm.knn_bruteforce(x, np.arange(6, dtype=np.uint32), np.zeros((1, 3), F))
    assert t == 0
    s = F(1e-3)
    x = np.array([[s, 0, 0], [0, np.nextafter(s, F(1)), 0], [3, 0, 0], [4, 0, 0], [5, 0, 0], [6, 0, 0]], F)
    _, d2, t = nm.knn_bruteforce(x, np.arange(6, dtype=np.uint32), np.zeros((1, 3), F))
    assert d2[0, 0] != d2[0, 1] and t == 1


def test_kdtree_candidates_fall_back_to_brute_force_when_the_guard_fails():
    rng = np.random.default_rng(3)
    n = 20000
    xyz = rng.uniform(-20, 20, (n, 3)).astype(F)
    slots = np.arange(n, dtype=np.uint32) * 3
    # a query at the centre of a sphere of 40 points at (nearly) one radius: the 24 candidates end inside the shell, so the
    # last candidate is not clearly beyond the 6th best and the query must be searched by brute force
    c = np.array([100.0, 100.0, 100.0], F)
    u = rng.normal(size=(40, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    shell = (c + 2.0 * u).astype(F)
    xyz = np.concatenate([xyz, shell]).astype(F)
    slots = np.concatenate([slots, np.arange(40, dtype=np.uint32) * 3 + 1])
    q = np.concatenate([c[None], rng.uniform(-20, 20, (500, 3)).astype(F)]).astype(F)
    st = {}
    idx, d2, ties = nm.knn_bruteforce(xyz, slots, q, stats=st)
    assert st["fallback"] >= 1
    bi, bd, bt = nm.knn_bruteforce(xyz, slots, q, kd_from=10 ** 9)
    assert np.array_equal(idx, bi) and np.array_equal(d2, bd) and ties == bt
    # a tiny candidate count forces the fallback nearly everywhere; the answer does not change
    st = {}
    idx2, d22, t2 = nm.knn_bruteforce(xyz, slots, q, kd_k=6, stats=st)
    assert st["fallback"] > 100 and np.array_equal(idx2, bi) and np.array_equal(d22, bd) and t2 == bt


def test_box_predicate_is_half_open_in_float32():
    b = np.array([0, 0, 0, 1, 1, 1], F)
    pts = np.array([[0, 0, 0], [-0.0, 0.5, 0.5], [1, 0.5, 0.5], [np.nextafter(F(1), F(0)), 0.5, 0.5],
                    [np.nextafter(F(0), F(-1)), 0.5, 0.5], [0.5, 0.5, 1]], F)
    assert nm.in_box(pts, b).tolist() == [True, True, False, True, False, False]
    assert not nm.in_box(pts, np.array([0, 0, 0, 0, 1, 1], F)).any()                       # min == max on one axis
    inf = np.array([-np.inf, -np.inf, -np.inf, np.inf, np.inf, np.inf], F)
    assert nm.in_box(pts, inf).all()


def _face_points():
    """Lattice points (multiples of 0.5), their +-1 ulp neighbours, and -0.0 / +0.0 on the faces at 0."""
    g = np.arange(-2.0, 2.01, 0.5, dtype=F)
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(F)
    up = np.nextafter(lat, F(np.inf)); dn = np.nextafter(lat, F(-np.inf))
    rng = np.random.default_rng(11)
    mix = np.where(rng.uniform(size=lat.shape) < 0.5, up, dn).astype(F)
    z = lat.copy(); z[z == 0] = F(-0.0)
    return np.concatenate([lat, up, dn, mix, z]).astype(F)


def _face_boxes():
    return np.array([[0, 0, 0, 0.5, 0.5, 0.5], [-1, -0.5, 0, 0, 0.5, 1], [-2, -2, -2, -1.5, 2, 2], [0.5, 0.5, 0.5, 0.5, 1, 1],
                     [1, 1, 1, 1, 1, 1], [-0.5, -0.5, -0.5, 0.0, 0.0, 0.0], [1.5, -1, 0.5, 2.0, 1.5, 1.0]], F)


@pytest.mark.skipif(not po.ref_available(), reason="oracle/_ref (the real ikd_Tree.cpp) was not built")
def test_mirror_face_rule_equals_the_real_tree_on_box_faces():
    pts = _face_points()
    ny = np.full(len(pts), 0.001, F)
    ids = np.arange(len(pts), dtype=np.int32)
    # Delete_Point_Boxes, box by box, including degenerate ones
    for b in _face_boxes():
        tree = po.RefTree(box_length=0.5); mir = nm.MirrorMap()
        tree.build(pts, ny, ids); mir.build(pts, ny, ids)
        assert tree.delete_boxes(b[None]) == mir.delete_boxes(b[None]), b
        tree.wait_rebuild()
        fx, fny, fid = tree.flatten_points()
        lx, lny, lid = mir.live_points()
        assert np.array_equal(np.sort(fid), np.sort(lid)), b
        tree.close()
    # Box_Search over the voxel boxes of 0.5 m whose faces carry the points (collect_voxel_sync)
    tree = po.RefTree(box_length=0.5)
    tree.build(pts, ny, ids)
    seeds = np.array([[0.25, 0.25, 0.25], [-0.25, 0.25, -0.25], [1.75, -1.75, 0.25], [-0.25, -0.25, -0.25]], F)
    s = tree.collect_sync(seeds, 0.5)
    mir = nm.MirrorMap(); mir.build(pts, ny, ids)
    at = 0
    for b, c in zip(s["boxes"], s["counts"]):
        m = mir._inside(b)
        got = s["ids"][at: at + int(c)]; at += int(c)
        assert np.array_equal(np.sort(got), np.sort(mir.ids[m])), b
        assert m.sum() > 0
    tree.close()
