"""The session layer's restatement (tests/prior_extend_ref.py) pinned to the real ikd-Tree: build the tree from a live set, call
Add_Points(admitted ADD, true) and Add_Points(admitted NO_DOWNSAMPLE, false), and the tree's points must equal the live set plus
the restatement's inserts, as a multiset, bit for bit.  Planted cases sit one float32 ulp either side of box faces, on a box's
max face, in both downsample_size/8 branches of the fold with equal normal_y and within EPSS, and put a no-downsample point
beside a fold winner; each deliberately wrong variant changes one of them."""
import numpy as np
import pytest

import prior_extend_ref as E
import pyoracle as po
from malio_b200 import capi

F = np.float32
ADD, NODS = capi.MAP_ADD, capi.MAP_ADD_NO_DOWNSAMPLE


def _face(f, ds):
    return F(F(f) * F(ds))


def _mid(f, ds):
    lo = _face(f, ds)
    hi = F(lo + F(ds))
    return F(np.float64(lo) + np.float64(F(hi - lo)) / 2.0)


def _row(r, ds):
    """y, z of planted row r: the centre of box (10 + 3 r, 4) so that rows never share a box."""
    return _mid(10 + 3 * r, ds), _mid(4, ds)


def _rounded_down_face(ds):
    """A box index whose float min face lies below f * ds (exact): a live point there is inside the float box only.  At a power
    of two every face is exact: any face serves."""
    for f in range(160, 4000):
        if np.float64(_face(f, ds)) < np.float64(f) * np.float64(F(ds)):
            return f
    return 160


def planted(ds):
    """(live xyz, live ids, cls, world) of the planted cases; live ids < 0 are session points."""
    live, lids, cls, pts = [], [], [], []
    up, dn = (lambda v: np.nextafter(v, F(np.inf))), (lambda v: np.nextafter(v, F(-np.inf)))

    def cand(x, r, c=ADD, dy=F(0), dz=F(0)):
        y, z = _row(r, ds)
        pts.append([x, F(y + dy), F(z + dz)]); cls.append(c)

    # 0: one ulp either side of a box face, and on it
    lo = _face(40, ds)
    for k, x in enumerate((dn(lo), lo, up(lo))):
        cand(x, 0 + k)
    # 3: a box whose only live point lies on its max face (half-open: the box is empty, the candidate admitted) and one whose
    # live point lies on its min face (not admitted)
    y, z = _row(3, ds)
    live.append([_face(61, ds), y, z]); lids.append(7)
    cand(_mid(60, ds), 3)
    y, z = _row(4, ds)
    live.append([_face(70, ds), y, z]); lids.append(8)
    cand(_mid(70, ds), 4)
    # 5: two candidates near the centre (squared distance < downsample_size/8, equal normal_y: the newer one wins), three
    # with a far one in the middle (the distance branch: the nearer one is kept), two within EPSS of each other, two at equal
    # distances on either side, far from the centre (strict <: the newer one wins)
    m = _mid(80, ds); e = F(ds * 0.05)
    cand(F(m + e), 5); cand(F(m - e), 5)
    m = _mid(90, ds); a = F(0.45 * ds)
    cand(F(m + e), 6); cand(F(m + a), 6, ADD, a, a); cand(F(m - F(ds * 0.02)), 6)
    m = _mid(100, ds)
    cand(F(m + F(ds * 0.3)), 7); cand(up(F(m + F(ds * 0.3))), 7)
    m = _mid(110, ds); d = F(0.125 if ds < 0.375 else 0.1875)      # exact offsets: both distances are the same float
    cand(F(m + d), 8, ADD, d, d); cand(F(m - d), 8, ADD, -d, -d)
    # 9: a no-downsample point in the box of a fold winner, and two no-downsample points in one box
    m = _mid(120, ds)
    cand(m, 9); cand(F(m + e), 9, NODS)
    m = _mid(130, ds)
    cand(m, 10, NODS); cand(F(m + e), 10, NODS)
    # 11: a box holding a prior point and one holding a session point
    m = _mid(140, ds)
    y, z = _row(11, ds)
    live.append([F(m + e), y, z]); lids.append(9)
    cand(m, 11)
    y, z = _row(12, ds)
    live.append([F(m + e), y, z]); lids.append(-1)
    cand(m, 12)
    # 13: a live point on a float min face that lies below f * ds: inside the float box, outside the double one
    f = _rounded_down_face(ds)
    y, z = _row(13, ds)
    live.append([_face(f, ds), y, z]); lids.append(10)
    cand(_mid(f, ds), 13)
    # skipped / dropped points are never candidates
    cand(_mid(150, ds), 14, capi.MAP_SKIP); cand(_mid(151, ds), 14, capi.MAP_DROP)
    rng = np.random.default_rng(3)
    far = rng.uniform(-30, -5, (400, 3)).astype(F)         # live points away from every planted box
    live = np.concatenate([np.array(live, F), far])
    lids = np.concatenate([np.array(lids, np.int32), np.arange(100, 500, dtype=np.int32)])
    return live, lids, np.array(cls, np.uint8), np.array(pts, F)


def _rows(xyz, ny):
    a = np.concatenate([np.asarray(xyz, F).reshape(-1, 3), np.asarray(ny, F).reshape(-1, 1)], axis=1)
    return sorted(map(bytes, a))


def _tree_matches(live, lids, cls, world, ds):
    r = E.extend(cls, world, ds, live, lids)
    t = po.RefTree(box_length=F(ds))
    t.build(live, np.full(len(live), E.SESSION_NY, F), lids)
    a, nd = world[r["add_mask"]], world[r["nods_mask"]]
    if len(a):
        t.add_points(a, np.full(len(a), E.SESSION_NY, F), downsample=True)
    if len(nd):
        t.add_points(nd, np.full(len(nd), E.SESSION_NY, F), downsample=False)
    t.wait_rebuild()
    xyz, ny, _ = t.flatten_points()
    t.close()
    ins = world[r["inserted"]]
    assert _rows(xyz, ny) == _rows(np.concatenate([live, ins]), np.full(len(live) + len(ins), E.SESSION_NY, F))
    return r


needs_ref = pytest.mark.skipif(not po.ref_available(), reason="oracle/_ref (the real ikd-Tree) is not built")


@needs_ref
@pytest.mark.parametrize("ds", [0.5, 0.3, 0.4])
def test_planted_cases_equal_the_real_tree(ds):
    live, lids, cls, world = planted(ds)
    r = _tree_matches(live, lids, cls, world, ds)
    assert r["n_candidates"] == int(np.sum((cls == ADD) | (cls == NODS)))
    ins = set(r["inserted"].tolist())
    if ds == 0.5:                                          # exact faces: the ulp cases land in three boxes (elsewhere the
        assert {0, 1, 2} <= ins                            # sole-box rule may hold one back; the tree check covers that)
    assert 3 in ins and 4 not in ins                       # max face: the box is empty; min face: occupied
    assert 6 in ins and 5 not in ins                       # /8 branch, equal normal_y: the newer point wins
    assert 9 in ins and not {7, 8} & ins                   # the far one loses to the kept one, which loses to the last
    assert 11 in ins and 10 not in ins                     # within EPSS: the newer point
    assert 13 in ins and 12 not in ins                     # equal distances, strict <: the newer point wins
    assert {14, 15, 16, 17} <= ins                         # no-downsample points beside a winner and beside each other
    assert not {18, 19, 20, 21, 22} & ins                  # prior point, session point, rounded-down face, skip, drop
    order = r["inserted"]
    nods = np.flatnonzero(r["nods_mask"])
    assert np.array_equal(order[-len(nods):], nods)        # winners by caller index, then the no-downsample points
    assert np.all(np.diff(order[:-len(nods)]) > 0)


@needs_ref
@pytest.mark.parametrize("ds", [0.3, 0.4, 0.5])
def test_random_candidates_at_box_faces_equal_the_real_tree(ds):
    """Candidates clustered on box faces, corners and near each other, against a live set with gaps: the sole-box rule keeps the
    fold exact where the faces round."""
    rng = np.random.default_rng(int(ds * 10))
    d = F(ds)
    idx = rng.integers(0, 12, (3000, 3)).astype(F)
    faces = (idx * d).astype(F)
    jitter = rng.integers(-2, 3, (3000, 3))
    world = faces.copy()
    for _ in range(2):
        world = np.where(jitter > 0, np.nextafter(world, F(np.inf)), np.where(jitter < 0, np.nextafter(world, F(-np.inf)), world))
    inner = rng.random(3000) < 0.5
    world[inner] = (faces[inner] + rng.uniform(0, ds, (int(inner.sum()), 3))).astype(F)
    cls = rng.choice([ADD, ADD, ADD, NODS, capi.MAP_DROP], 3000).astype(np.uint8)
    live = rng.uniform(0, 12 * ds, (300, 3)).astype(F)
    r = _tree_matches(live, np.arange(300, dtype=np.int32), cls, world, ds)
    assert r["n_admitted"] > 50 and len(r["inserted"]) < r["n_admitted"]


def test_each_wrong_variant_changes_a_planted_case():
    ds = 0.3
    live, lids, cls, world = planted(ds)
    want = E.extend(cls, world, ds, live, lids)["inserted"].tolist()
    for v in E.VARIANTS:
        got = E.extend(cls, world, ds, live, lids, variant=v)["inserted"].tolist()
        assert got != want, v


def test_session_window_keeps_prior_and_session_in_the_cube():
    """The restated window: first call prior ∩ cube then session ∩ cube; a move appends (new ∖ old) of each."""
    rng = np.random.default_rng(5)
    prior = rng.uniform(-60, 0, (3000, 3)).astype(F)
    w = E.SessionWindow(prior, np.full(3000, 0.001, F), np.arange(3000, dtype=np.int32), 40.0, 5.0)
    w.step((0.0, 0.0, 0.0))
    world = rng.uniform(0, 19, (500, 3)).astype(F)
    rep = w.extend(np.full(500, ADD, np.uint8), world, 0.5)
    assert rep["n_inserted"] > 0 and np.all(w.ids[-1] < 0)
    ids0 = set(w.ids.tolist())
    w.step((-15.0, 0.0, 0.0))          # slide away: session points past the new cube's max face leave
    w.step((15.0, 0.0, 0.0))           # and back: they re-enter after the prior's share
    cube = w.cube
    want_p = set(np.flatnonzero(np.all((cube[:3] <= prior) & (prior < cube[3:]), axis=1)).tolist())
    s = w.sxyz
    want_s = set((-1 - np.flatnonzero(np.all((cube[:3] <= s) & (s < cube[3:]), axis=1))).tolist())
    assert set(w.ids.tolist()) == {int(i) for i in w.pids[[i in want_p for i in w.pids]]} | want_s
    assert ids0 & want_s
