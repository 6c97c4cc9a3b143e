"""The edge instances of test_gpu_reloc_edges.py without a GPU: each one is built to tell a mistake apart, so each planted
mistake in the restatements (tests/reloc_ref.py, tests/place_ref.py) must change the expected result on at least one of them:
the voxel of w * (1 / res) instead of w / res, non-finite points counted, ties to the last maximum, a pyramid whose z axis stops
splitting with x and y, truncating division for the lattice start, query columns by floor or by round-half-even, '>' at sector
boundaries, stage-2 ties to the largest shift, and occlusion that also empties the blocking bin.  The planted properties
themselves are asserted too: dz > dxy, negative lattice starts that are not multiples of the step, half-boundary query points
and 45-degree offsets in the stencil."""
import numpy as np
import pytest

import place_ref as PR
import reloc_ref as RR
import test_gpu_reloc_edges as E


# ------------------------------------------------------------------ malio_relocalize
def _result(r):
    return (r["yaw_index"], r["offset"], r["score"], r["n_points"])


def test_reciprocal_voxels_change_the_face_instance(monkeypatch):
    case = E.faces(0.7)
    want = E.reloc_want(case)
    w = case["pts"]["xyz"].astype(np.float64)
    assert (np.floor(w[:, :2] / 0.7) != np.floor(w[:, :2] * (1.0 / 0.7))).all()
    for res in (0.1, 0.3):                         # no float32 multiple of these splits the two forms
        allw, d = E.face_coords(res)
        assert len(d) == 0 and len(allw) == 3001
    base = RR.base_voxels

    def reciprocal(s, tc, pts, q, res):
        b, n = base(s, tc, pts, q, res)
        w = RR.world_ref.register_world(RR._with_rot(s, q), tc, pts["xyz"], pts["lidar"].astype(np.int64), 0.0)[:, :3]
        w = w[np.all(np.isfinite(w), axis=1)].astype(np.float64)
        return np.floor(w * (1.0 / res)).astype(np.int64), n

    monkeypatch.setattr(RR, "base_voxels", reciprocal)
    bad = E.reloc_want(case)
    assert _result(bad) != _result(want) and bad["score"] < want["score"]


def test_counting_non_finite_points_changes_the_non_finite_instances(monkeypatch):
    mixed, none = E.nonfinite(0, "mixed"), E.nonfinite(1, "none")
    want = [E.reloc_want(c) for c in (mixed, none)]
    assert want[0]["n_points"] == len(mixed["pts"]) - 20 and want[1]["n_points"] == 0 and want[1]["score"] == 0
    base = RR.base_voxels

    def counted(s, tc, pts, q, res):
        b, _ = base(s, tc, pts, q, res)
        return b, len(pts)

    monkeypatch.setattr(RR, "base_voxels", counted)
    bad = E.reloc_want(mixed)
    assert bad["n_points"] == len(mixed["pts"]) != want[0]["n_points"]


def test_ties_to_the_last_maximum_change_the_ground_instance():
    want = E.reloc_want(E.ground_tie())
    sc = want["scores"]
    assert sc.size == 13122 and (sc == sc.max()).all()
    last = sc.size - 1 - int(np.argmax(sc.ravel()[::-1]))
    assert np.unravel_index(last, sc.shape) != (want["yaw_index"], 0, 0, 0)
    assert want["offset"] == (-40, -40, 0) and want["yaw_index"] == 0


def _pyramid_z_stops_with_xy(g0, half_xy, half_z):
    dxy, dz = RR.ceil_log2(2 * half_xy + 1), RR.ceil_log2(2 * half_z + 1)
    levels = [g0]
    for l in range(1, max(dxy, dz) + 1):
        g, s = levels[-1], 1 << (l - 1)
        if l <= dxy:
            g = RR._shift_or(RR._shift_or(g, 0, s), 1, s)
            if l <= dz:
                g = RR._shift_or(g, 2, s)
        levels.append(g)
    return levels, dxy, dz


def _top_bound(case, want, pyramid):
    """The top node's bound (yaw of the best candidate, corner 0) over the box the device builds."""
    a = case["args"]
    b, _ = RR.base_voxels(case["guess"], case["tc"], case["pts"], want["rot"], a["res"])
    H = np.array([a["half_xy"], a["half_xy"], a["half_z"]])
    W = 2 * H + 1
    d = np.array([RR.ceil_log2(w) for w in W])
    lo = b.min(axis=0) - H
    g0 = RR._occupancy(RR.prior_voxels(case["prior"], a["res"]), lo, b.max(axis=0) - b.min(axis=0) + W + (1 << d))
    levels, _, _ = pyramid(g0, a["half_xy"], a["half_z"])
    return RR.node_bound(levels[-1], b - b.min(axis=0), (0, 0, 0))


def test_a_pyramid_whose_z_stops_with_xy_is_not_admissible_on_the_z_deeper_instances():
    below = 0
    for hxy, hz in E.Z_DEEPER:
        assert RR.ceil_log2(2 * hz + 1) > RR.ceil_log2(2 * hxy + 1)
        case = E.z_deeper(hxy, hz)
        want = E.reloc_want(case)
        assert _top_bound(case, want, RR.pyramid) >= want["score"] > 0
        below += _top_bound(case, want, _pyramid_z_stops_with_xy) < want["score"]
    assert below >= 1


# ------------------------------------------------------------------ the place database
def _lattice_cases():
    return [c for c in E.db_cases() if c[0].startswith("lattice")]


def test_lattice_instances_start_at_negative_columns_that_are_not_multiples():
    for name, prior, args in _lattice_cases():
        p = prior()
        m = int(round(args.step / args.cell))
        ilo = int(np.floor(p[:, 0].astype(np.float64) / args.cell).min())
        jlo = int(np.floor(p[:, 1].astype(np.float64) / args.cell).min())
        assert ilo < 0 and jlo < 0 and ilo % m and jlo % m, name


def _occupied(p, cell):
    return {(int(i), int(j)) for i, j in zip(np.floor(p[:, 0].astype(np.float64) / cell), np.floor(p[:, 1].astype(np.float64) / cell))}


def test_truncating_division_for_the_lattice_start_changes_a_lattice_instance():
    changed = 0
    for name, prior, args in _lattice_cases():
        p = prior()
        m = int(round(args.step / args.cell))
        occ = _occupied(p, args.cell)
        ilo, jlo = min(i for i, _ in occ), min(j for _, j in occ)
        want = sorted((j, i) for i, j in occ if i % m == 0 and j % m == 0)
        db = PR.database(p, args)
        assert [tuple(c) for c in db["cols"][:, ::-1].tolist()] == want, name
        ia, ja = int((ilo + m - 1) / m) * m, int((jlo + m - 1) / m) * m      # C's (a + m - 1) / m: a ceiling only for a >= 0
        bad = sorted((j, i) for i, j in occ if i % m == 0 and j % m == 0 and i >= ia and j >= ja)
        changed += bad != want
    assert changed >= 1


def test_forty_five_degree_offsets_are_in_the_stencil_and_a_strict_boundary_changes_the_database(monkeypatch):
    name, prior, args = [c for c in E.db_cases() if c[0] == "sectors-8"][0]
    tab = PR.table(args)
    diag = (tab["ox"] == tab["oy"]) & (tab["ox"] > 0)
    assert diag.sum() >= 10 and (tab["sector"][diag] == 1).all()      # on the boundary: the counter-clockwise sector
    p = prior()
    want = PR.database(p, args)
    sector_of = PR.sector_of

    def strict(a, x, y, b=None):
        a = PR._args_dict(a)
        bx, by = PR.boundaries(a) if b is None else b
        s = sector_of(a, x, y, b)
        Q = a["n_sector"] // 4
        q = s // Q
        u, v = [(x, y), (y, -x), (-x, -y), (-y, x)][q]
        return q * Q + sum(1 for j in range(1, Q) if bx[j] * v - by[j] * u > 0.0)

    monkeypatch.setattr(PR, "sector_of", strict)
    assert (PR.table(args)["sector"][diag] == 0).all()
    bad = PR.database(p, args)
    assert not np.array_equal(bad["levels"], want["levels"])


def test_occlusion_that_empties_the_blocking_bin_changes_the_database(monkeypatch):
    name, prior, args = [c for c in E.db_cases() if c[0] == "block-1"][0]
    p = prior()
    want = PR.database(p, args)

    def with_blocker(a, d):
        a = PR._args_dict(a)
        X = np.asarray(d, np.int64).reshape(a["n_ring"], a["n_sector"]).copy()
        for c in range(a["n_sector"]):
            hit = np.flatnonzero(X[:, c] >= a["block_level"])
            if len(hit):
                X[hit[0]:, c] = 0
        return X.ravel()

    monkeypatch.setattr(PR, "occlude", with_blocker)
    assert not np.array_equal(PR.database(p, args)["levels"], want["levels"])


# ------------------------------------------------------------------ the query and the ranking
@pytest.mark.parametrize("column", [lambda rel, cell: np.floor(rel / cell), lambda rel, cell: np.rint(rel / cell)],
                         ids=["floor", "half-even"])
def test_query_columns_by_another_rounding_change_the_half_boundary_instance(monkeypatch, column):
    case = E.query_case("half", 8)
    args, pts = case["args"], case["pts"][0]
    w = pts["xyz"].astype(np.float64)
    fin = np.all(np.isfinite(w), axis=1)
    t = w[fin, 0] / args.cell + 0.5
    assert (t == np.floor(t)).sum() >= (fin.sum() - 4) // 2                  # half-boundary points (rel = w: identity pose)
    assert (~fin).sum() == 5 and (np.abs(w[fin, :2]).max(axis=1) > args.r_max).sum() == 4
    q, _ = PR.query(case["guess"], None, pts, args)
    monkeypatch.setattr(PR, "query_column", column)
    bad, _ = PR.query(case["guess"], None, pts, args)
    assert not np.array_equal(bad, q)


def test_stage_two_ties_to_the_largest_shift_change_the_quarter_instance():
    case = E.query_case("quarter", 8)
    args = case["args"]
    want = E.query_want(case)
    p0 = E.quarter_position(want["db"])
    Q = args.n_sector // 4
    ds = PR.shift_distances(want["q"], want["db"]["levels"][p0], args.n_ring, args.n_sector)
    assert ds.min() == 0 and [s for s in range(args.n_sector) if ds[s] == 0][:4] == [0, Q, 2 * Q, 3 * Q]
    k = want["p2"].tolist().index(p0)
    assert want["sh"][k] == 0
    last = args.n_sector - 1 - int(np.argmin(ds[::-1]))
    assert last == 3 * Q != want["sh"][k]
