"""Localization in a prior map without a GPU: the restated lasermap_fov_segment (tests/prior_map_ref.py) at the move threshold,
on the slab faces and through the real ikd-Tree, and malio_read_pcd against the files this library and PCL write."""
import ctypes as C
import os

import numpy as np
import pytest

import prior_map_ref as R
import pyoracle as po
from malio_b200 import capi, plugin

F = np.float32
INF = F(np.inf)


def up(v, k=1):
    v = F(v)
    for _ in range(k):
        v = np.nextafter(v, INF)
    return v


def down(v, k=1):
    v = F(v)
    for _ in range(k):
        v = np.nextafter(v, -INF)
    return v


# ---------------------------------------------------------------- the move decision and the new cube
CUBE, DET = 1000.0, 100.0          # thr = 150.0f, mov_dist = (1000 - 300) * 0.45 = 315.0f


def test_initial_cube_is_the_float_of_the_double_half_length():
    pos = (0.1, -1e5 + 0.3, 7.7)
    c = R.init_cube(pos, 1000.1)
    for i in range(3):
        assert c[i] == F(pos[i] - 1000.1 / 2.0) and c[3 + i] == F(pos[i] + 1000.1 / 2.0)
    assert c.dtype == F


@pytest.mark.parametrize("face", ["min", "max"])
def test_move_threshold_at_one_ulp(face):
    cube = R.init_cube((0.0, 0.0, 0.0), CUBE)            # [-500, 500)^3
    thr = F(150.0)
    for i in range(3):
        for d, moves in ((thr, True), (down(thr), True), (up(thr), False)):
            pos = np.zeros(3)
            pos[i] = float(cube[i]) + float(d) if face == "min" else float(cube[3 + i]) - float(d)
            moved, new, slabs = R.segment(cube, pos, CUBE, DET)
            assert moved == moves, (i, d)
            if not moves:
                assert np.array_equal(new, cube) and slabs.shape == (0, 6)
                continue
            exp = cube.copy()
            sgn = -1 if face == "min" else 1
            exp[i] = F(cube[i] + sgn * F(315.0)); exp[3 + i] = F(cube[3 + i] + sgn * F(315.0))
            assert np.array_equal(new, exp)
            slab = cube.copy()
            if face == "min":
                slab[i] = F(cube[3 + i] - F(315.0))
            else:
                slab[3 + i] = F(cube[i] + F(315.0))
            assert np.array_equal(slabs, slab[None])


def test_distance_is_rounded_to_float_before_the_comparison():
    """|pos - min| = 150 + 1e-9 in double moves the cube: the reference stores the distance as a float first (:191)."""
    cube = R.init_cube((0.0, 0.0, 0.0), CUBE)
    moved, _, _ = R.segment(cube, (-350.0 + 1e-9, 0.0, 0.0), CUBE, DET)
    assert moved
    assert np.float64(-350.0 + 1e-9) - np.float64(cube[0]) > 150.0     # a double comparison would not move


@pytest.mark.parametrize("pos,axes", [((-400.0, 0.0, 0.0), [0]), ((400.0, 450.0, 0.0), [0, 1]), ((-420.0, 420.0, -499.0), [0, 1, 2])])
def test_moves_along_one_two_and_three_axes(pos, axes):
    cube = R.init_cube((0.0, 0.0, 0.0), CUBE)
    moved, new, slabs = R.segment(cube, pos, CUBE, DET)
    assert moved and slabs.shape == (len(axes), 6)
    for i in range(3):
        shift = 0.0 if i not in axes else (-315.0 if pos[i] < 0 else 315.0)
        assert new[i] == F(cube[i] + F(shift)) and new[3 + i] == F(cube[3 + i] + F(shift))


def test_jump_longer_than_the_cube_moves_by_mov_dist_once():
    """Beyond the cube both distances exceed the threshold on the far side only: the reference tests the min face first."""
    cube = R.init_cube((0.0, 0.0, 0.0), CUBE)
    moved, new, slabs = R.segment(cube, (3000.0, 0.0, 0.0), CUBE, DET)
    # dist to min = 3500, dist to max = 2500: neither <= 150, no move (the reference keeps its cube)
    assert not moved
    moved, new, slabs = R.segment(cube, (640.0, 0.0, 0.0), CUBE, DET)   # past max by 140: |pos - max| = 140 <= 150
    assert moved and new[0] == F(-185.0) and new[3] == F(815.0)
    assert np.array_equal(slabs[0], np.array([-500, -500, -500, -185, 500, 500], F))


def test_mov_dist_small_cube_takes_the_det_range_branch():
    assert R.mov_dist(100.0, 100.0) == F(50.0)            # (100 - 300) * 0.45 < 0 -> DET_RANGE * 0.5f
    assert R.mov_dist(1000.0, 100.0) == F(315.0)
    assert R.mov_dist(1000.1, 100.0) == F((1000.1 - 300.0) * 0.45)


# ---------------------------------------------------------------- the slabs are exactly old ∖ new
def _face_points(boxes, extra=()):
    """Points on every face of every box, one ulp either side, on every axis; plus the box corners and `extra`."""
    pts = []
    for b in np.asarray(boxes, F).reshape(-1, 6):
        mid = [F((np.float64(b[a]) + np.float64(b[3 + a])) / 2) for a in range(3)]
        for a in range(3):
            for v in (b[a], b[3 + a]):
                for w in (down(v), F(v), up(v)):
                    p = list(mid)
                    p[a] = w
                    pts.append(p)
        pts.append(list(b[:3])); pts.append(list(b[3:]))
    pts.extend(extra)
    return np.array(pts, F).reshape(-1, 3)


@pytest.mark.parametrize("offset", [0.0, 1e5, -1e5])
@pytest.mark.parametrize("pos", [(-400.0, 0.0, 0.0), (400.0, 0.0, 0.0), (0.0, -400.0, 0.0), (0.0, 400.0, 0.0),
                                 (0.0, 0.0, -400.0), (0.0, 0.0, 400.0), (-420.0, 420.0, -420.0), (440.0, 440.0, 440.0)])
def test_slabs_union_to_old_minus_new(pos, offset):
    cube = R.init_cube((offset, offset, 0.0), 1000.0)
    p = (pos[0] + offset, pos[1] + offset, pos[2])
    moved, new, slabs = R.segment(cube, p, 1000.0, 100.0)
    assert moved
    xyz = _face_points(np.concatenate([cube[None], new[None], slabs]), extra=[[-0.0, -0.0, -0.0], [0.0, -0.0, 0.0]])
    old_in, new_in, killed = R.in_box(xyz, cube), R.in_box(xyz, new), R.in_any(xyz, slabs)
    assert np.array_equal(old_in & killed, old_in & ~new_in)
    assert np.array_equal(old_in & ~killed, old_in & new_in)
    assert (old_in & killed).any() and (old_in & ~killed).any()


# ---------------------------------------------------------------- through the real ikd-Tree
def _tree_live_ids(tree):
    nodes, _, ids, _, _ = tree.snapshot()
    return np.sort(ids[(nodes["link"] & capi.LINK_POINT_DELETED) == 0])


def _prior(rng, n, half, offset=0.0):
    xyz = np.column_stack([rng.uniform(-half, half, n), rng.uniform(-half, half, n), rng.uniform(-20, 20, n)]) + [offset, offset, 0]
    return xyz.astype(F)


@pytest.mark.skipif(not po.ref_available(), reason="oracle/_ref (the reference's ikd_Tree.cpp) is not built")
@pytest.mark.parametrize("offset", [0.0, 1e5])
def test_reference_tree_holds_prior_cap_cube_after_every_slide(offset):
    rng = np.random.default_rng(3)
    cube_len, det = 40.0, 5.0
    prior = _prior(rng, 6000, 80.0, offset)
    w = R.Window(prior, cube_len, det)
    origin = (offset, offset, 0.0)
    w.step(R.drive_pos(w, R.DRIVE[0], origin))
    prior = np.concatenate([prior, _face_points(w.cube[None])])   # points on the first cube's faces, one ulp either side
    w = R.Window(prior, cube_len, det)
    tree = po.RefTree(box_length=0.5)
    moves = 0
    for k, d in enumerate(R.DRIVE):
        pos = R.drive_pos(w, d, origin)
        before = w.live() if w.cube is not None else None
        init, moved, slabs = w.step(pos)
        moves += moved
        live = w.live()
        if init:
            tree.build(prior[live], np.full(len(live), 0.001, F), live.astype(np.int32))
        elif moved:
            tree.delete_boxes(slabs)
            enter = np.setdiff1d(live, before)
            tree.add_points(prior[enter], np.full(len(enter), 0.001, F), enter.astype(np.int32), downsample=False)
        tree.wait_rebuild()
        assert np.array_equal(_tree_live_ids(tree), np.sort(live)), k
    assert moves >= 12
    tree.close()


# ---------------------------------------------------------------- the test can see a wrong restatement
def test_wrong_variants_change_a_planted_outcome():
    cube = R.init_cube((0.0, 0.0, 0.0), CUBE)
    on_thr = (float(cube[0]) + 150.0, 0.0, 0.0)
    assert R.segment(cube, on_thr, CUBE, DET)[0] and not R.segment(cube, on_thr, CUBE, DET, "strict")[0]
    c2 = R.init_cube((0.0, 0.0, 0.0), 1000.1)
    p2 = (float(c2[0]) + 100.0, 0.0, 0.0)
    _, new, _ = R.segment(c2, p2, 1000.1, DET)
    _, new_d, _ = R.segment(c2, p2, 1000.1, DET, "double_mov")
    assert not np.array_equal(new, new_d)
    face = np.array([[F(cube[3]), 0.0, 0.0]], F)                        # on the max face: outside a half-open box
    assert not R.in_box(face, cube)[0] and R.in_box(face, cube, "closed")[0]


# ---------------------------------------------------------------- malio_read_pcd
def _pcd(path, fields, sizes, types, counts, recs, n, data="binary", points=None, width=None, height=1):
    hdr = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\n"
           f"FIELDS {' '.join(fields)}\nSIZE {' '.join(map(str, sizes))}\nTYPE {' '.join(types)}\nCOUNT {' '.join(map(str, counts))}\n"
           f"WIDTH {n if width is None else width}\nHEIGHT {height}\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n if points is None else points}\n"
           f"DATA {data}\n")
    with open(path, "wb") as f:
        f.write(hdr.encode() + recs)


def test_read_pcd_round_trips_the_writer_byte_for_byte(tmp_path):
    rng = np.random.default_rng(0)
    xyzi = rng.normal(0, 100, (70001, 4)).astype(F)
    xyzi[5] = [-0.0, np.inf, np.nan, 1e-45]
    a, b = str(tmp_path / "a.pcd"), str(tmp_path / "b.pcd")
    plugin.write_pcd_binary(a, xyzi)
    back = plugin.read_pcd(a)
    assert back.tobytes() == xyzi.tobytes()
    plugin.write_pcd_binary(b, back)
    assert open(a, "rb").read() == open(b, "rb").read()


@pytest.mark.parametrize("layout", ["PointXYZ", "PointXYZI", "PointXYZINormal", "padded"])
def test_read_pcd_layouts(tmp_path, layout):
    rng = np.random.default_rng(1)
    n = 1000
    xyzi = rng.normal(0, 10, (n, 4)).astype(F)
    if layout == "PointXYZ":
        spec = (["x", "y", "z"], [4, 4, 4], ["F", "F", "F"], [1, 1, 1]); rec = xyzi[:, :3]
        want = np.column_stack([xyzi[:, :3], np.zeros(n, F)])
    elif layout == "PointXYZI":
        spec = (["x", "y", "z", "intensity"], [4] * 4, ["F"] * 4, [1] * 4); rec = xyzi; want = xyzi
    elif layout == "PointXYZINormal":
        spec = (["x", "y", "z", "intensity", "normal_x", "normal_y", "normal_z", "curvature"], [4] * 8, ["F"] * 8, [1] * 8)
        rec = np.column_stack([xyzi, rng.normal(0, 1, (n, 4)).astype(F)]); want = xyzi
    else:   # a PCLPointCloud2 layout: padding field "_", a double, an rgb word, intensity before xyz
        dt = np.dtype([("intensity", "<f4"), ("_", "u1", 4), ("x", "<f4"), ("t", "<f8"), ("y", "<f4"), ("z", "<f4"), ("rgb", "<u4")])
        r = np.zeros(n, dt); r["x"], r["y"], r["z"], r["intensity"] = xyzi.T; r["t"] = 1.5; r["rgb"] = 7
        spec = (["intensity", "_", "x", "t", "y", "z", "rgb"], [4, 1, 4, 8, 4, 4, 4], ["F", "U", "F", "F", "F", "F", "U"], [1, 4, 1, 1, 1, 1, 1])
        rec = r; want = xyzi
    p = str(tmp_path / "l.pcd")
    _pcd(p, *spec, np.ascontiguousarray(rec).tobytes(), n)
    assert plugin.read_pcd(p).tobytes() == np.ascontiguousarray(want).tobytes()


def test_read_pcd_refuses_without_crashing(tmp_path):
    lib = capi.load()
    xyz = np.zeros((10, 4), F).tobytes()
    spec = (["x", "y", "z", "intensity"], [4] * 4, ["F"] * 4, [1] * 4)
    cases = {
        "ascii": dict(data="ascii"), "compressed": dict(data="binary_compressed"), "truncated": dict(cut=5),
        "points_mismatch": dict(points=11), "width_mismatch": dict(width=5), "height": dict(height=2),
    }
    for name, kw in cases.items():
        p = str(tmp_path / f"{name}.pcd")
        cut = kw.pop("cut", 0)
        _pcd(p, *spec, xyz[: len(xyz) - cut], 10, **kw)
        with pytest.raises(capi.MalioError) as e:
            plugin.read_pcd(p)
        assert e.value.status == capi.ERR_INVALID_ARG, name
    bad = {"double_x": (["x", "y", "z"], [8, 4, 4], ["F", "F", "F"], [1, 1, 1]), "no_z": (["x", "y"], [4, 4], ["F", "F"], [1, 1]),
           "int_x": (["x", "y", "z"], [4, 4, 4], ["I", "F", "F"], [1, 1, 1]), "size_count": (["x", "y", "z"], [4, 4], ["F"] * 3, [1] * 3)}
    for name, sp in bad.items():
        p = str(tmp_path / f"{name}.pcd")
        _pcd(p, *sp, xyz, 10)
        with pytest.raises(capi.MalioError) as e:
            plugin.read_pcd(p)
        assert e.value.status == capi.ERR_INVALID_ARG, name
    for junk in (b"", b"VERSION 0.7\n", b"\x00" * 4096, b"FIELDS x y z\nDATA binary\n"):
        p = str(tmp_path / "junk.pcd")
        open(p, "wb").write(junk)
        n = C.c_uint64(0)
        assert lib.malio_read_pcd(p.encode(), None, 0, C.byref(n)) == capi.ERR_INVALID_ARG
    assert lib.malio_read_pcd(str(tmp_path / "missing.pcd").encode(), None, 0, C.byref(C.c_uint64())) == capi.ERR_INVALID_ARG
    # a buffer smaller than the file's points: nothing read, the size reported
    p = str(tmp_path / "ok.pcd")
    _pcd(p, *spec, xyz, 10)
    out = np.full((4, 4), 7, F)
    n = C.c_uint64(0)
    assert lib.malio_read_pcd(p.encode(), capi.ptr(out), 4, C.byref(n)) == capi.ERR_CAPACITY
    assert n.value == 10 and np.all(out == 7)
    assert lib.malio_read_pcd(p.encode(), None, 4, C.byref(n)) == capi.ERR_INVALID_ARG
    assert lib.malio_read_pcd(p.encode(), capi.ptr(out), 4, None) == capi.ERR_INVALID_ARG


def test_prior_map_entry_points_refuse_a_null_handle():
    lib = capi.load()
    pos = np.zeros(3)
    rep = capi.WindowReport()
    assert lib.malio_prior_map_load(None, None, None, None, 0) == capi.ERR_INVALID_ARG
    assert lib.malio_prior_map_load_device(None, None, None, None, 0, None) == capi.ERR_INVALID_ARG
    assert lib.malio_prior_map_window(None, capi.ptr(pos), 1000.0, 100.0, C.byref(rep)) == capi.ERR_INVALID_ARG
    assert lib.malio_prior_map_info(None, None, None, None) == capi.ERR_INVALID_ARG
    assert lib.malio_prior_map_clear(None) == capi.ERR_INVALID_ARG
    assert C.sizeof(capi.WindowReport) == 4 * (2 + 6 + 1 + 18 + 3)
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "malio_b200.h")).read()
    assert "int malio_prior_map_window(malio_handle* h, const double pos_lid[3], double cube_len, float det_range" in hdr
