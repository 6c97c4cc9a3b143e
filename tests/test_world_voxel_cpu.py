"""The saved map as a voxel map without a GPU: the float32 restatement (tests/world_voxel_ref.py) pinned to the oracle's
pcl::VoxelGrid restatement (orc_voxel_grid, oracle/oracle_undistort.cpp) on the concatenation of the accumulated clouds, at voxel
faces, one ulp either side of them, -0.0 and non-finite points; then the new C-ABI signatures against the header, NULL handles
(in a subprocess: a missing check would be a segmentation fault), and the Python wrappers' argument checks, which run before
anything reaches the library."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import pyoracle as po
import world_voxel_ref as V
from malio_b200 import capi, plugin

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(clouds, leaf):
    """orc_voxel_grid of the concatenated clouds, curvature and the normals padded as 0: float32 (m, 4)."""
    cat = np.concatenate([np.asarray(c, F).reshape(-1, 4) for c in clouds])
    p8 = np.zeros((cat.shape[0], 8), F)
    p8[:, :4] = cat
    out, _ = po.voxel_grid(p8, leaf)
    return out[:, :4]


def _cloud(rng, n, center, spread, tag):
    c = np.zeros((n, 4), F)
    c[:, :3] = (np.asarray(center) + rng.normal(0, spread, (n, 3))).astype(F)
    c[:, 3] = tag
    return c


def _faces(leaf, ks, tag):
    """Points on voxel faces k * leaf (as float32, and as il-exact multiples) and one ulp either side, on every axis."""
    il = F(1.0) / F(leaf)
    vals = []
    for k in ks:
        for v in (F(k) * F(leaf), F(k) / il):
            vals += [v, np.nextafter(v, F(np.inf)), np.nextafter(v, F(-np.inf))]
    vals = np.array(vals, F)
    rng = np.random.default_rng(len(vals))
    pts = np.zeros((3 * vals.shape[0], 4), F)
    for ax in range(3):
        blk = pts[ax * vals.shape[0]:(ax + 1) * vals.shape[0]]
        blk[:, :3] = rng.uniform(-3, 3, (vals.shape[0], 3)).astype(F)
        blk[:, ax] = vals
    pts[:, 3] = tag
    return pts


def _both(clouds, leaf):
    a, b = V.VoxelMapRef(), V.VoxelMapRef()
    for c in clouds:
        a.accumulate(c, leaf)
        b.accumulate_fast(c, leaf)
    assert a.centroids().tobytes() == b.centroids().tobytes()
    assert a.cnt == b.cnt
    return a


@pytest.mark.parametrize("leaf", [0.5, 0.2, 0.1, 0.3])
def test_restatement_equals_the_oracle_voxel_grid_on_the_concatenation(leaf):
    rng = np.random.default_rng(int(leaf * 100))
    clouds = [_cloud(rng, 3000, [1.0 * k, -2.0, 0.5], 1.5, F(k % 3)) for k in range(4)]
    clouds.append(_faces(leaf, [-7, -1, 0, 1, 2, 13], F(1)))
    ref = _both(clouds, leaf)
    assert ref.centroids().tobytes() == _oracle(clouds, leaf).tobytes()
    assert sum(ref.cnt.values()) == sum(c.shape[0] for c in clouds)


def test_negative_zero_and_non_finite_points():
    leaf = 0.25
    c = np.array([[-0.0, 0.1, 0.1, 1], [0.0, 0.1, 0.1, 2], [0.1, -0.0, -0.0, 1], [np.nan, 0, 0, 5], [0, np.inf, 0, 5],
                  [0, 0, -np.inf, 5], [0.2, 0.2, 0.2, 3]], F)
    ref = _both([c, c[::-1].copy()], leaf)
    assert ref.centroids().tobytes() == _oracle([c, c[::-1]], leaf).tobytes()
    assert sum(ref.cnt.values()) == 8                     # the six non-finite rows are skipped
    ijk, finite, _ = V.voxel_index(c[:, :3], leaf)
    assert np.array_equal(ijk[0], ijk[1]) and finite.sum() == 4


def test_order_is_z_then_y_then_x_whatever_the_minimum():
    leaf = 1.0
    pts = np.array([[5, 0, 0], [-5, 1, 0], [0, -3, 0], [0, 0, -1], [3, 3, 3], [-9, -9, 2]], F)
    c = np.concatenate([pts, np.zeros((6, 1), F)], axis=1)
    ref = _both([c], leaf)
    keys = ref.keys()
    assert [tuple(k) for k in keys] == sorted(tuple(k) for k in keys)
    assert np.array_equal(ref.centroids()[:, :3], pts[np.lexsort((pts[:, 0], pts[:, 1], pts[:, 2]))])
    assert ref.centroids().tobytes() == _oracle([c], leaf).tobytes()


def test_sums_continue_across_clouds_and_are_not_reassociated():
    """One voxel fed by many clouds: the centroid is the running float32 sum over the concatenation, which differs from
    (old sum) + (this cloud's sum) for these values."""
    rng = np.random.default_rng(4)
    clouds = [np.concatenate([rng.uniform(0.0, 0.999, (37, 3)).astype(F), np.full((37, 1), F(0.1) * k, F)], axis=1)
              for k in range(30)]
    ref = _both(clouds, 1.0)
    assert len(ref.sums) == 1
    assert ref.centroids().tobytes() == _oracle(clouds, 1.0).tobytes()
    reassoc = np.zeros(4, F)
    for c in clouds:
        s = np.zeros(4, F)
        for row in c:
            s += row
        reassoc += s
    assert not np.array_equal(reassoc, ref.sums[(0, 0, 0)])


def test_refusals_leave_the_map_as_it_was():
    ref = V.VoxelMapRef()
    c = np.array([[1, 2, 3, 0], [1.1, 2, 3, 1]], F)
    ref.accumulate(c, 0.5)
    before = ref.centroids().tobytes()
    with pytest.raises(V.CapacityError):
        ref.accumulate(np.array([[0, 0, 0, 0], [3e9 * 0.5, 0, 0, 0]], F), 0.5)   # floor(x / leaf) = 3e9 > INT_MAX
    with pytest.raises(V.CapacityError):
        ref.accumulate_fast(np.array([[0, 0, -1.2e9, 0]], F), 0.5)
    with pytest.raises(V.LeafError):
        ref.accumulate(c, 0.25)
    assert ref.centroids().tobytes() == before and ref.leaf == F(0.5)
    ref.clear()
    ref.accumulate(c, 0.25)                               # a cleared map takes a new leaf
    assert ref.leaf == F(0.25)
    # the largest indices inside int are kept
    big = np.array([[2147483520.0, -2147483648.0, 0, 1]], F)
    m = V.VoxelMapRef()
    m.accumulate(big, 1.0)
    assert m.keys().tolist() == [[0, -2147483648, 2147483520]]


# ------------------------------------------------------------------ the C-ABI and the wrappers
NEW = ("malio_world_voxel_accumulate", "malio_world_voxel_download_device", "malio_world_voxel_save_pcd", "malio_world_voxel_info")
SCALARS = (("uint64_t", C.c_uint64), ("float", C.c_float), ("int", C.c_int))


def _header_args(name):
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    out = []
    for a in (re.sub(r"/\*.*?\*/", "", a).strip() for a in m.group(1).split(",")):
        if a.startswith("const char*"):
            out.append(C.c_char_p)
        elif "*" in a:
            out.append(C.c_void_p)
        else:
            types = [t for word, t in SCALARS if a.split()[0] == word]
            assert len(types) == 1, f"{name}: unexpected argument {a!r}"
            out.append(types[0])
    return out


@pytest.mark.parametrize("name", NEW)
def test_ctypes_signatures_match_the_header(name):
    fn = getattr(capi.load(), name)
    assert fn.argtypes == _header_args(name)
    assert fn.restype is C.c_int
    assert name in capi.EXPORTS


def test_header_signatures_carry_their_scalars():
    assert _header_args("malio_world_voxel_accumulate")[3] is C.c_float
    assert _header_args("malio_world_voxel_download_device")[2] is C.c_uint64
    assert _header_args("malio_world_voxel_save_pcd") == [C.c_void_p, C.c_char_p, C.c_int]


def test_null_handle_returns_an_error():
    code = textwrap.dedent("""
        import ctypes as C
        from malio_b200 import capi
        lib = capi.load()
        s, t, n = capi.PassState(), (C.c_float * 3)(), C.c_uint64(0)
        print("acc", lib.malio_world_voxel_accumulate(None, None, None, 0.5, None), flush=True)
        print("acc-args", lib.malio_world_voxel_accumulate(None, C.addressof(s), C.addressof(t), 0.5, C.addressof(n)), flush=True)
        print("down", lib.malio_world_voxel_download_device(None, None, 0, None, None), flush=True)
        print("down-count", lib.malio_world_voxel_download_device(None, None, 0, C.addressof(n), None), flush=True)
        print("save", lib.malio_world_voxel_save_pcd(None, None, 0), flush=True)
        print("save-path", lib.malio_world_voxel_save_pcd(None, b"/nonexistent/x.pcd", 1), flush=True)
        print("info", lib.malio_world_voxel_info(None, C.addressof(n), None, None), flush=True)
        print("DONE")
    """)
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "ma-lio_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "DONE" and len(lines) == 8
    for l in lines[:-1]:
        assert l.split()[-1] == str(capi.ERR_INVALID_ARG), l


class _Lib:
    """Stands in for the library: any call reaching it fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _model(L=3):
    m = object.__new__(plugin.MeasurementModel)   # no handle (no GPU here): only the Python-side checks can run
    m.lib, m._h, m.device, m.n_lidar, m.n_points, m._slot_rows = _Lib(), C.c_void_p(), 0, L, 0, {}
    return m


@pytest.mark.parametrize("leaf", [0.0, -0.5, float("nan"), float("inf"), 1e39, "x", None])
def test_voxel_map_accumulate_rejects_a_bad_leaf_before_the_call(leaf):
    with pytest.raises(ValueError):
        _model().voxel_map_accumulate(capi.PassState(), np.zeros(3, F), leaf)
    with pytest.raises(ValueError):
        plugin.PcdSaver(_model(), "/tmp", 5, leaf=leaf if leaf is not None else 0.0)


@pytest.mark.parametrize("n_tags", [0, 2, 4])
def test_voxel_map_accumulate_wants_one_tag_per_slot(n_tags):
    with pytest.raises(ValueError):
        _model().voxel_map_accumulate(capi.PassState(), np.zeros(n_tags, F), 0.5)


class _FakeModel:
    """Records which accumulate / save a PcdSaver calls."""
    def __init__(self):
        self.calls = []

    def pcd_accumulate(self, s, tag):
        self.calls.append(("dense",))
        return 100

    def voxel_map_accumulate(self, s, tag, leaf):
        self.calls.append(("voxel", leaf))
        return 7

    def pcd_save(self, path, clear):
        self.calls.append(("dense-save", os.path.basename(path), clear))

    def voxel_map_save(self, path, clear):
        self.calls.append(("voxel-save", os.path.basename(path), clear))


def test_pcd_saver_with_a_leaf_keeps_names_and_interval():
    for leaf, acc, save in ((None, ("dense",), "dense-save"), (0.2, ("voxel", float(F(0.2))), "voxel-save")):
        fm = _FakeModel()
        ps = plugin.PcdSaver(fm, "/out", 2, leaf=leaf)
        paths = [ps.after_update(None, [0.0]) for _ in range(7)]
        assert paths == [None, None, "/out/scans_1.pcd", None, None, "/out/scans_2.pcd", None]
        assert ps.finish() == "/out/result.pcd"
        assert [c for c in fm.calls if c[0] == acc[0]] == [acc] * 7
        assert [c for c in fm.calls if c[0] == save] == [(save, "scans_1.pcd", True), (save, "scans_2.pcd", True),
                                                         (save, "result.pcd", False)]
