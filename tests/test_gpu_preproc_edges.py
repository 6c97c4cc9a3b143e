"""GPU tests of the undistortion (SURVEY.md §8f N2) and the voxel grid (N3) at the motions, time ties, list edges, handle
reuse and grid edges the default synthetic inputs never reach.

Undistortion, against the CPU oracle at the bars of tests/test_gpu_preproc.py (table index, spline flag and pop points
identical; pose <= 1e-9; compensated points <= 1 float ulp and > 99.9 % bit-identical) and against the independent
scipy/numpy reference of tests/helpers.py (pose <= 1e-9, points <= 2 ulp).  Voxel grid bit-exact against the oracle."""
import ctypes as C
import time

import numpy as np
import pytest

import helpers as H
import pyoracle as po
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu

REGIMES = [(m, True, "default") for m in synth.UNDISTORT_MOTIONS] + [
    ("generic", False, "default"), ("generic", True, "empty_cov"), ("straight", True, "last_cov"), ("heading_y", True, "max"),
    ("fast", False, "max"), ("stationary", True, "max")]


def _rid(r):
    return f"{r[0]}{'-ties' if r[1] else ''}-{r[2]}"


def _lt(c):
    ok, q, p = po.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], c["end_time"])
    assert ok
    return q, p


def _device(m, c, lidar=0, want_pose=True):
    return m.undistort(lidar, c["pts"], c["beg_time"], c["extrinsic"], _lt(c), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"],
                       c["cov_pointer"], want_pose=want_pose)


def _oracle(c, want_pose=True):
    return po.undistort(c["pts"], c["beg_time"], c["extrinsic"], _lt(c), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"],
                        want_pose=want_pose)


def _check_vs_oracle(g, o, c):
    assert np.array_equal(g["ok"], o["ok"])
    assert np.array_equal(g["idx"], o["idx"]), "table index (intensity) must be identical"
    assert np.array_equal(g["pop_point"], o["pop_point"]) and len(g["pop_point"]) == min(o["n_pops"], len(c["imu_cov_t"]))
    t = o["ok"] > 0
    if t.any():
        assert np.abs(g["pose"][t] - o["pose"][t]).max() < 1e-9
        assert H.ulp_diff(g["xyz"], o["xyz"]) <= 1.0
        assert (g["xyz"] == o["xyz"]).all(axis=1).mean() > 0.999
    assert np.array_equal(g["xyz"][~t], c["pts"]["xyz"][~t])


def _check_vs_reference(g, c):
    r = H.undistort_ref(c, _lt(c))
    t = r["ok"]
    assert np.array_equal(g["ok"] > 0, t)
    assert np.array_equal(g["idx"].astype(np.int64), r["idx"])
    assert np.array_equal(g["pop_point"], r["pop_point"])
    if t.any():
        assert H.quat_close(g["pose"][t, :4], r["P"][t, :3, :3], 1e-9)[0]
        assert np.abs(g["pose"][t, 4:] - r["P"][t, :3, 3]).max() < 1e-9
    assert H.ulp_diff(g["xyz"], r["xyz"]) <= 2.0
    return r


@pytest.mark.parametrize("regime", REGIMES, ids=_rid)
def test_undistort_regimes(regime):
    motion, ties, lists = regime
    c = synth.undistort_case(3000, lidar=2, motion=motion, ties=ties, lists=lists)
    m = plugin.MeasurementModel(3)
    g = _device(m, c, lidar=2)
    m.close()
    _check_vs_oracle(g, _oracle(c), c)
    _check_vs_reference(g, c)
    t = g["ok"] > 0
    if motion == "stationary":
        assert H.ulp_diff(g["xyz"][t], c["pts"]["xyz"][t]) <= 1.0
    if motion == "straight":   # commuting turns: the heading is the b-weighted sum of the pair increments (see the CPU test)
        ct = c["ctrl_t"]
        steps = np.array(synth.STRAIGHT_YAW_STEPS)[np.arange(ct.shape[0]) % len(synth.STRAIGHT_YAW_STEPS)]
        yaw = np.concatenate([[0.0], np.cumsum(steps[:-1])])
        ts = c["pts"]["curvature"][t].astype(np.float64) / 1000.0 + c["beg_time"]
        i1 = np.searchsorted(ct, ts, side="right") - 1
        u = (ts - ct[i1]) / (ct[i1 + 1] - ct[i1])
        expect = (yaw[i1 - 1] + (5 + 3 * u - 3 * u * u + u ** 3) / 6 * steps[i1 - 1] + (1 + 3 * u + 3 * u * u - 2 * u ** 3) / 6 * steps[i1]
                  + u ** 3 / 6 * steps[i1 + 1])
        Rz = synth.q_to_R(synth.q_exp([0.1, -0.05, 0.7])).T @ np.stack([synth.q_to_R(q) for q in g["pose"][t, :4]])
        assert np.abs(np.arctan2(Rz[:, 1, 0], Rz[:, 0, 0]) - expect).max() < 1e-14


@pytest.mark.parametrize("n", [1025, 2049])
def test_undistort_scan_chunk_edges_with_saturated_pops(n):
    """Point counts just past the scan kernel's 1024-point chunks, with an IMU list whose every entry lies inside the scan
    at 3.5 kHz: the walk pops all n_cov entries (the pop table is full)."""
    c = synth.undistort_case(n, lidar=1, imu_hz=3500.0, ties=True, lists="last_cov")
    t1 = float(c["pts"]["curvature"][1]) / 1000.0 + c["beg_time"]
    c["imu_cov_t"] = c["imu_cov_t"][c["imu_cov_t"] > t1]
    c["cov_pointer"] = c["imu_cov_t"].shape[0] - 1
    assert c["cov_pointer"] > 300
    m = plugin.MeasurementModel(3)
    g = _device(m, c, lidar=1)
    m.close()
    o = _oracle(c)
    assert o["n_pops"] == c["imu_cov_t"].shape[0] == len(g["pop_point"])
    _check_vs_oracle(g, o, c)
    _check_vs_reference(g, c)


def test_handle_reuse_grow_shrink_empty():
    """One handle, sizes 131072 -> 1 -> 0 -> 60000 on one LiDAR slot and across slots, with and without the pose output:
    every result equals a fresh handle's.  An empty undistortion gives an empty part of the merged scan."""
    cases = {n: synth.undistort_case(n, lidar=0, seed=70 + k, ties=True) for k, n in enumerate((131072, 1, 0, 60000))}
    fresh = {}
    for n, c in cases.items():
        for want_pose in (True, False):
            f = plugin.MeasurementModel(3)
            fresh[n, want_pose] = (_device(f, c, 0, want_pose), f.voxel_grid(0, None, 0.5))
            f.close()
    o = _oracle(cases[60000])
    _check_vs_oracle(fresh[60000, True][0], o, cases[60000])
    m = plugin.MeasurementModel(3)
    for slot_of in ((0, 0, 0, 0), (0, 1, 2, 1), (2, 2, 0, 0)):
        for want_pose in (True, False, None):
            for (n, c), slot in zip(cases.items(), slot_of):
                wp = bool(n % 2) if want_pose is None else want_pose   # None: alternate with and without
                g = _device(m, c, slot, wp)
                ref, ref_ds = fresh[n, wp]
                for k in ("xyz", "idx", "ok", "pop_point"):
                    assert np.array_equal(g[k], ref[k]), (n, slot, wp, k)
                if wp:
                    assert np.array_equal(g["pose"], ref["pose"]), (n, slot, wp)
                assert np.array_equal(m.voxel_grid(slot, None, 0.5), ref_ds), (n, slot, wp)
    case = synth.make_case("reuse", 500, 20000, 3, 3)
    m.undistort(0, cases[0]["pts"], cases[0]["beg_time"], cases[0]["extrinsic"], _lt(cases[1]), cases[1]["ctrl_t"],
                cases[1]["ctrl_T"], cases[1]["imu_cov_t"], cases[1]["cov_pointer"])
    assert m.voxel_grid(0, None, 0.5).shape[0] == 0
    n1 = m.voxel_grid(1, None, 0.5).shape[0]
    n2 = m.voxel_grid(2, np.zeros((0, 5), np.float32), 0.5).shape[0]
    assert n1 > 0 and n2 == 0
    assert m.upload_scan_device(case.table, case.table_off, case.temporal_comp) == n1
    m.close()


# ------------------------------------------------------------------ voxel grid
def _to8(p5):
    p8 = np.zeros((p5.shape[0], 8), np.float32)
    p8[:, :4] = p5[:, :4]
    p8[:, 7] = p5[:, 4]
    return p8


def _assert_vg_equal(out, p5, leaf):
    ref, _ = po.voxel_grid(_to8(p5), leaf)
    assert out.shape[0] == ref.shape[0], (out.shape, ref.shape)
    assert np.array_equal(out[:, :4].view(np.uint32), ref[:, :4].view(np.uint32)) and np.array_equal(out[:, 4].view(np.uint32), ref[:, 7].view(np.uint32))


def _face_cloud(leaf, seed):
    """Coordinates exactly on voxel faces k*leaf (k = -40..40), one float ulp either side of them, and -0.0."""
    rng = np.random.default_rng(seed)
    f = (np.arange(-40, 41) * np.float32(leaf)).astype(np.float32)
    vals = np.concatenate([f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf)), [np.float32(-0.0)] * 20])
    n = 30000
    p = np.zeros((n, 5), np.float32)
    p[:, :3] = rng.choice(vals, size=(n, 3))
    p[:, 3] = rng.integers(0, 40, n)
    p[:, 4] = rng.uniform(0, 100, n).astype(np.float32)
    p[:50, :3] = np.float32(-0.0)
    return p


@pytest.mark.parametrize("leaf", [0.1, 0.3, 0.7, 0.5])
def test_voxel_grid_points_on_faces(leaf):
    p = _face_cloud(leaf, 3)
    m = plugin.MeasurementModel(1)
    _assert_vg_equal(m.voxel_grid(0, p, leaf), p, leaf)
    q = p.copy()
    q[:, :3] += np.float32(3.0 * leaf)   # the same faces away from the origin, minimum on a face
    q[:, :3] = q[:, :3].astype(np.float32)
    _assert_vg_equal(m.voxel_grid(0, q, leaf), q, leaf)
    m.close()


def test_voxel_grid_one_voxel_of_20k_points():
    """A single voxel holding 20k points (the per-voxel rank is quadratic in the voxel's count); the time is printed."""
    rng = np.random.default_rng(4)
    p = np.zeros((20000, 5), np.float32)
    p[:, :3] = rng.uniform(1.01, 1.49, (20000, 3))
    p[:, 3] = rng.integers(0, 30, 20000)
    p[:, 4] = rng.uniform(0, 100, 20000)
    m = plugin.MeasurementModel(1)
    m.voxel_grid(0, p, 0.5)   # warm-up
    t0 = time.perf_counter()
    out = m.voxel_grid(0, p, 0.5)
    ms = (time.perf_counter() - t0) * 1e3
    print(f"\nvoxel_grid, one voxel of 20000 points: {ms:.2f} ms for two calls (count + fetch)")
    assert out.shape[0] == 1
    _assert_vg_equal(out, p, 0.5)
    m.close()


def test_voxel_grid_non_finite_and_truncated_output():
    m = plugin.MeasurementModel(1)
    p = np.full((5000, 5), np.nan, np.float32)
    p[::3, 0] = np.inf
    assert m.voxel_grid(0, p, 0.5).shape[0] == 0
    p[1234] = (1.25, -3.5, 0.75, 7.0, 42.0)
    out = m.voxel_grid(0, p, 0.5)
    assert out.shape[0] == 1 and np.array_equal(out[0], p[1234])
    # out_cap below the voxel count: the first out_cap centroids are delivered, *n_out is still the full count
    q = _face_cloud(0.3, 8)
    ref = m.voxel_grid(0, q, 0.3)
    assert ref.shape[0] > 100
    out = np.full((40, 5), -7.0, np.float32)
    big = np.full((ref.shape[0] + 8, 5), -7.0, np.float32)
    n_out = C.c_uint32(0)
    for buf, cap in ((out, 37), (big, ref.shape[0] + 8)):
        assert m.lib.malio_voxel_grid(m._h, 0, capi.ptr(q), q.shape[0], C.c_float(0.3), capi.ptr(buf), cap, C.byref(n_out)) == capi.OK
        assert n_out.value == ref.shape[0]
    assert np.array_equal(out[:37], ref[:37]) and (out[37:] == -7.0).all()
    assert np.array_equal(big[: ref.shape[0]], ref) and (big[ref.shape[0]:] == -7.0).all()
    m.close()


def test_voxel_grid_rejects_grids_it_cannot_index():
    """More than 2^28 cells, more than 2^24 voxels along one axis (PCL's float index would round up to the axis' size) and
    voxel indices outside int are MALIO_ERR_CAPACITY; the handle stays usable."""
    m = plugin.MeasurementModel(1)
    clouds = [
        ([[0.0, 0.0, 0.0], [100.0, 100.0, 100.0]], 0.01),        # 1e12 cells
        ([[1.0, 0.0, 0.0], [float(1 << 25), 0.0, 0.0]], 1.0),   # dx = 2^25, dy = dz = 1: 2^25 cells
        ([[0.0, 1.0, 0.0], [0.0, float(1 << 26), 0.0]], 2.0),   # dy = 2^25 + 1
        ([[1e10, 0.0, 0.0]], 1.0),                              # one point, index beyond int
        ([[0.0, 0.0, -3e38], [0.0, 0.0, 1.0]], 0.1),            # x / leaf overflows to -inf
    ]
    for xyz, leaf in clouds:
        p = np.zeros((len(xyz), 5), np.float32)
        p[:, :3] = xyz
        with pytest.raises(capi.MalioError) as e:
            m.voxel_grid(0, p, leaf)
        assert e.value.status == capi.ERR_CAPACITY, (xyz, leaf)
    # exactly 2^24 voxels along x is still indexed
    p = np.zeros((3, 5), np.float32)
    p[:, 0] = (0.0, 5.0, float((1 << 24) - 1))
    _assert_vg_equal(m.voxel_grid(0, p, 1.0), p, 1.0)
    q = _face_cloud(0.3, 5)
    _assert_vg_equal(m.voxel_grid(0, q, 0.3), q, 0.3)
    m.close()
