"""The saved map as a voxel map on the device (malio_world_voxel_*), bit for bit:
  - against malio_voxel_grid on the concatenation of the same scans' dense clouds (curvature padded as 0) wherever that dense
    grid can index the cloud, and against the float32 restatement (tests/world_voxel_ref.py) everywhere, including clouds the
    dense grid refuses (an extent over 2^28 cells, coordinates at +-1e5 m, a 2 km drive at a 0.1 m leaf);
  - L = 1, 2, 3 with empty slots, one voxel hit by 20k points of one scan and by points of 100 scans, faces +-1 ulp, non-finite
    points, the leaf mismatch, the clear, two runs giving the same bytes, the download around a save, the PCD bytes;
  - the device-memory contract of the download (stream order, pointer classes, the size protocol), the dense accumulation
    interleaved on the same handle, and a 300-scan loop over one area whose voxel map stops growing.
Planted clouds go through malio_undistort with control points that end before the scan, so every point keeps its raw
coordinates, and an identity state: the world points are the planted floats."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import world_ref as W
import world_voxel_ref as V
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
Q_ID = np.array([1.0, 0.0, 0.0, 0.0])


def _identity_state(L, pos=(0.0, 0.0, 0.0)):
    return synth.make_state(pos, Q_ID, [Q_ID] * L, [np.zeros(3)] * L)


def _plant(m, slot, xyz):
    """malio_undistort of raw points whose times lie past the spline: the slot's cloud is xyz, bit for bit."""
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    ctrl_t = np.array([-10.0, -9.0, -8.0, -7.0])
    ctrl_T = np.tile(np.eye(4), (4, 1, 1))
    m.undistort(slot, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), ctrl_t, ctrl_T, np.zeros(0), -1)


def _real(m, slot, n, seed):
    """A synthetic undistorted scan (as tests/test_gpu_world.py makes them)."""
    c = synth.undistort_case(n, lidar=slot, seed=seed)
    ok, q, p = plugin.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], min(c["end_time"], c["ctrl_t"][-3]))
    assert ok
    m.undistort(slot, c["pts"], c["beg_time"], c["extrinsic"], (q, p), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])


def _model_with_tcomp(L, tc):
    case = synth.make_case("world-vox", 200, 5000, L, 3)
    m = plugin.MeasurementModel(L, params=case.params)
    m.upload_scan(case.pts, case.table, case.table_off, tc)
    return m


def _download(m):
    return m.voxel_map_tensor().cpu().numpy()


def _pad5(clouds):
    cat = np.concatenate(clouds).reshape(-1, 4)
    p5 = np.zeros((cat.shape[0], 5), F)
    p5[:, :4] = cat
    return p5


def _grid(m, clouds, leaf):
    """malio_voxel_grid of the concatenated dense clouds, or None where it refuses the grid (MALIO_ERR_CAPACITY)."""
    try:
        return m.voxel_grid(0, _pad5(clouds), leaf)[:, :4]
    except capi.MalioError as e:
        assert e.status == capi.ERR_CAPACITY
        return None


def _same(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.shape, b.shape)
    assert a.tobytes() == b.tobytes(), what


SIZES = {1: [[7001], [9000], [0], [12000]], 2: [[0, 9000], [8000, 5000], [3000, 0], [0, 0]],
         3: [[12000, 0, 5003], [4000, 6000, 7000], [0, 0, 9000], [5000, 5000, 5000]]}


@pytest.mark.parametrize("L", [1, 2, 3])
def test_real_scans_equal_voxel_grid_and_restatement(L, tmp_path):
    """Four registered scans per L, empty slots among them, dense accumulation interleaved on the same handle."""
    leaf = 0.5
    ref = V.VoxelMapRef()
    dense = []
    m = None
    for k, sizes in enumerate(SIZES[L]):
        s, tc = W.far_state(L, seed=40 + 3 * k + L)
        if m is None:
            m = _model_with_tcomp(L, tc)
        else:
            case = synth.make_case("world-vox", 200, 5000, L, 3)
            m.upload_scan(case.pts, case.table, case.table_off, tc)
        for l, n in enumerate(sizes):
            _real(m, l, n, seed=500 + 10 * k + l)
        tags = np.array([(l + k) % 3 for l in range(L)], F)
        d = m.publish_frame_world(s, True, tags)
        dense.append(d)
        assert m.pcd_accumulate(s, tags) == sum(x.shape[0] for x in dense)
        n_vox = m.voxel_map_accumulate(s, tags, leaf)
        assert n_vox == ref.accumulate_fast(d, leaf)
        got = _download(m)
        _same(got, ref.centroids(), ("restatement", k))
        g = _grid(m, dense, leaf)
        assert g is not None
        _same(got, g, ("voxel_grid", k))
    # the dense cloud is still the concatenation, and the voxel file is the PCD writer's bytes of the download
    p = tmp_path / "dense.pcd"
    m.pcd_save(str(p), clear=False)
    _, rec = W.read_pcd(str(p))
    _same(W.xyzi(rec), np.concatenate(dense), "dense cloud")
    pv, pw = tmp_path / "vox.pcd", tmp_path / "ref.pcd"
    m.voxel_map_save(str(pv), clear=False)
    plugin.write_pcd_binary(str(pw), got)
    assert pv.read_bytes() == pw.read_bytes()
    m.close()


def _faces(leaf, ks, rng):
    il = F(1.0) / F(leaf)
    vals = []
    for k in ks:
        for v in (F(k) * F(leaf), F(k) / il):
            vals += [v, np.nextafter(v, F(np.inf)), np.nextafter(v, F(-np.inf))]
    vals = np.array(vals, F)
    out = []
    for ax in range(3):
        b = rng.uniform(-2, 2, (vals.shape[0], 3)).astype(F)
        b[:, ax] = vals
        out.append(b)
    return np.concatenate(out)


@pytest.mark.parametrize("leaf", [0.1, 0.3])
def test_planted_faces_and_non_finite_points(leaf):
    L = 2
    m = plugin.MeasurementModel(L)
    s = _identity_state(L)
    rng = np.random.default_rng(int(leaf * 10))
    ref = V.VoxelMapRef()
    dense = []
    for k in range(3):
        a = _faces(leaf, [-5, -1, 0, 1, 7], rng)
        b = rng.normal(0, 1.0, (4000, 3)).astype(F)
        b[::97] = np.nan
        b[5::211, 1] = np.inf
        _plant(m, 0, a)
        _plant(m, 1, b)
        tags = np.array([1.0, 2.0], F)
        d = m.publish_frame_world(s, True, tags)
        fin = np.isfinite(b).all(axis=1)                 # (an identity rotation turns inf into NaN: still skipped)
        assert np.array_equal(d[: a.shape[0], :3], a) and np.array_equal(d[a.shape[0]:, :3][fin], b[fin])
        assert not np.isfinite(d[a.shape[0]:, :3][~fin]).all(axis=1).any()
        dense.append(d)
        assert m.voxel_map_accumulate(s, tags, leaf) == ref.accumulate_fast(d, leaf)
    got = _download(m)
    _same(got, ref.centroids(), "restatement")
    _same(got, _grid(m, dense, leaf), "voxel_grid")
    m.close()


@pytest.mark.parametrize("where", ["far", "drive", "cells"])
def test_clouds_the_dense_grid_refuses(where):
    """+-1e5 m, a 2 km drive at 0.1 m (moving the state), and an extent over 2^28 cells: restatement only."""
    L = 1
    m = plugin.MeasurementModel(L)
    ref = V.VoxelMapRef()
    rng = np.random.default_rng(7)
    dense = []
    leaf = 0.1 if where != "cells" else 0.05
    raw = np.concatenate([rng.uniform(-40, 40, (20000, 2)), rng.uniform(-2, 3, (20000, 1))], axis=1).astype(F)
    scans = 40 if where == "drive" else 4
    for k in range(scans):
        if where == "far":
            pts = (raw + F(1e5) * F(1 if k % 2 else -1)).astype(F)
            pts[::3, 2] = -pts[::3, 2]
            s = _identity_state(L)
        elif where == "drive":
            pts = raw
            s = _identity_state(L, pos=(50.0 * k, 3.0 * np.sin(k / 5.0), 0.02 * k))
        else:
            pts = (raw * F(1.5 + k)).astype(F)
            s = _identity_state(L)
        _plant(m, 0, pts)
        d = m.publish_frame_world(s, True, np.array([0.5], F))
        dense.append(d)
        assert m.voxel_map_accumulate(s, np.array([0.5], F), leaf) == ref.accumulate_fast(d, leaf)
    _same(_download(m), ref.centroids(), "restatement")
    assert _grid(m, dense, leaf) is None
    if where == "drive":
        assert np.ptp(np.concatenate(dense)[:, 0]) > 2000.0
    m.close()


def test_one_voxel_from_one_scan_and_from_100_scans():
    L = 1
    m = plugin.MeasurementModel(L)
    s = _identity_state(L)
    rng = np.random.default_rng(11)
    ref = V.VoxelMapRef()
    dense = []
    for k in range(101):
        n = 20000 if k == 0 else 50
        pts = rng.uniform(2.0, 2.999, (n, 3)).astype(F)
        _plant(m, 0, pts)
        tag = np.array([F(0.1) * (k % 7)], F)
        d = m.publish_frame_world(s, True, tag)
        dense.append(d)
        assert m.voxel_map_accumulate(s, tag, 1.0) == ref.accumulate_fast(d, 1.0) == 1
        if k in (0, 1, 100):
            got = _download(m)
            _same(got, ref.centroids(), ("restatement", k))
            _same(got, _grid(m, dense, 1.0), ("voxel_grid", k))
    assert ref.cnt[(2, 2, 2)] == 25000
    m.close()


def test_leaf_capacity_clear_and_state_errors(tmp_path):
    L = 2
    m = plugin.MeasurementModel(L)
    lib, h = m.lib, m._h
    s = _identity_state(L)
    ps = s.pass_state()
    tags = np.array([0.0, 1.0], F)
    n = C.c_uint64(0)
    _plant(m, 0, np.random.default_rng(1).normal(0, 3, (3000, 3)))
    assert lib.malio_world_voxel_accumulate(h, C.byref(ps), capi.ptr(tags), 0.5, C.byref(n)) == capi.ERR_STATE   # slot 1
    _plant(m, 1, np.zeros((0, 3), F))                                                                            # empty slot
    assert lib.malio_world_voxel_accumulate(h, C.byref(ps), None, 0.5, C.byref(n)) == capi.ERR_INVALID_ARG
    for bad in (0.0, -0.5, float("nan"), float("inf")):
        assert lib.malio_world_voxel_accumulate(h, C.byref(ps), capi.ptr(tags), bad, C.byref(n)) == capi.ERR_INVALID_ARG
    p = tmp_path / "empty.pcd"
    assert lib.malio_world_voxel_save_pcd(h, os.fsencode(str(p)), 0) == capi.ERR_STATE and not p.exists()
    n0 = m.voxel_map_accumulate(s, tags, 0.5)
    before = _download(m)
    assert before.shape[0] == n0 > 0
    assert lib.malio_world_voxel_accumulate(h, C.byref(ps), capi.ptr(tags), 0.25, C.byref(n)) == capi.ERR_INVALID_ARG
    # a point whose index falls outside int: refused, the map unchanged, the good points of that scan not folded either
    far = np.random.default_rng(2).normal(0, 3, (5000, 3)).astype(F)
    far[4321] = [0.0, 2.0e9, 0.0]
    _plant(m, 1, far)
    assert lib.malio_world_voxel_accumulate(h, C.byref(ps), capi.ptr(tags), 0.5, C.byref(n)) == capi.ERR_CAPACITY
    _same(_download(m), before, "after the refusal")
    assert m.voxel_map_info()["n_voxels"] == n0
    # save without clear keeps the map; the file equals the writer's bytes of the download; clear releases the leaf
    p1, p2 = tmp_path / "a.pcd", tmp_path / "b.pcd"
    m.voxel_map_save(str(p1), clear=False)
    _same(_download(m), before, "after a save without clear")
    plugin.write_pcd_binary(str(p2), before)
    assert p1.read_bytes() == p2.read_bytes()
    bad = tmp_path / "missing_dir" / "x.pcd"
    assert lib.malio_world_voxel_save_pcd(h, os.fsencode(str(bad)), 1) == capi.ERR_INVALID_ARG and not bad.exists()
    _same(_download(m), before, "a failed save does not clear")
    m.voxel_map_save(str(p1), clear=True)
    assert m.voxel_map_info()["n_voxels"] == 0 and _download(m).shape == (0, 4)
    _plant(m, 1, np.zeros((0, 3), F))
    ref = V.VoxelMapRef()
    d = m.publish_frame_world(s, True, tags)
    assert m.voxel_map_accumulate(s, tags, 0.25) == ref.accumulate_fast(d, 0.25)   # a new leaf after the clear
    _same(_download(m), ref.centroids(), "after the clear")
    m.close()


def _run(seed):
    L = 3
    s, tc = W.far_state(L, seed=seed)
    m = _model_with_tcomp(L, tc)
    out = []
    for k in range(3):
        for l in range(L):
            _real(m, l, 6000 + 1000 * l, seed=seed + 10 * k + l)
        m.voxel_map_accumulate(s, np.array([0.0, 1.0, 2.0], F), 0.3)
        out.append(_download(m))
    m.close()
    return out


def test_two_runs_give_identical_bytes():
    a, b = _run(900), _run(900)
    for x, y in zip(a, b):
        _same(x, y, "runs")


def test_download_is_ordered_on_the_caller_stream_and_checks_its_pointers():
    L = 1
    m = plugin.MeasurementModel(L)
    lib, h = m.lib, m._h
    s = _identity_state(L)
    _plant(m, 0, np.random.default_rng(3).normal(0, 5, (60000, 3)))
    n = m.voxel_map_accumulate(s, np.array([1.0], F), 0.2)
    ref = _download(m)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    k = C.c_uint64(0)
    with torch.cuda.stream(side):
        buf = torch.empty((n, 4), device="cuda")
        torch.cuda._sleep(200_000_000)
        buf.fill_(-7.0)                                    # behind the sleep: the download must come after it
        assert lib.malio_world_voxel_download_device(h, buf.data_ptr(), n, C.byref(k), side.cuda_stream) == capi.OK
        total = buf.double().sum()                         # right behind the call, on the same stream
    side.synchronize()
    assert k.value == n
    _same(buf.cpu().numpy(), ref, "side stream")
    np.testing.assert_allclose(float(total), ref.astype(np.float64).sum(), rtol=1e-9)
    # size protocol: NULL with cap 0 asks, a short cap writes cap rows and leaves the rest
    st = torch.cuda.current_stream().cuda_stream
    assert lib.malio_world_voxel_download_device(h, None, 0, C.byref(k), st) == capi.OK and k.value == n
    assert lib.malio_world_voxel_download_device(h, None, 5, C.byref(k), st) == capi.ERR_INVALID_ARG
    assert lib.malio_world_voxel_download_device(h, buf.data_ptr(), n, None, st) == capi.ERR_INVALID_ARG
    part = torch.full((n, 4), -3.0, device="cuda")
    cap = n // 3
    assert lib.malio_world_voxel_download_device(h, part.data_ptr(), cap, C.byref(k), st) == capi.OK and k.value == n
    got = part.cpu().numpy()
    _same(got[:cap], ref[:cap], "cap rows")
    assert np.all(got[cap:] == -3.0)
    # pointer classes: refused before anything is enqueued
    hp = np.zeros(n * 4, F)
    pin = torch.empty(n * 4).pin_memory()
    bad = {"host": hp.ctypes.data, "pinned": pin.data_ptr(), "misaligned 4": buf.data_ptr() + 4,
           "misaligned 8": buf.data_ptr() + 8, "misaligned 12": buf.data_ptr() + 12, "misaligned 2": buf.data_ptr() + 2}
    if torch.cuda.device_count() > 1:
        other = torch.empty(n * 4, device="cuda:1")
        bad["other device"] = other.data_ptr()
    c0 = m.counters()
    for what, p in bad.items():
        assert lib.malio_world_voxel_download_device(h, p, n, C.byref(k), st) == capi.ERR_INVALID_ARG, what
    c1 = m.counters()
    assert c1.kernel_launches == c0.kernel_launches
    _same(_download(m), ref, "after the refusals")
    m.close()


def test_300_scans_over_one_area_stay_bounded(tmp_path):
    """The voxel map of a loop over the same area stops growing, in voxels, capacity and device bytes, while the dense cloud
    keeps growing; a download holds an entry-sized sort area, which the next save releases; the result still equals the
    restatement."""
    L = 1
    m = plugin.MeasurementModel(L)
    rng = np.random.default_rng(13)
    raw = np.concatenate([rng.uniform(-30, 30, (10000, 2)), rng.uniform(-1, 2, (10000, 1))], axis=1).astype(F)
    _plant(m, 0, raw)
    ref = V.VoxelMapRef()
    tag = np.array([1.0], F)
    hist = []
    for k in range(300):
        s = _identity_state(L, pos=(2.0 * (k % 10), 1.0 * (k % 3), 0.0))
        d = m.publish_frame_world(s, True, tag)
        n_dense = m.pcd_accumulate(s, tag)
        assert m.voxel_map_accumulate(s, tag, 0.2) == ref.accumulate_fast(d, 0.2)
        hist.append((m.voxel_map_info(), n_dense))
        if k % 50 == 49:                                  # a download and a save inside the loop
            before = hist[-1][0]["device_bytes"]
            got = _download(m)
            held = m.voxel_map_info()["device_bytes"]
            assert held > before                          # 32 B per voxel of sort area while the download's result is used
            p = tmp_path / f"scans_{k}.pcd"
            m.voxel_map_save(str(p), clear=False)
            after = m.voxel_map_info()["device_bytes"]
            assert after < before                         # the save released the sort area and CUB's storage
            _, rec = W.read_pcd(str(p))
            _same(W.xyzi(rec), got, ("save", k))
            p.unlink()
    vox = [i["n_voxels"] for i, _ in hist]
    cap = [i["capacity"] for i, _ in hist]
    byt = [i["device_bytes"] for i, _ in hist]
    assert vox[30] == vox[-1] and cap[30] == cap[-1] and byt[30] == byt[-1]
    assert [nd for _, nd in hist] == [10000 * (k + 1) for k in range(300)]
    assert cap[-1] < 2 * (vox[-1] + 10000) and byt[-1] < hist[-1][1] * 16
    _same(_download(m), ref.centroids(), "restatement")
    m.close()
