"""publish_frame_world and the saved map on the device (laserMapping.cpp:448-489, :1083-1091), against the host restatement of
RGBpointBodyToWorld (tests/world_ref.py, itself pinned to scipy and to the oracle's map_incremental in test_world_cpu.py):
  dense         the device-resident undistorted clouds of slots 0..L-1 (feats_undistort), intensity = slot_tag[slot]
  down-sampled  the scan after the update in caller order, intensity = the last pass's normal_y
  accumulate    pcl_wait_save kept on the device across scans and written as binary PCD
The dense cloud is compared through the device's OWN undistortion output: device and oracle undistortion agree only to 1 ulp
(device sin/cos), the registration itself must be bit-exact."""
import ctypes as C
import os

import numpy as np
import pytest

import helpers as H
import world_ref as W
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu


def _undistort(m, slot, n, seed, partial=False):
    """malio_undistort of a synth.undistort_case on LiDAR slot `slot`; partial: the spline ends inside the scan, so some
    points keep their raw coordinates.  Returns the device's undistorted xyz (the cloud the dense source registers)."""
    c = synth.undistort_case(n, lidar=slot, seed=seed)
    if partial:
        keep = slice(2, -6)
        c = dict(c, ctrl_t=c["ctrl_t"][keep], ctrl_T=c["ctrl_T"][keep])
    ok, q, p = plugin.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], min(c["end_time"], c["ctrl_t"][-3]))
    assert ok
    g = m.undistort(slot, c["pts"], c["beg_time"], c["extrinsic"], (q, p), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
    if partial and n > 10:
        assert 0 < g["ok"].sum() < n - 1
    return g["xyz"]


def _model_with_tcomp(L, tc):
    """A handle whose last uploaded scan carries the temporal compensation tc (the dense source reads it from there)."""
    case = synth.make_case("world-tc", 200, 5000, L, 3)
    m = plugin.MeasurementModel(L, params=case.params)
    m.upload_scan(case.pts, case.table, case.table_off, tc)
    return m


def _dense_ref(s, tc, clouds, tags):
    return np.concatenate([W.register_world(s, tc, xyz, l, tags[l]) for l, xyz in enumerate(clouds)]).reshape(-1, 4)


DENSE_SIZES = {1: [7001], 2: [0, 9000], 3: [12000, 0, 5003]}


@pytest.mark.parametrize("L", [1, 2, 3])
def test_dense_registration_bit_exact(L):
    s, tc = W.far_state(L, seed=20 + L)
    m = _model_with_tcomp(L, tc)
    clouds = [_undistort(m, l, n, seed=70 + l, partial=(l == L - 1)) for l, n in enumerate(DENSE_SIZES[L])]
    tags = np.array([2.5, 0.5, 1.5][:L], np.float32)      # lidar_buffer positions need not be the slot numbers
    out = m.publish_frame_world(s, True, tags)
    ref = _dense_ref(s, tc, clouds, tags)
    assert out.shape == (sum(DENSE_SIZES[L]), 4)
    assert out.tobytes() == ref.tobytes()
    at = 0
    for l, xyz in enumerate(clouds):                      # slot order, each slot in its buffer order
        assert np.all(out[at:at + len(xyz), 3] == tags[l])
        at += len(xyz)
    # a pass-through check of the far-field arithmetic: within 1 ulp of the scipy restatement
    sp = np.concatenate([W.register_world_scipy(s, tc, xyz, l) for l, xyz in enumerate(clouds)]).reshape(-1, 3)
    assert H.ulp_diff(out[:, :3], sp.astype(np.float32)) <= 1.0
    m.close()


@pytest.fixture(scope="module")
def c2():
    case = synth.case_C2()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    return case, snap


@pytest.mark.parametrize("sort_queries", [True, False])
def test_downsampled_registration_after_update(c2, sort_queries):
    case, snap = c2
    m = H.make_model(case, snap, sort_queries=sort_queries)
    x, P = case.x_prop.copy(), case.P_prop.copy()
    m.update_iterated_dyn_share_modified(x, P, case.max_iter)
    out = m.publish_frame_world(x, False)
    a = m.aux(nn_idx=False, nn_sqdist=False, selected=False, world=False)
    ref = W.register_world(x, case.temporal_comp, case.pts["xyz"], case.pts["lidar"], a["normal_y"])
    assert out.shape == (case.pts.shape[0], 4)
    assert out[:, :3].tobytes() == ref[:, :3].tobytes()
    assert out[:, 3].tobytes() == a["normal_y"].tobytes()
    cls, w = m.map_incremental(x, 0.5, True)
    keep = cls != capi.MAP_SKIP
    assert keep.sum() > 0.5 * len(cls)
    assert out[keep, :3].tobytes() == w[keep].tobytes()
    m.close()


def test_accumulate_across_scans_and_save(tmp_path):
    """8 scans of 30-90k points, enough for the accumulated cloud (first 65536 points, then at least doubling) to be regrown
    with its content copied at least twice.  Every saved file must be the concatenation of the per-scan
    publish_frame_world(dense) clouds, bit for bit."""
    L = 3
    m = None
    per_scan = []
    total = 0
    cap, regrown = 0, 0                                   # the growth rule of malio_world_accumulate
    rng = np.random.default_rng(5)
    for k in range(8):
        s, tc = W.far_state(L, seed=100 + k)
        if m is None:
            m = _model_with_tcomp(L, tc)
        else:
            case = synth.make_case("world-tc", 200, 5000, L, 3)
            m.upload_scan(case.pts, case.table, case.table_off, tc)
        sizes = rng.integers(10000, 30000, L)
        clouds = [_undistort(m, l, int(sizes[l]), seed=300 + 7 * k + l, partial=(k % 3 == 1 and l == 0)) for l in range(L)]
        tags = np.array([(L - 1 - l + k) % L for l in range(L)], np.float32)
        out = m.publish_frame_world(s, True, tags)
        assert out.tobytes() == _dense_ref(s, tc, clouds, tags).tobytes()
        per_scan.append(out)
        n_total = m.pcd_accumulate(s, tags)
        if total + out.shape[0] > cap:
            regrown += total > 0
            cap = max(total + out.shape[0], 2 * cap, 65536)
        total += out.shape[0]
        assert n_total == total
        if k == 5:
            p1 = str(tmp_path / "scans_1.pcd")
            m.pcd_save(p1, clear=False)
            _, rec = W.read_pcd(p1)
            assert W.xyzi(rec).tobytes() == np.concatenate(per_scan).tobytes()
            for f in ("normal_x", "normal_y", "normal_z", "curvature"):
                assert rec[f].view(np.uint32).max() == 0
    assert regrown >= 2
    p2 = str(tmp_path / "result.pcd")
    m.pcd_save(p2, clear=True)                            # everything since the first scan, then empty
    _, rec = W.read_pcd(p2)
    assert rec.shape[0] == total and W.xyzi(rec).tobytes() == np.concatenate(per_scan).tobytes()
    for l in range(L):                                    # empty slots: the cloud stays empty, the count reads 0
        _undistort(m, l, 0, seed=1)
    assert m.pcd_accumulate(W.far_state(L, 1)[0], np.zeros(L, np.float32)) == 0
    p3 = tmp_path / "again.pcd"
    assert m.lib.malio_world_save_pcd(m._h, os.fsencode(str(p3)), 0) == capi.ERR_STATE
    assert not p3.exists()
    m.close()


def test_no_side_effects_on_other_outputs():
    """download_aux, map_incremental, voxel_grid(NULL) and upload_scan_device (and the pass that follows it) give the same
    results before and after register / accumulate on the same handle."""
    case = synth.make_case("world-fx", 20000, 200000, 3, 3)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    m = H.make_model(case, snap)
    for l in range(3):
        _undistort(m, l, 15000 + 4000 * l, seed=90 + l)
    vg0 = [m.voxel_grid(l, None, 0.5) for l in range(3)]
    n0 = m.upload_scan_device(case.table, case.table_off, case.temporal_comp)
    ok0, HTH0, HTh0, _ = m.h_share_model(case.x_prop, True)
    m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    x, P = case.x_prop.copy(), case.P_prop.copy()
    m.update_iterated_dyn_share_modified(x, P, case.max_iter)
    aux0 = m.aux()
    mi0 = m.map_incremental(x, 0.5, True)
    tags = np.array([1.0, 2.0, 0.0], np.float32)

    def touch():
        m.publish_frame_world(x, False)
        m.publish_frame_world(x, True, tags)
        m.pcd_accumulate(x, tags)

    touch()
    aux1 = m.aux()
    mi1 = m.map_incremental(x, 0.5, True)
    for k in aux0:
        assert np.array_equal(aux0[k], aux1[k]), k
    assert np.array_equal(mi0[0], mi1[0]) and mi0[1].tobytes() == mi1[1].tobytes()
    touch()
    vg1 = [m.voxel_grid(l, None, 0.5) for l in range(3)]
    for a, b in zip(vg0, vg1):
        assert a.tobytes() == b.tobytes()
    touch()
    n1 = m.upload_scan_device(case.table, case.table_off, case.temporal_comp)
    ok1, HTH1, HTh1, _ = m.h_share_model(case.x_prop, True)
    assert n1 == n0 and ok1 == ok0 and np.array_equal(HTH0, HTH1) and np.array_equal(HTh0, HTh1)
    m.close()


def test_argument_and_state_errors(tmp_path):
    L = 3
    s, tc = W.far_state(L, seed=3)
    m = _model_with_tcomp(L, tc)
    lib, h = m.lib, m._h
    ps = s.pass_state()
    tags = np.array([0.0, 1.0, 2.0], np.float32)
    n = C.c_uint32(7)
    # dense before every slot 0..L-1 has been undistorted
    a = _undistort(m, 0, 3000, seed=1)
    c = _undistort(m, 2, 2000, seed=2)
    assert lib.malio_world_register(h, C.byref(ps), capi.WORLD_DENSE, capi.ptr(tags), None, 0, C.byref(n)) == capi.ERR_STATE
    assert lib.malio_world_accumulate(h, C.byref(ps), capi.ptr(tags), None) == capi.ERR_STATE
    _undistort(m, 1, 0, seed=3)                           # an empty slot is a valid one
    assert lib.malio_world_register(h, C.byref(ps), capi.WORLD_DENSE, capi.ptr(tags), None, 0, C.byref(n)) == capi.OK
    assert n.value == a.shape[0] + c.shape[0]
    # down-sampled before any pass on the current scan
    assert lib.malio_world_register(h, C.byref(ps), capi.WORLD_DOWNSAMPLED, None, None, 0, C.byref(n)) == capi.ERR_STATE
    # bad source, missing slot_tag, missing outputs
    for src in (-1, 2):
        assert lib.malio_world_register(h, C.byref(ps), src, capi.ptr(tags), None, 0, C.byref(n)) == capi.ERR_INVALID_ARG
    assert lib.malio_world_register(h, C.byref(ps), capi.WORLD_DENSE, None, None, 0, C.byref(n)) == capi.ERR_INVALID_ARG
    assert lib.malio_world_register(h, C.byref(ps), capi.WORLD_DENSE, capi.ptr(tags), None, 5, C.byref(n)) == capi.ERR_INVALID_ARG
    assert lib.malio_world_register(h, None, capi.WORLD_DENSE, capi.ptr(tags), None, 0, C.byref(n)) == capi.ERR_INVALID_ARG
    assert lib.malio_world_accumulate(h, C.byref(ps), None, None) == capi.ERR_INVALID_ARG
    # cap below the count: cap points written, the rest of the buffer untouched, n_out = the full count
    full = m.publish_frame_world(s, True, tags)
    cap = 1234
    buf = np.full((cap + 16, 4), -7.0, np.float32)
    assert lib.malio_world_register(h, C.byref(ps), capi.WORLD_DENSE, capi.ptr(tags), capi.ptr(buf), cap, C.byref(n)) == capi.OK
    assert n.value == full.shape[0] and buf[:cap].tobytes() == full[:cap].tobytes() and np.all(buf[cap:] == -7.0)
    # save: empty cloud, NULL path, unopenable path; none leaves a file
    p = tmp_path / "x.pcd"
    assert lib.malio_world_save_pcd(h, os.fsencode(str(p)), 1) == capi.ERR_STATE
    assert lib.malio_world_save_pcd(h, None, 0) == capi.ERR_INVALID_ARG
    assert m.pcd_accumulate(s, tags) == full.shape[0]
    bad = tmp_path / "missing_dir" / "x.pcd"
    assert lib.malio_world_save_pcd(h, os.fsencode(str(bad)), 1) == capi.ERR_INVALID_ARG
    assert not bad.exists() and os.listdir(tmp_path) == []
    m.pcd_save(str(p), clear=True)                        # the failed save did not clear
    _, rec = W.read_pcd(str(p))
    assert W.xyzi(rec).tobytes() == full.tobytes()
    m.close()
