"""malio_scan_uncertainty: the scan's pose-uncertainty lists, temporal compensation and pose_unc table built on the device from
its undistortion (IMU_Processing.hpp:474-523, laserMapping.cpp:1028-1048).
  - bit for bit: the host malio_compound_* fed the pop poses malio_undistort reports give the same bytes (shared code,
    -fmad=false), and the per-slot undistort outputs are those of a handle that undistorted that slot alone;
  - against the numpy reference (tests/scan_unc_ref.py): T within 1e-9, covariance within 1e-9 of the entry's largest element,
    in every motion regime, with time ties, with the list layouts, for slots of 0 and 1 pops and an unreachable pop point;
  - end to end: raw clouds -> undistort -> scan_uncertainty -> voxel grid -> upload_scan_device -> IESKF update equals the same
    scan uploaded from the host with the numpy-built table;
  - every error code, with no kernel launched."""
import ctypes as C

import numpy as np
import pytest

import helpers as H
import np_oracle as npo
import scan_unc_ref as R
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
BAR = 1e-9


def _undistort_all(m, slots):
    return [m.undistort(l, c["pts"], c["beg_time"], c["extrinsic"], c["lt"], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"],
                        want_pose=True) for l, c in enumerate(slots)]


def _device(slots, imu_cov, ext, unc):
    m = plugin.MeasurementModel(len(slots))
    g = _undistort_all(m, slots)
    r = m.scan_uncertainty(imu_cov, R.to_capi(ext), unc, want_lists=True)
    return m, g, r


def _host_compound(slots, g, imu_cov, ext_c, unc):
    """The same build through the host C-ABI, fed the pop poses malio_undistort returned."""
    lib = capi.load()
    L = len(slots)
    init = lambda t, q, cov: _pose_initial(lib, t, q, cov)
    ltl = [init(c["lt"][1], c["lt"][0], unc if l == 0 else imu_cov[c["cov_pointer"]]) for l, c in enumerate(slots)]
    lists = []
    for l, c in enumerate(slots):
        lst = np.zeros(len(g[l]["pop_point"]), capi.POSE)
        for k, i in enumerate(g[l]["pop_point"]):
            q, t = (g[l]["pose"][i, :4], g[l]["pose"][i, 4:]) if g[l]["ok"][i] else (np.array([1.0, 0, 0, 0]), np.zeros(3))
            pt = init(t, q, imu_cov[c["cov_pointer"] - k])
            pc = lst[k:k + 1]
            e = ext_c[l:l + 1]
            lib.malio_compound_pose_with_cov(pt.ctypes.data, pt["cov"].ctypes.data, e.ctypes.data, e["cov"].ctypes.data, pc.ctypes.data,
                                             pc["cov"].ctypes.data)
            for first in (ltl[l], e):
                lib.malio_compound_inv_pose_with_cov(first.ctypes.data, first["cov"].ctypes.data, pc.ctypes.data, pc["cov"].ctypes.data,
                                                     pc.ctypes.data, pc["cov"].ctypes.data)
        lists.append(lst)
    tc = np.zeros(max(L - 1, 0), capi.POSE)
    for l in range(1, L):
        o = tc[l - 1:l]
        lib.malio_compound_inv_pose_with_cov(ltl[0].ctypes.data, ltl[0]["cov"].ctypes.data, ltl[l].ctypes.data, ltl[l]["cov"].ctypes.data,
                                             o.ctypes.data, o["cov"].ctypes.data)
    table, off = plugin.build_pose_unc(ext_c, tc if L > 1 else None, lists)
    return lists, tc, table, off


def _pose_initial(lib, t, q, cov):
    p = np.zeros(1, capi.POSE)
    lib.malio_pose_initial(p.ctypes.data, capi.ptr(np.ascontiguousarray(t, np.float64)), capi.ptr(np.ascontiguousarray(q, np.float64)),
                           capi.ptr(np.ascontiguousarray(cov, np.float64).reshape(36)))
    return p


@pytest.mark.parametrize("L,motion", [(1, "generic"), (2, "fast"), (3, "generic"), (3, "heading_y")])
def test_bit_identical_to_host_compounding(L, motion):
    slots, imu_cov, ext, unc = R.make_scan(L, n=[30000, 20000, 25000][:L], seed=30 + L, motion=motion)
    m, g, r = _device(slots, imu_cov, ext, unc)
    lists, tc, table, off = _host_compound(slots, g, imu_cov, R.to_capi(ext), unc)
    assert [len(a) for a in r["lidar_unc"]] == [len(a) for a in lists] and all(len(a) > 10 for a in lists)
    for a, b in zip(r["lidar_unc"], lists):
        assert a.tobytes() == b.tobytes()
    assert r["temporal_comp"].tobytes() == tc.tobytes()
    assert np.array_equal(r["table_off"], off) and r["table"].tobytes() == table.tobytes()
    assert np.array_equal(r["temporal_comp_rigid"]["q"] if L > 1 else [], tc["q"] if L > 1 else [])
    # each slot's per-point outputs are those of a handle that undistorted that slot alone, and the device-resident
    # undistorted cloud the voxel grid reads was not disturbed by the later slots or by scan_uncertainty
    for l, c in enumerate(slots):
        solo = plugin.MeasurementModel(L)
        s = solo.undistort(l, c["pts"], c["beg_time"], c["extrinsic"], c["lt"], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"],
                           want_pose=True)
        for k in ("xyz", "idx", "ok", "pop_point", "pose"):
            assert np.array_equal(g[l][k], s[k]), (l, k)
        assert np.array_equal(m.voxel_grid(l, None, 0.5), solo.voxel_grid(l, None, 0.5))
        solo.close()
    m.close()


def _check_ref(slots, imu_cov, ext, unc, r):
    lists, tcs, table = R.scan_uncertainty(slots, imu_cov, ext, unc)
    worst = 0.0

    def cmp(dev, ref):
        nonlocal worst
        assert np.abs(dev["T"] - ref.T).max() <= BAR
        rel = np.abs(dev["cov"] - ref.cov).max() / np.abs(ref.cov).max()
        assert rel <= BAR, rel
        worst = max(worst, rel)

    assert [len(a) for a in r["lidar_unc"]] == [len(a) for a in lists]
    for dev, ref in zip(r["lidar_unc"], lists):
        for k in range(len(ref)):
            cmp(dev[k], ref[k])
    for k, ref in enumerate(tcs):
        cmp(r["temporal_comp"][k], ref)
    flat = [p for t in table for p in t]
    assert r["table"].shape[0] == len(flat)
    assert np.array_equal(np.diff(r["table_off"]), [len(t) for t in table])
    for k, ref in enumerate(flat):
        cmp(r["table"][k], ref)
    print(f"largest covariance error / largest element: {worst:.3g}")
    return lists, worst


@pytest.mark.parametrize("motion", synth.UNDISTORT_MOTIONS)
def test_against_numpy_reference_motions(motion):
    slots, imu_cov, ext, unc = R.make_scan(3, n=[20000, 15000, 12000], seed=40, motion=motion)
    m, _, r = _device(slots, imu_cov, ext, unc)
    lists, _ = _check_ref(slots, imu_cov, ext, unc, r)
    assert all(len(a) > 10 for a in lists)
    m.close()


@pytest.mark.parametrize("L,kw", [(3, dict(ties=True)), (1, dict(lists="empty_cov")), (3, dict(lists="last_cov")),
                                  (3, dict(lists="max", imu_hz=4000.0)), (2, dict(lists="max", ties=True, imu_hz=4000.0))])
def test_against_numpy_reference_lists(L, kw):
    slots, imu_cov, ext, unc = R.make_scan(L, n=[40000, 30000, 30000][:L], seed=50 + L, **kw)
    if kw.get("lists") == "max":
        assert imu_cov.shape[0] == capi.MAX_COV
    m, _, r = _device(slots, imu_cov, ext, unc)
    lists, _ = _check_ref(slots, imu_cov, ext, unc, r)
    if kw.get("lists") == "empty_cov":
        assert lists == [[]] and r["table"].shape[0] == 0 and list(r["table_off"]) == [0, 0]
    else:
        assert all(len(a) > 10 for a in lists)
    m.close()


def test_zero_one_pop_slots_and_unreachable_pop_point():
    """Slot 0: the spline ends inside the scan, so the first pops (at the last points) are points get_pose cannot reach: their
    entries are built from the identity pose.  Slot 1: a single point (no pop).  Slot 2: cov_pointer set so that exactly one
    entry lies above the points' times (one pop, so no table entry)."""
    slots, imu_cov, ext, unc = R.make_scan(3, n=[8000, 1, 8000], seed=61)
    keep = slice(0, -5)
    slots[0] = dict(slots[0], ctrl_t=slots[0]["ctrl_t"][keep], ctrl_T=slots[0]["ctrl_T"][keep])
    c = slots[2]
    t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
    c["cov_pointer"] = int(np.searchsorted(c["imu_cov_t"], t[1], side="right"))
    assert c["imu_cov_t"][c["cov_pointer"] - 1] <= t[1] < c["imu_cov_t"][c["cov_pointer"]]
    m, g, r = _device(slots, imu_cov, ext, unc)
    assert g[0]["ok"][g[0]["pop_point"][0]] == 0 and g[0]["ok"][g[0]["pop_point"]].any()
    assert [len(a) for a in r["lidar_unc"]][1:] == [0, 1]
    assert list(np.diff(r["table_off"]))[1:] == [0, 0]
    _check_ref(slots, imu_cov, ext, unc, r)
    lists, tc, table, off = _host_compound(slots, g, imu_cov, R.to_capi(ext), unc)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(r["lidar_unc"], lists)) and r["table"].tobytes() == table.tobytes()
    m.close()


def test_end_to_end_update():
    """3 raw clouds -> undistort -> scan_uncertainty -> voxel grid -> upload_scan_device -> IESKF update, against the same
    merged scan uploaded from the host with the numpy-built table and temporal compensation."""
    case = synth.make_case("scan-unc", 30000, 120000, 3, 4)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    counts = [int((case.pts["lidar"] == l).sum()) for l in range(3)]
    # a stationary spline: the compensation is the identity and so is the temporal compensation, so the raw clouds are the
    # case's surface points re-expressed without the case's own temporal compensation
    slots, imu_cov, ext, unc = R.make_scan(3, n=counts, seed=70, motion="stationary")
    for l, c in enumerate(slots):
        p = case.pts["xyz"][case.pts["lidar"] == l].astype(np.float64)
        if l:
            Re, et = synth.q_to_R(case.x_true.ext[l].q[:]), np.array(case.x_true.ext[l].t[:])
            tc = case.temporal_comp[l - 1]
            b = (p @ Re.T + et) @ synth.q_to_R(tc["q"]).T + tc["t"]
            p = (b - et) @ Re
        c["pts"]["xyz"] = p.astype(np.float32)
    m = plugin.MeasurementModel(3, params=case.params)
    m.upload_map(snap)
    _undistort_all(m, slots)
    r = m.scan_uncertainty(imu_cov, R.to_capi(ext), unc)
    parts = []
    for l in range(3):
        ds = m.voxel_grid(l, None, 0.5)
        sp = np.zeros(ds.shape[0], capi.SCAN_PT)
        sp["xyz"] = ds[:, :3]; sp["lidar"] = l
        sp["table_idx"] = np.clip(ds[:, 3].astype(np.int32), 0, 65535).astype(np.uint16)
        parts.append(sp)
    merged = np.concatenate(parts)
    # every index is inside its slot's table, or the last (dropped) entry's index, which the reference also produces
    for l in range(3):
        keep = int(r["table_off"][l + 1] - r["table_off"][l])
        idx = parts[l]["table_idx"].astype(np.int64)
        assert idx.max() <= keep and (idx < keep).mean() > 0.5
    n = m.upload_scan_device(r["table"], r["table_off"], r["temporal_comp_rigid"])
    assert n == merged.shape[0]
    x_dev, P_dev = case.x_prop.copy(), case.P_prop.copy()
    rep_dev = m.update_iterated_dyn_share_modified(x_dev, P_dev, case.max_iter)

    lists, tcs, table = R.scan_uncertainty(slots, imu_cov, ext, unc)
    ref_table = np.zeros(sum(len(t) for t in table), capi.POSE_ENTRY)
    flat = [p for t in table for p in t]
    for k, p in enumerate(flat):
        ref_table[k]["T"], ref_table[k]["cov"] = p.T, p.cov
    ref_off = np.concatenate([[0], np.cumsum([len(t) for t in table])]).astype(np.uint32)
    ref_tc = np.zeros(2, capi.RIGID)
    for k, p in enumerate(tcs):
        ref_tc[k]["q"], ref_tc[k]["t"] = p.q, p.t
    h = plugin.MeasurementModel(3, params=case.params)
    h.upload_map(snap)
    h.upload_scan(merged, ref_table, ref_off, ref_tc)
    x_h, P_h = case.x_prop.copy(), case.P_prop.copy()
    rep_h = h.update_iterated_dyn_share_modified(x_h, P_h, case.max_iter)
    assert rep_dev.n_eff_last == rep_h.n_eff_last > 0 and rep_dev.passes == rep_h.passes
    v_dev, v_h = synth.state_to_vec(x_dev, 3), synth.state_to_vec(x_h, 3)
    assert np.abs(v_dev - v_h).max() <= BAR
    # regression: the synthetic table of the case, unrelated to these indices, gives another state
    h.upload_scan(merged, case.table, case.table_off, ref_tc)
    x_c, P_c = case.x_prop.copy(), case.P_prop.copy()
    h.update_iterated_dyn_share_modified(x_c, P_c, case.max_iter)
    assert np.abs(synth.state_to_vec(x_c, 3) - v_h).max() > 1e3 * BAR
    m.close(); h.close()


def _raw_call(m, a, table, cap, off, tc, lu=None, counts=None):
    return m.lib.malio_scan_uncertainty(m._h, C.byref(a) if a is not None else None, capi.ptr(table), cap, capi.ptr(off), capi.ptr(tc),
                                        capi.ptr(lu), capi.ptr(counts))


def test_error_returns_launch_nothing():
    slots, imu_cov, ext, unc = R.make_scan(2, n=[3000, 3000], seed=81)
    ext_c = R.to_capi(ext)
    cov = np.ascontiguousarray(imu_cov.reshape(-1, 36))
    u = np.ascontiguousarray(unc.reshape(36))
    a = capi.ScanUncArgs()
    a.imu_cov, a.n_cov, a.extrinsic, a.uncertainty = cov.ctypes.data, cov.shape[0], ext_c.ctypes.data, u.ctypes.data
    table = np.zeros(2 * capi.MAX_COV, capi.POSE_ENTRY)
    off = np.zeros(3, np.uint32)
    tc = np.zeros(1, capi.POSE)
    m = plugin.MeasurementModel(2)
    launches = lambda: m.counters().kernel_launches
    k0 = launches()
    assert _raw_call(m, a, table, table.shape[0], off, tc) == capi.ERR_STATE            # nothing undistorted yet
    c = slots[0]
    m.undistort(0, c["pts"], c["beg_time"], c["extrinsic"], c["lt"], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
    k0 = launches()
    assert _raw_call(m, a, table, table.shape[0], off, tc) == capi.ERR_STATE            # slot 1 missing
    c = slots[1]
    m.undistort(1, c["pts"], c["beg_time"], c["extrinsic"], c["lt"], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
    k0 = launches()
    assert _raw_call(m, None, table, table.shape[0], off, tc) == capi.ERR_INVALID_ARG
    assert _raw_call(m, a, None, table.shape[0], off, tc) == capi.ERR_INVALID_ARG
    assert _raw_call(m, a, table, table.shape[0], None, tc) == capi.ERR_INVALID_ARG
    assert _raw_call(m, a, table, table.shape[0], off, None) == capi.ERR_INVALID_ARG     # L = 2 needs temporal_comp
    for field in ("extrinsic", "uncertainty", "imu_cov"):
        b = capi.ScanUncArgs.from_buffer_copy(a)
        setattr(b, field, None)
        assert _raw_call(m, b, table, table.shape[0], off, tc) == capi.ERR_INVALID_ARG, field
    b = capi.ScanUncArgs.from_buffer_copy(a)
    b.n_cov = a.n_cov - 1
    assert _raw_call(m, b, table, table.shape[0], off, tc) == capi.ERR_INVALID_ARG       # not the list undistort saw
    assert _raw_call(m, a, table, 3, off, tc) == capi.ERR_CAPACITY
    need = int(off[2])
    assert need > 3 and "needs" in m.lib.malio_last_error(m._h).decode()
    assert launches() == k0
    assert _raw_call(m, a, table, need, off, tc) == capi.OK and launches() == k0 + 1
    # a LiDAR >= 1 whose cov_pointer is -1 has no imu_cov[cov_pointer] for its lt_lidar_frame (:471)
    m.undistort(1, c["pts"], c["beg_time"], c["extrinsic"], c["lt"], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], -1)
    k0 = launches()
    assert _raw_call(m, a, table, table.shape[0], off, tc) == capi.ERR_INVALID_ARG and launches() == k0
    m.close()
