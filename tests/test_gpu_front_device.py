"""The front half of a scan on device memory (malio_undistort_device, malio_voxel_grid_device, malio_scan_uncertainty_resident,
malio_upload_scan_resident) through their torch wrappers: bit-identical to the host-pointer calls stage by stage and through
the whole chain to the update and every output, ordered on the caller's stream, an unordered cloud and every bad pointer refused
by a host-side or flag-word check, and the transfer counters of a scan that never crosses the bus."""
import ctypes as C

import numpy as np
import pytest
import torch

import scan_unc_ref as R
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
LEAF = 0.5


def _raw(c_or_pts):
    """capi.RAW_PT records -> the float32 (n, 4) CUDA tensor undistort_tensor takes (the same bytes)."""
    pts = c_or_pts["pts"] if isinstance(c_or_pts, dict) else c_or_pts
    return torch.from_numpy(np.ascontiguousarray(pts).view(F).reshape(-1, 4)).cuda()


def _np(t):
    return t.cpu().numpy()


def _same_bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what


def _args(c):
    return (c["beg_time"], c["extrinsic"], c["lt"], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])


def _ud_host(m, l, c, pts=None):
    return m.undistort(l, c["pts"] if pts is None else pts, *_args(c), want_pose=True)


def _ud_dev(m, l, c, raw=None, **kw):
    return m.undistort_tensor(l, _raw(c) if raw is None else raw, *_args(c), **kw)


def _assert_undistort_equal(g, t, pts, what):
    """g: undistort()'s dict, t: undistort_tensor()'s with every output."""
    cloud = _np(t["cloud"])
    _same_bits(cloud[:, :3], g["xyz"], (what, "xyz"))
    _same_bits(cloud[:, 3], np.where(g["ok"] != 0, g["idx"], 0).astype(F), (what, "intensity"))
    _same_bits(cloud[:, 4], pts["curvature"], (what, "curvature"))
    for k in ("idx", "ok", "pop_point", "pose"):
        _same_bits(_np(t[k]), g[k], (what, k))
    assert t["n_pops"] == g["pop_point"].shape[0]


# ------------------------------------------------------------------ 1. stage by stage
@pytest.mark.parametrize("kw", [dict(motion="generic"), dict(motion="stationary"), dict(ties=True)], ids=["generic", "stationary", "ties"])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_stages_equal_host_calls(L, kw):
    slots, _, _, _ = R.make_scan(L, n=[30011, 20002, 25003][:L], seed=110 + L, **kw)
    host, dev = plugin.MeasurementModel(L), plugin.MeasurementModel(L)
    st = torch.cuda.current_stream().cuda_stream
    for l, c in enumerate(slots):
        g = _ud_host(host, l, c)
        t = _ud_dev(dev, l, c)
        assert g["ok"].any() and t["n_pops"] > 5
        _assert_undistort_equal(g, t, c["pts"], l)
        # the voxel grid from the slot ...
        ref = host.voxel_grid(l, None, LEAF)
        out = dev.voxel_grid_tensor(l, None, LEAF)
        assert 0 < ref.shape[0] < c["pts"].shape[0]
        _same_bits(_np(out), ref, (l, "slot"))
        # ... from an explicit tensor, with non-finite points among them ...
        cloud = t["cloud"].clone()
        cloud[5, 0], cloud[77, 1], cloud[1234, 2], cloud[9, 3] = float("nan"), float("inf"), float("-inf"), float("nan")
        ref = host.voxel_grid(l, _np(cloud), 0.3)
        _same_bits(_np(dev.voxel_grid_tensor(l, cloud, 0.3)), ref, (l, "explicit"))
        # ... and into a buffer that is too small: the full count, the first rows only
        n, m = cloud.shape[0], ref.shape[0]
        for cap in (1, m // 3, m - 1):
            buf = torch.full((m, 5), -7.0, device="cuda")
            k = C.c_uint32(0)
            assert dev.lib.malio_voxel_grid_device(dev._h, l, cloud.data_ptr(), n, C.c_float(0.3), buf.data_ptr(), cap, C.addressof(k), st) == capi.OK
            b = _np(buf)
            assert k.value == m and np.all(b[cap:] == -7.0)
            _same_bits(b[:cap], ref[:cap], (l, cap))
        # a cloud without a finite point
        assert dev.voxel_grid_tensor(l, torch.full((100, 5), float("nan"), device="cuda"), LEAF).shape == (0, 5)
    host.close()
    dev.close()


def test_wanted_outputs_only():
    slots, _, _, _ = R.make_scan(1, n=[9001], seed=120)
    c = slots[0]
    m = plugin.MeasurementModel(1)
    full = _ud_dev(m, 0, c)
    for want in ((), ("idx",), ("cloud", "pop_point")):
        t = _ud_dev(m, 0, c, want=want)
        assert set(t) == set(want) | {"n_pops"} and t["n_pops"] == full["n_pops"]
        for k in want:
            _same_bits(_np(t[k]), _np(full[k]), k)
    m.close()


# ------------------------------------------------------------------ 2. the whole chain
def _chain_inputs(case, seed, **kw):
    """Raw clouds whose stationary undistortion gives the case's scan points per LiDAR (as test_gpu_scan_uncertainty's
    end-to-end test builds them), with one shared IMU list."""
    L = case.n_lidar
    counts = [int((case.pts["lidar"] == l).sum()) for l in range(L)]
    slots, imu_cov, ext, unc = R.make_scan(L, n=counts, seed=seed, motion="stationary", **kw)
    for l, c in enumerate(slots):
        p = case.pts["xyz"][case.pts["lidar"] == l].astype(np.float64)
        if l:
            Re, et = synth.q_to_R(case.x_true.ext[l].q[:]), np.array(case.x_true.ext[l].t[:])
            tc = case.temporal_comp[l - 1]
            b = (p @ Re.T + et) @ synth.q_to_R(tc["q"]).T + tc["t"]
            p = (b - et) @ Re
        c["pts"]["xyz"] = p.astype(F)
    return slots, imu_cov, R.to_capi(ext), unc


def _host_chain(m, slots, imu_cov, ext, unc):
    for l, c in enumerate(slots):
        m.undistort(l, c["pts"], *_args(c))
    r = m.scan_uncertainty(imu_cov, ext, unc)
    for l in range(len(slots)):
        m.voxel_grid(l, None, LEAF)
    n = m.upload_scan_device(r["table"], r["table_off"], r["temporal_comp_rigid"])
    return n, r["table_off"], r["temporal_comp"]


def _tensor_chain(m, slots, imu_cov, ext, unc, raws=None):
    for l, c in enumerate(slots):
        m.undistort_tensor(l, _raw(c) if raws is None else raws[l], *_args(c), want=())
    off, tc = m.scan_uncertainty_resident(imu_cov, ext, unc)
    for l in range(len(slots)):
        m.voxel_grid_tensor(l, None, LEAF)
    return m.upload_scan_resident(), off, tc


def _after(m, case):
    """The update and every output that reads the scan, the table or the undistorted clouds."""
    x, P = case.x_prop.copy(), case.P_prop.copy()
    rep = m.update_iterated_dyn_share_modified(x, P, case.max_iter)
    aux = m.aux()
    cls, w = m.map_incremental(x, 0.5, True)
    tags = np.array([2.5, 0.5, 1.5][: case.n_lidar], F)
    return dict(x=synth.state_to_vec(x, case.n_lidar), P=P, cls=cls, w=w, dense=m.publish_frame_world(x, True, tags),
                down=m.publish_frame_world(x, False), **aux), (rep.passes, rep.searches, rep.converged_count, rep.last_status,
                                                               rep.n_eff_last, bytes(rep.dx_last))


def _model(case, mode):
    m = plugin.MeasurementModel(case.n_lidar, params=case.params)
    if mode == "snapshot":
        m.upload_map(plugin.build_static_snapshot(case.map_xyz, case.map_normal_y))
    else:
        m.map_build(case.map_xyz, case.map_normal_y)
    return m


@pytest.mark.parametrize("L,mode,kw", [(3, "snapshot", {}), (3, "devmap", dict(lists="max", imu_hz=4000.0)),
                                       (2, "snapshot", dict(lists="max", imu_hz=4000.0)), (1, "devmap", {})],
                         ids=["L3-snapshot", "L3-devmap-max", "L2-snapshot-max", "L1-devmap"])
def test_chain_equals_host_chain(L, mode, kw):
    base = synth.make_case("front", 30000, 120000, L, 3)
    host, dev = _model(base, mode), _model(base, mode)
    # the second scan is larger (every buffer grows behind calls that returned after enqueueing), the third smaller
    for k, N in enumerate((30000, 60000, 12000)):
        case = base if k == 0 else synth.make_case("front", N, 120000, L, 3, seed_scan=400 + k, seed_state=500 + k, map_xyz=base.map_xyz)
        slots, imu_cov, ext, unc = _chain_inputs(case, 130 + k, **kw)
        if kw:
            assert imu_cov.shape[0] == capi.MAX_COV and slots[0]["ctrl_t"].shape[0] == synth.MAX_CTRL
        na, off_a, tc_a = _host_chain(host, slots, imu_cov, ext, unc)
        nb, off_b, tc_b = _tensor_chain(dev, slots, imu_cov, ext, unc)
        assert na == nb > 1000
        _same_bits(off_a, off_b, (k, "table_off"))
        _same_bits(tc_a, tc_b, (k, "temporal_comp"))
        assert all(int(off_a[l + 1] - off_a[l]) > 5 for l in range(L))
        a, rep_a = _after(host, case)
        b, rep_b = _after(dev, case)
        assert rep_a == rep_b and rep_a[4] > 500, (k, rep_a[:5])
        for key in a:
            _same_bits(a[key], b[key], (k, key))
    host.close()
    dev.close()


# ------------------------------------------------------------------ 3. stream order
def test_stream_order():
    slots, _, _, _ = R.make_scan(1, n=[131072], seed=140)
    c = slots[0]
    host, dev = plugin.MeasurementModel(1), plugin.MeasurementModel(1)
    g = _ud_host(host, 0, c)
    ref = host.voxel_grid(0, None, LEAF)
    _ud_dev(dev, 0, c)                                        # same sizes once: the calls below grow nothing
    dev.voxel_grid_tensor(0, None, LEAF)
    torch.cuda.synchronize()
    good = _raw(c)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        raw = torch.zeros_like(good)                          # an ordered cloud of zeros until the side stream passes the sleep
        torch.cuda._sleep(200_000_000)
        raw.copy_(good)
        t = _ud_dev(dev, 0, c, raw=raw)                       # waits for its verdict: sees the copy
        raw.zero_()                                           # the caller may reuse its buffer: nothing reads it after the call
    side.synchronize()
    _assert_undistort_equal(g, t, c["pts"], "side stream")
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        cloud = t["cloud"].clone()                            # enqueued behind the sleep: the filter must wait for it
        out = dev.voxel_grid_tensor(0, cloud, LEAF)
        total = out.double().sum()                            # right behind the call, on the same stream
        cloud.zero_()
    side.synchronize()
    _same_bits(_np(out), ref, "voxel grid")
    np.testing.assert_allclose(float(total), ref.astype(np.float64).sum(), rtol=1e-9)   # (summation orders differ)
    host.close()
    dev.close()


# ------------------------------------------------------------------ 4. refusals
def _unordered(pts, pos):
    bad = pts.copy()
    if pos == 1:
        bad["curvature"][0] = bad["curvature"][2]             # point 1 lies before point 0
        assert bad["curvature"][1] < bad["curvature"][0]
    else:
        bad["curvature"][pos] = np.nextafter(bad["curvature"][pos - 1], F(-np.inf))
    return bad


def _status(fn, *a, **k):
    try:
        fn(*a, **k)
    except capi.MalioError as e:
        return e.status, str(e)
    return capi.OK, ""


def test_unordered_cloud_is_refused_and_the_slot_recovers():
    case = synth.make_case("front-bad", 20000, 100000, 2, 3)
    slots, imu_cov, ext, unc = _chain_inputs(case, 150)
    ref = _model(case, "snapshot")
    _host_chain(ref, slots, imu_cov, ext, unc)
    a, rep_a = _after(ref, case)
    m = _model(case, "snapshot")
    _tensor_chain(m, slots, imu_cov, ext, unc)
    c = slots[1]
    n = c["pts"].shape[0]
    for pos in (1, n // 2, n - 1):
        bad = _unordered(c["pts"], pos)
        assert _status(_ud_host, m, 1, c, bad)[0] == capi.ERR_INVALID_ARG      # the host call refuses before it touches the slot
        assert m.voxel_grid(1, None, LEAF).shape[0] > 0
        k0 = m.counters()
        status, msg = _status(_ud_dev, m, 1, c, _raw(bad))
        assert status == capi.ERR_INVALID_ARG and "sorted by curvature" in msg, pos
        k1 = m.counters()
        assert k1.kernel_launches - k0.kernel_launches == 4 and k1.d2h_bytes == k0.d2h_bytes
        # the slot holds no result until it is undistorted again
        assert _status(m.voxel_grid, 1, None, LEAF)[0] == capi.ERR_STATE
        assert _status(m.voxel_grid_tensor, 1, None, LEAF)[0] == capi.ERR_STATE
        assert _status(m.scan_uncertainty, imu_cov, ext, unc)[0] == capi.ERR_STATE
        assert _status(m.scan_uncertainty_resident, imu_cov, ext, unc)[0] == capi.ERR_STATE
        assert _status(m.upload_scan_resident)[0] == capi.ERR_STATE
        assert _status(m.publish_frame_world, case.x_prop, True, np.zeros(2, F))[0] == capi.ERR_STATE
        assert m.voxel_grid(0, None, LEAF).shape[0] > 0                          # the other slot is not affected
        _ud_dev(m, 1, c, want=())
        assert m.voxel_grid(1, None, LEAF).shape[0] > 0
    _tensor_chain(m, slots, imu_cov, ext, unc)
    b, rep_b = _after(m, case)
    assert rep_a == rep_b
    for key in a:
        _same_bits(a[key], b[key], key)
    ref.close()
    m.close()


def test_nan_time_is_accepted_where_the_host_call_accepts_it():
    slots, _, _, _ = R.make_scan(1, n=[20000], seed=160)
    c = slots[0]
    host, dev = plugin.MeasurementModel(1), plugin.MeasurementModel(1)
    for pos in (0, 1, 7000, 19999):
        pts = c["pts"].copy()
        pts["curvature"][pos] = np.nan
        _assert_undistort_equal(_ud_host(host, 0, c, pts), _ud_dev(dev, 0, c, _raw(pts)), pts, pos)
    host.close()
    dev.close()


def test_pointer_classes_launch_nothing_and_leave_the_slot():
    slots, _, _, _ = R.make_scan(1, n=[6000], seed=170)
    c = slots[0]
    m = plugin.MeasurementModel(1)
    lib, h = m.lib, m._h
    st = torch.cuda.current_stream().cuda_stream
    n = c["pts"].shape[0]
    t = _ud_dev(m, 0, c)
    ref = _np(m.voxel_grid_tensor(0, None, LEAF))
    a, cv, keep = plugin._undistort_args(*_args(c))
    raw = _raw(c)
    outs = [torch.empty((n, 5), device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"),
            torch.empty(n + 8, dtype=torch.uint8, device="cuda"), torch.empty(cv.shape[0], dtype=torch.int32, device="cuda"),
            torch.empty((n, 7), dtype=torch.float64, device="cuda")]
    k = C.c_uint32(0)

    def undistort(pts, o):
        return lib.malio_undistort_device(h, 0, pts, n, C.addressof(a), *o, C.addressof(k), st)

    def voxel(inp, out):
        return lib.malio_voxel_grid_device(h, 0, inp, n, C.c_float(LEAF), out, n, C.addressof(k), st)

    hp = np.zeros(n * 16, F)
    pin = torch.empty(n * 16).pin_memory()
    bad = {"host": hp.ctypes.data, "pinned": pin.data_ptr(), "misaligned": outs[0].data_ptr() + 2}
    if torch.cuda.device_count() > 1:
        other = torch.empty(n * 16, device="cuda:1")
        bad["other device"] = other.data_ptr()
    good = [o.data_ptr() for o in outs]
    c0 = m.counters()
    assert undistort(None, good) == capi.ERR_INVALID_ARG
    for what, p in bad.items():
        assert undistort(p, good) == capi.ERR_INVALID_ARG, what
        for j in range(5):
            o = list(good)
            o[j] = p
            assert undistort(raw.data_ptr(), o) == capi.ERR_INVALID_ARG, (what, j)
        assert voxel(p, None) == capi.ERR_INVALID_ARG, what
        assert voxel(t["cloud"].data_ptr(), p) == capi.ERR_INVALID_ARG, what
        assert voxel(None, p) == capi.ERR_INVALID_ARG, what
    # the host call's own argument checks come first and are the host call's
    assert lib.malio_undistort_device(h, 3, raw.data_ptr(), n, C.addressof(a), *good, C.addressof(k), st) == capi.ERR_INVALID_ARG
    assert lib.malio_undistort_device(h, 0, raw.data_ptr(), n, None, *good, C.addressof(k), st) == capi.ERR_INVALID_ARG
    b = capi.UndistortArgs.from_buffer_copy(a)
    b.cov_pointer = b.n_cov
    assert lib.malio_undistort_device(h, 0, raw.data_ptr(), n, C.addressof(b), *good, C.addressof(k), st) == capi.ERR_INVALID_ARG
    b = capi.UndistortArgs.from_buffer_copy(a)
    b.n_ctrl = synth.MAX_CTRL + 1
    assert lib.malio_undistort_device(h, 0, raw.data_ptr(), n, C.addressof(b), *good, C.addressof(k), st) == capi.ERR_CAPACITY
    assert lib.malio_voxel_grid_device(h, 0, None, 0, C.c_float(0.0), None, 0, C.addressof(k), st) == capi.ERR_INVALID_ARG
    assert lib.malio_voxel_grid_device(h, 3, None, 0, C.c_float(LEAF), None, 0, C.addressof(k), st) == capi.ERR_INVALID_ARG
    c1 = m.counters()
    assert c1.kernel_launches == c0.kernel_launches and c1.h2d_bytes == c0.h2d_bytes and c1.d2h_bytes == c0.d2h_bytes
    # none of the refused calls touched the slot
    _same_bits(_np(m.voxel_grid_tensor(0, None, LEAF)), ref, "slot")
    assert undistort(raw.data_ptr(), good) == capi.OK and k.value == t["n_pops"]
    _same_bits(_np(outs[0]), _np(t["cloud"]), "cloud")
    for bad_t in (raw.cpu(), raw.double(), raw[:, :3].contiguous(), torch.empty((n, 8), device="cuda")[:, ::2]):
        with pytest.raises(ValueError):
            m.undistort_tensor(0, bad_t, *_args(c))
    m.close()


def test_upload_scan_resident_states_and_empty_slots():
    slots, imu_cov, ext, unc = R.make_scan(2, n=[8000, 8000], seed=180)
    ext = R.to_capi(ext)
    m = plugin.MeasurementModel(2)
    assert _status(m.upload_scan_resident)[0] == capi.ERR_STATE                  # nothing undistorted, no table
    for l, c in enumerate(slots):
        _ud_dev(m, l, c, want=())
    assert _status(m.upload_scan_resident)[0] == capi.ERR_STATE                  # no table yet
    off, tc = m.scan_uncertainty_resident(imu_cov, ext, unc)
    assert _status(m.upload_scan_resident)[0] == capi.ERR_STATE                  # no down-sampled clouds
    for l in range(2):
        m.voxel_grid_tensor(l, None, LEAF)
    n = m.upload_scan_resident()
    assert n > 0 and m.upload_scan_resident() == n                               # the table stays resident
    r = m.scan_uncertainty(imu_cov, ext, unc)                                    # the host-table call leaves its table resident too
    _same_bits(r["table_off"], off, "table_off")
    assert m.upload_scan_resident() == n
    _ud_dev(m, 1, slots[1], want=())                                             # a slot undistorted again: the table is stale
    status, msg = _status(m.upload_scan_resident)
    assert status == capi.ERR_STATE and "table" in msg
    # a LiDAR with a single point has no pop and so no table entry: the upload refuses it as malio_upload_scan_device does
    one = dict(slots[1], pts=slots[1]["pts"][:1].copy())
    _ud_dev(m, 1, one, want=())
    off, _ = m.scan_uncertainty_resident(imu_cov, ext, unc)
    assert off[2] == off[1]
    m.voxel_grid_tensor(1, None, LEAF)
    status, msg = _status(m.upload_scan_resident)
    assert status == capi.ERR_INVALID_ARG and "2 entries" in msg
    # an empty slot: nothing is launched, nothing is read
    c0 = m.counters()
    t = m.undistort_tensor(1, torch.empty((0, 4), device="cuda"), *_args(slots[1]))
    assert t["n_pops"] == 0 and t["cloud"].shape == (0, 5) and t["pop_point"].shape == (0,)
    assert m.voxel_grid_tensor(1, None, LEAF).shape == (0, 5)
    assert m.voxel_grid_tensor(1, torch.empty((0, 5), device="cuda"), LEAF).shape == (0, 5)
    assert m.counters().kernel_launches == c0.kernel_launches
    m.close()


# ------------------------------------------------------------------ 5. counters
def test_counters_of_a_scan_that_stays_on_the_device():
    L = 3
    case = synth.make_case("front-ctr", 24000, 100000, L, 3)
    slots, imu_cov, ext, unc = _chain_inputs(case, 190)
    n_cov = imu_cov.shape[0]
    lists = sum(c["ctrl_t"].shape[0] * 17 * 8 + n_cov * 8 for c in slots)
    host, dev = _model(case, "snapshot"), _model(case, "snapshot")
    h0, d0 = host.counters(), dev.counters()
    n_scan, off, _ = _host_chain(host, slots, imu_cov, ext, unc)
    assert _tensor_chain(dev, slots, imu_cov, ext, unc)[0] == n_scan
    h1, d1 = host.counters(), dev.counters()
    pose, entry = capi.POSE.itemsize, capi.POSE_ENTRY.itemsize
    n_raw, n_tab = sum(c["pts"].shape[0] for c in slots), int(off[L])
    # the tensor chain: the control points and IMU times of every slot and imu_cov in, the compensations out
    assert d1.h2d_bytes - d0.h2d_bytes == lists + n_cov * 36 * 8
    assert d1.d2h_bytes - d0.d2h_bytes == (L - 1) * pose
    # the host chain as it has always counted: raw points and the table in (the table twice: out and in again), the
    # undistorted points, the table and the down-sampled clouds out; undistort() fetches xyz, idx and ok
    assert h1.h2d_bytes - h0.h2d_bytes == n_raw * 16 + lists + n_cov * 36 * 8 + n_tab * entry
    assert h1.d2h_bytes - h0.d2h_bytes == n_raw * 25 + n_tab * entry + (L - 1) * pose + n_scan * 20
    # one more launch per undistortion (the order check); voxel_grid() runs the filter twice (its size query)
    assert (d1.kernel_launches - d0.kernel_launches) - L == (h1.kernel_launches - h0.kernel_launches) - 8 * L
    host.close()
    dev.close()
