"""The measurement path on device memory (malio_upload_scan_from_device, malio_download_aux_device, malio_map_incremental_device,
malio_world_register_device) through their torch wrappers: bit-identical to the host-pointer calls, ordered on the caller's
stream, argument and state errors caught before anything is launched, and a bad scan refused without touching the resident one."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
AUX = ("normal_y", "nn_idx", "nn_sqdist", "selected", "world")


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _records(pts):
    """capi.SCAN_PT records -> the int32 (n, 4) CUDA tensor upload_scan_tensor takes (the same bytes)."""
    return _cuda(np.ascontiguousarray(pts).view(np.int32).reshape(-1, 4))


def _np(t):
    return None if t is None else t.cpu().numpy()


def _same_bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.tobytes() == b.tobytes(), what


def _model(case, mode, sort):
    m = plugin.MeasurementModel(case.n_lidar, sort_queries=sort, params=case.params)
    if mode == "snapshot":
        m.upload_map(plugin.build_static_snapshot(case.map_xyz, case.map_normal_y))
    else:
        m.map_build(case.map_xyz, case.map_normal_y)
    return m


def _report(rep):
    return (rep.passes, rep.searches, rep.converged_count, rep.last_status, rep.n_eff_last, bytes(rep.dx_last))


def _scan(m, case, upload_dev, out_dev):
    """One scan: upload, the IESKF update, every per-point output.  upload_dev / out_dev pick the device-memory calls."""
    if upload_dev:
        m.upload_scan_tensor(_records(case.pts), case.table, case.table_off, case.temporal_comp)
    else:
        m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    x, P = case.x_prop.copy(), case.P_prop.copy()
    rep = m.update_iterated_dyn_share_modified(x, P, case.max_iter)
    if out_dev:
        aux = {k: _np(v) for k, v in m.aux_tensor().items()}
        aux["nn_idx"] = aux["nn_idx"].view(np.uint32)
        cls, w = (_np(t) for t in m.map_incremental_tensor(x, 0.5, True))
        reg = _np(m.publish_frame_world_tensor(x, False))
    else:
        aux = m.aux()
        cls, w = m.map_incremental(x, 0.5, True)
        reg = m.publish_frame_world(x, False)
    return dict(x=synth.state_to_vec(x, case.n_lidar), P=P, rep=_report(rep), cls=cls, w=w, reg=reg, **aux)


def _assert_same(a, b):
    for k in a:
        if k == "rep":
            assert a[k] == b[k], k
        else:
            _same_bits(a[k], b[k], k)


@pytest.mark.parametrize("mode", ["snapshot", "devmap"])
@pytest.mark.parametrize("sort", [True, False])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_tensor_path_equals_host_calls(L, sort, mode):
    case = synth.make_case(f"scan-dev L{L}", 9001, 90000, L, 3, varied_map_cov=True)
    host, dev = _model(case, mode, sort), _model(case, mode, sort)
    a = _scan(host, case, False, False)
    b = _scan(dev, case, True, True)
    _assert_same(a, b)
    assert (a["cls"] != capi.MAP_SKIP).sum() > 0.5 * len(a["cls"])
    # mixed: a host upload with device outputs, and the reverse, on the same two handles
    _assert_same(a, _scan(host, case, False, True))
    _assert_same(a, _scan(dev, case, True, False))
    host.close()
    dev.close()


def test_c2_size_equals_host_calls():
    case = synth.case_C2()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    host = plugin.MeasurementModel(case.n_lidar, params=case.params)
    dev = plugin.MeasurementModel(case.n_lidar, params=case.params)
    host.upload_map(snap)
    dev.upload_map(snap)
    _assert_same(_scan(host, case, False, False), _scan(dev, case, True, True))
    host.close()
    dev.close()


def _undistort_slots(m, sizes):
    for slot, n in enumerate(sizes):
        c = synth.undistort_case(n, lidar=slot, seed=90 + slot)
        ok, q, p = plugin.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], min(c["end_time"], c["ctrl_t"][-3]))
        assert ok
        m.undistort(slot, c["pts"], c["beg_time"], c["extrinsic"], (q, p), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])


@pytest.mark.parametrize("L", [1, 2, 3])
def test_dense_registration_equals_host_call(L):
    case = synth.make_case(f"dense L{L}", 500, 5000, L, 3)
    m = plugin.MeasurementModel(L, params=case.params)
    m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    _undistort_slots(m, [8001, 0, 5003][:L])
    tags = np.array([2.5, 0.5, 1.5][:L], F)
    ref = m.publish_frame_world(case.x_true, True, tags)
    out = m.publish_frame_world_tensor(case.x_true, True, tags)
    assert out.dtype == torch.float32 and tuple(out.shape) == ref.shape
    _same_bits(_np(out), ref, "dense")
    m.close()


def _masked_add_host(m, cls, w, ny):
    keep = (cls == capi.MAP_ADD) | (cls == capi.MAP_ADD_NO_DOWNSAMPLE)
    m.map_add_points(w[keep], ny[keep])


def _masked_add_tensor(m, cls, w, ny):
    keep = (cls == capi.MAP_ADD) | (cls == capi.MAP_ADD_NO_DOWNSAMPLE)
    m.map_add_points_tensor(w[keep].contiguous(), ny[keep].contiguous())


def test_ten_scan_loop_on_twin_handles():
    base = synth.make_case("loop", 4000, 60000, 3, 3)
    host = plugin.MeasurementModel(3, params=base.params)
    dev = plugin.MeasurementModel(3, params=base.params)
    host.map_build(base.map_xyz, base.map_normal_y)
    dev.map_build_tensor(_cuda(base.map_xyz), _cuda(base.map_normal_y))
    for k in range(10):
        case = synth.make_case("loop", 4000, 60000, 3, 3, seed_scan=200 + k, seed_state=300 + k, map_xyz=base.map_xyz)
        host.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
        dev.upload_scan_tensor(_records(case.pts), case.table, case.table_off, case.temporal_comp)
        xa, Pa = case.x_prop.copy(), case.P_prop.copy()
        xb, Pb = case.x_prop.copy(), case.P_prop.copy()
        ra = host.update_iterated_dyn_share_modified(xa, Pa, case.max_iter)
        rb = dev.update_iterated_dyn_share_modified(xb, Pb, case.max_iter)
        assert _report(ra) == _report(rb), k
        _same_bits(synth.state_to_vec(xa, 3), synth.state_to_vec(xb, 3), k)
        _same_bits(Pa, Pb, k)
        cls, w = host.map_incremental(xa, 0.5, True)
        ny = host.aux(nn_idx=False, nn_sqdist=False, selected=False, world=False)["normal_y"]
        tcls, tw = dev.map_incremental_tensor(xb, 0.5, True)
        tny = dev.aux_tensor(nn_idx=False, nn_sqdist=False, selected=False, world=False)["normal_y"]
        _masked_add_host(host, cls, w, ny)
        _masked_add_tensor(dev, tcls, tw, tny)
        a, b = host.map_download(), dev.map_download()
        for key in a:
            _same_bits(a[key], b[key], (k, key))
        assert a["xyz"].shape[0] > base.map_xyz.shape[0]
    host.close()
    dev.close()


def test_stream_order():
    case = synth.make_case("order", 20000, 100000, 2, 3)
    host = _model(case, "snapshot", True)
    dev = _model(case, "snapshot", True)
    a = _scan(host, case, False, False)
    _scan(dev, case, True, True)                          # same sizes once: the timed calls below grow nothing
    torch.cuda.synchronize()
    good = _records(case.pts)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        rec = torch.zeros_like(good)                      # all-zero records (valid ids) until the side stream passes the sleep
        torch.cuda._sleep(200_000_000)
        rec.copy_(good)
        dev.upload_scan_tensor(rec, case.table, case.table_off, case.temporal_comp)   # waits for the check: sees the copy
        rec.zero_()                                       # the caller may reuse its buffer: the scan was copied
    side.synchronize()
    x, P = case.x_prop.copy(), case.P_prop.copy()
    dev.update_iterated_dyn_share_modified(x, P, case.max_iter)
    _same_bits(synth.state_to_vec(x, case.n_lidar), a["x"], "x")
    with torch.cuda.stream(side):
        torch.cuda._sleep(400_000_000)                    # ~0.2 s at 1.98 GHz
        t0 = time.perf_counter()
        aux = dev.aux_tensor()
        cls, w = dev.map_incremental_tensor(x, 0.5, True)
        reg = dev.publish_frame_world_tensor(x, False)
        dt = time.perf_counter() - t0
        pending = not side.query()
        sums = torch.stack([aux["normal_y"].double().sum(), aux["nn_sqdist"].double().sum(), (aux["nn_idx"] >= 0).sum().double(),
                            aux["selected"].double().sum(), cls.double().sum(), w.double().sum(), reg.double().sum()])
    side.synchronize()
    assert pending
    assert dt < 0.05, dt
    ref = [a["normal_y"].astype(np.float64).sum(), a["nn_sqdist"].astype(np.float64).sum(), float((a["nn_idx"] != 0xFFFFFFFF).sum()),
           a["selected"].astype(np.float64).sum(), a["cls"].astype(np.float64).sum(), a["w"].astype(np.float64).sum(),
           a["reg"].astype(np.float64).sum()]
    np.testing.assert_allclose(sums.cpu().numpy(), ref, rtol=1e-9, atol=1e-6)   # (summation orders differ)
    _same_bits(_np(reg), a["reg"], "reg")
    _same_bits(_np(cls), a["cls"], "cls")
    _same_bits(_np(aux["nn_idx"]).view(np.uint32), a["nn_idx"], "nn_idx")
    host.close()
    dev.close()


def test_bad_lidar_id_is_refused_and_the_scan_stays():
    case = synth.make_case("bad-id", 5003, 50000, 2, 3)
    m = _model(case, "snapshot", True)
    m.upload_scan_tensor(_records(case.pts), case.table, case.table_off, case.temporal_comp)
    ok0, H0, h0, s0 = m.h_share_model(case.x_prop, True)
    assert ok0
    n = case.pts.shape[0]
    for pos in (0, n // 2, n - 1):
        bad = case.pts.copy()
        bad["lidar"][pos] = case.n_lidar
        c0 = m.counters()
        with pytest.raises(capi.MalioError) as e:
            m.upload_scan_tensor(_records(bad), case.table, case.table_off, case.temporal_comp)
        assert e.value.status == capi.ERR_INVALID_ARG and "lidar" in str(e.value)
        c1 = m.counters()
        assert c1.kernel_launches - c0.kernel_launches == 1 and c1.h2d_bytes == c0.h2d_bytes    # the check only
        m.rearm_scan()
        ok, H1, h1, s1 = m.h_share_model(case.x_prop, True)
        assert ok and s1.n_eff == s0.n_eff
        _same_bits(H1, H0, pos)
        _same_bits(h1, h0, pos)
    m.close()


def test_pointer_classes_and_state_errors_launch_nothing():
    case = synth.make_case("errors", 3000, 40000, 2, 3)
    m = _model(case, "snapshot", True)
    lib, h = m.lib, m._h
    st = torch.cuda.current_stream().cuda_stream
    ps = case.x_prop.pass_state()
    n = case.pts.shape[0]
    rec = _records(case.pts)
    f1 = torch.empty(n, device="cuda")
    u8 = torch.empty(n, dtype=torch.uint8, device="cuda")
    out4 = torch.empty((n + 1, 4), device="cuda")
    tag = np.zeros(2, F)
    args = (capi.ptr(case.table), capi.ptr(case.table_off), capi.ptr(case.temporal_comp))
    m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    # STATE before a measurement pass / before the undistortion, with valid pointers
    c0 = m.counters()
    assert lib.malio_download_aux_device(h, f1.data_ptr(), None, None, None, None, st) == capi.ERR_STATE
    assert lib.malio_map_incremental_device(h, C.byref(ps), 0.5, 1, u8.data_ptr(), None, st) == capi.ERR_STATE
    nn = C.c_uint32(7)
    for src in (capi.WORLD_DOWNSAMPLED, capi.WORLD_DENSE):
        assert lib.malio_world_register_device(h, C.byref(ps), src, capi.ptr(tag), out4.data_ptr(), n, C.byref(nn), st) == capi.ERR_STATE
    assert m.counters().kernel_launches == c0.kernel_launches
    m.h_share_model(case.x_prop, True)
    c0 = m.counters()
    hp = np.zeros((n + 1) * 4, F)
    pin = torch.empty((n + 1) * 4).pin_memory()
    bad = {"host": hp.ctypes.data, "pinned": pin.data_ptr(), "misaligned": f1.data_ptr() + 2}
    for what, p in dict(bad, null=None).items():
        assert lib.malio_upload_scan_from_device(h, p, n, *args, st) == capi.ERR_INVALID_ARG, what
        assert lib.malio_map_incremental_device(h, C.byref(ps), 0.5, 1, p, None, st) == capi.ERR_INVALID_ARG, what
        if p is not None:
            for k in range(5):
                outs = [None] * 5
                outs[k] = p
                assert lib.malio_download_aux_device(h, *outs, st) == capi.ERR_INVALID_ARG, (what, k)
            assert lib.malio_map_incremental_device(h, C.byref(ps), 0.5, 1, u8.data_ptr(), p, st) == capi.ERR_INVALID_ARG, what
            assert lib.malio_world_register_device(h, C.byref(ps), 0, None, p, n, C.byref(nn), st) == capi.ERR_INVALID_ARG, what
    assert lib.malio_world_register_device(h, C.byref(ps), 0, None, None, n, C.byref(nn), st) == capi.ERR_INVALID_ARG
    for off in (4, 8, 12):                                # 4-byte aligned, not 16: world_kernel stores float4
        assert lib.malio_world_register_device(h, C.byref(ps), 0, None, out4.data_ptr() + off, n, C.byref(nn), st) == capi.ERR_INVALID_ARG
    if torch.cuda.device_count() > 1:
        other = torch.empty((n, 4), dtype=torch.int32, device="cuda:1")
        assert lib.malio_upload_scan_from_device(h, other.data_ptr(), n, *args, st) == capi.ERR_INVALID_ARG
        assert lib.malio_world_register_device(h, C.byref(ps), 0, None, other.data_ptr(), n, C.byref(nn), st) == capi.ERR_INVALID_ARG
    # the host call's own argument checks
    assert lib.malio_map_incremental_device(h, C.byref(ps), 0.0, 1, u8.data_ptr(), None, st) == capi.ERR_INVALID_ARG
    assert lib.malio_world_register_device(h, C.byref(ps), 5, None, out4.data_ptr(), n, C.byref(nn), st) == capi.ERR_INVALID_ARG
    assert lib.malio_world_register_device(h, C.byref(ps), capi.WORLD_DENSE, None, out4.data_ptr(), n, C.byref(nn), st) == capi.ERR_INVALID_ARG
    assert lib.malio_upload_scan_from_device(h, rec.data_ptr(), n, capi.ptr(case.table), capi.ptr(case.table_off), None, st) == capi.ERR_INVALID_ARG
    c1 = m.counters()
    assert c1.kernel_launches == c0.kernel_launches and c1.h2d_bytes == c0.h2d_bytes and c1.d2h_bytes == c0.d2h_bytes
    # none of the refused calls touched the scan or its outputs: they are still those of the host calls
    ref = m.aux()
    got = m.aux_tensor()
    for k in AUX:
        _same_bits(_np(got[k]).view(ref[k].dtype), ref[k], k)
    # the wrappers refuse before the call
    for t in (rec.cpu(), rec.float(), rec[:, :3].contiguous(), torch.empty((n, 8), dtype=torch.int32, device="cuda")[:, ::2]):
        with pytest.raises(ValueError):
            m.upload_scan_tensor(t, case.table, case.table_off, case.temporal_comp)
    m.close()


def test_counters_size_query_truncation_and_empty_scans():
    case = synth.make_case("counters", 6001, 50000, 3, 3)
    m = _model(case, "snapshot", True)
    st = torch.cuda.current_stream().cuda_stream
    n_tab = int(case.table_off[-1])
    c0 = m.counters()
    m.upload_scan_tensor(_records(case.pts), case.table, case.table_off, case.temporal_comp)
    c1 = m.counters()
    assert c1.kernel_launches - c0.kernel_launches == 1                       # the record check
    assert c1.h2d_bytes - c0.h2d_bytes == n_tab * capi.POSE_ENTRY.itemsize and c1.d2h_bytes == c0.d2h_bytes
    x, P = case.x_prop.copy(), case.P_prop.copy()
    m.update_iterated_dyn_share_modified(x, P, case.max_iter)
    ref = m.publish_frame_world(x, False)
    n = ref.shape[0]
    c2 = m.counters()
    m.aux_tensor()
    m.map_incremental_tensor(x, 0.5, True)
    full = m.publish_frame_world_tensor(x, False)
    c3 = m.counters()
    assert c3.kernel_launches - c2.kernel_launches == 3 and c3.d2h_bytes == c2.d2h_bytes and c3.h2d_bytes == c2.h2d_bytes
    _same_bits(_np(full), ref, "full")
    # size query and truncation: *n_out is the full count, at most cap points are written
    ps = x.pass_state()
    nn = C.c_uint32(0)
    assert m.lib.malio_world_register_device(m._h, C.byref(ps), 0, None, None, 0, C.byref(nn), st) == capi.OK and nn.value == n
    c4 = m.counters()
    assert c4.kernel_launches == c3.kernel_launches
    for cap in (1, n // 3, n - 1):
        out = torch.full((n, 4), -7.0, device="cuda")
        nn.value = 0
        assert m.lib.malio_world_register_device(m._h, C.byref(ps), 0, None, out.data_ptr(), cap, C.byref(nn), st) == capi.OK
        o = _np(out)
        assert nn.value == n
        _same_bits(o[:cap], ref[:cap], cap)
        assert np.all(o[cap:] == -7.0)
    # an empty scan: nothing is launched by the upload or by the output calls
    c5 = m.counters()
    m.upload_scan_tensor(torch.empty((0, 4), dtype=torch.int32, device="cuda"), case.table, case.table_off, case.temporal_comp)
    c6 = m.counters()
    assert c6.kernel_launches == c5.kernel_launches and c6.h2d_bytes - c5.h2d_bytes == n_tab * capi.POSE_ENTRY.itemsize
    ok, _, _, _ = m.h_share_model(case.x_prop, True)
    assert not ok
    c7 = m.counters()
    aux = m.aux_tensor()
    cls, w = m.map_incremental_tensor(x, 0.5, True)
    reg = m.publish_frame_world_tensor(x, False)
    c8 = m.counters()
    assert c8.kernel_launches == c7.kernel_launches
    assert all(t.shape[0] == 0 for t in list(aux.values()) + [cls, w, reg])
    m.close()


def test_knn_tensor_shares_the_scan_buffers_and_hands_its_fault_to_the_upload():
    from test_gpu_knn_device import _understated_chain
    case = synth.case_C1()
    m = _model(case, "snapshot", True)
    m.upload_scan_tensor(_records(case.pts), case.table, case.table_off, case.temporal_comp)
    m.h_share_model(case.x_prop, True)
    m.knn_tensor(torch.from_numpy(case.map_xyz[:100]).cuda())
    with pytest.raises(capi.MalioError) as e:
        m.h_share_model(case.x_prop, True)
    assert e.value.status == capi.ERR_STATE
    m.close()
    _, understated = _understated_chain()
    a = plugin.MeasurementModel(1, knn_cell_size=-1.0)
    a.upload_map(understated)
    a.knn_tensor(torch.tensor([[120.0, 0.0, 0.0], [120.5, 0.25, 0.0]], device="cuda"))   # the guard fires after the call returned
    with pytest.raises(capi.MalioError) as e:
        a.upload_scan_tensor(_records(case.pts), case.table, case.table_off, case.temporal_comp)
    assert e.value.status == capi.ERR_TREE_TOO_DEEP
    a.close()
