"""The device-memory entry points (malio_knn_device, malio_map_build_device, malio_map_add_points_device) through their torch
wrappers: bit-identical to the host-pointer calls, ordered on the caller's stream without a host wait, argument errors caught
before anything is launched, and the traversal fault handed to the next call on the handle."""
import math
import time

import numpy as np
import pytest
import torch

import helpers as H
import pyoracle as po
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32


def _same_as_host(m, q_np):
    """knn_tensor(q) against Nearest_Search(q) on the same handle, bit for bit; returns the host lists."""
    q = torch.from_numpy(np.ascontiguousarray(q_np, F)).cuda()
    idx, d2 = m.knn_tensor(q)
    torch.cuda.current_stream().synchronize()
    hi, hd, _ = m.Nearest_Search(q_np)
    assert idx.dtype == torch.int32 and d2.dtype == torch.float32 and tuple(idx.shape) == (q_np.shape[0], capi.K)
    di, dd = idx.cpu().numpy().view(np.uint32), d2.cpu().numpy()
    assert np.array_equal(di, hi)
    assert np.array_equal(dd.view(np.uint32), hd.view(np.uint32))
    return hi, hd


@pytest.mark.parametrize("sort", [True, False])
def test_c5_shape_equals_host_call(sort):
    xyz, q = synth.knn_microbench(M=1_000_000, Q=200_000)
    snap = plugin.build_static_snapshot(xyz)
    m = plugin.MeasurementModel(1, sort_queries=sort)
    m.upload_map(snap)
    c0 = m.counters()
    _same_as_host(m, q)
    c1 = m.counters()
    assert c1.knn_launches - c0.knn_launches == 2 and c1.knn_queries - c0.knn_queries == 2 * q.shape[0]
    assert c1.h2d_bytes - c0.h2d_bytes == 12 * q.shape[0] and c1.d2h_bytes - c0.d2h_bytes == 40 * q.shape[0]   # the host call's only
    m.close()


@pytest.mark.parametrize("sort", [True, False])
def test_live_churned_snapshot_and_edge_queries(sort):
    case = synth.make_case("kd", 2000, 200000, 3, 3)
    snap, _ = H.snapshot_for(case, churn=True)
    m = plugin.MeasurementModel(case.n_lidar, sort_queries=sort, params=case.params)
    m.upload_map(snap)
    rng = np.random.default_rng(3)
    near = case.map_xyz[rng.integers(0, case.map_xyz.shape[0], 20000)] + rng.normal(0, 0.3, (20000, 3)).astype(F)
    far = np.array([[1e4, 1e4, 1e4], [-3e5, 0, 0], [0, 0, 2e6]], F)
    dup = np.repeat(near[:5], 40, axis=0)
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan, np.nan, np.nan]], F)
    q = np.concatenate([near, far, dup, bad, case.map_xyz[:500]]).astype(F)
    hi, hd = _same_as_host(m, q)
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, near)
    assert np.array_equal(hi[:20000].astype(np.int64), o_idx.astype(np.int64)) and np.array_equal(hd[:20000], o_d2)
    m.close()


def test_query_counts_zero_one_and_buffer_growth():
    case = synth.case_C1()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    m = plugin.MeasurementModel(1)
    m.upload_map(snap)
    rng = np.random.default_rng(4)
    mk = lambda n: (case.map_xyz[rng.integers(0, case.map_xyz.shape[0], n)] + rng.normal(0, 0.2, (n, 3))).astype(F)
    _same_as_host(m, mk(1000))                    # sizes the per-point buffers for ~2k points
    _same_as_host(m, mk(1))
    c0 = m.counters()
    idx, d2 = m.knn_tensor(torch.empty((0, 3), dtype=torch.float32, device="cuda"))
    assert tuple(idx.shape) == (0, capi.K) and tuple(d2.shape) == (0, capi.K)
    c1 = m.counters()
    assert c1.kernel_launches == c0.kernel_launches and c1.knn_launches == c0.knn_launches
    # the device call grows the buffers (the host call only runs after it) while an earlier device call is still enqueued
    # behind a long kernel on the caller's stream
    small, big = mk(500), mk(300_000)
    qs, qb = torch.from_numpy(small).cuda(), torch.from_numpy(big).cuda()
    torch.cuda._sleep(50_000_000)
    i_s, d_s = m.knn_tensor(qs)
    i_b, d_b = m.knn_tensor(qb)
    torch.cuda.current_stream().synchronize()
    for (ti, td), q in (((i_s, d_s), small), ((i_b, d_b), big)):
        hi, hd, _ = m.Nearest_Search(q)
        assert np.array_equal(ti.cpu().numpy().view(np.uint32), hi) and np.array_equal(td.cpu().numpy(), hd)
    m.close()


def test_device_map_mode_with_exact_ties():
    rng = np.random.default_rng(5)
    x = np.round(rng.uniform(0, 40, (60000, 3)) * 4).astype(F) / F(4)    # a 0.25 lattice: many exactly tied distances
    x[:, 2] = np.round(rng.uniform(0, 3, 60000) * 4).astype(F) / F(4)
    q = np.concatenate([x[rng.integers(0, len(x), 4000)], x[:2000] + F(0.125),
                        rng.uniform(0, 40, (4000, 3)).astype(F)]).astype(F)
    for sort in (True, False):
        m2 = plugin.MeasurementModel(1, sort_queries=sort)
        m2.map_build(x, np.full(len(x), 0.001, F))
        m2.map_add_points(x[:3000], np.full(3000, 0.002, F))          # exact duplicates in later slots
        c0 = m2.counters().knn_tie_queries
        qt = torch.from_numpy(q).cuda()
        idx, d2 = m2.knn_tensor(qt)
        c1 = m2.counters().knn_tie_queries                                # folds the device call's statistics in
        hi, hd, _ = m2.Nearest_Search(q)
        c2 = m2.counters().knn_tie_queries
        assert np.array_equal(idx.cpu().numpy().view(np.uint32), hi) and np.array_equal(d2.cpu().numpy(), hd)
        assert c1 - c0 == c2 - c1 > 0, (c0, c1, c2)
        m2.close()


def test_stream_order_without_host_wait():
    case = synth.case_C1()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    m = plugin.MeasurementModel(1)
    m.upload_map(snap)
    rng = np.random.default_rng(6)
    q_np = (case.map_xyz[rng.integers(0, case.map_xyz.shape[0], 50000)] + rng.normal(0, 0.2, (50000, 3))).astype(F)
    hi, hd, _ = m.Nearest_Search(q_np)
    src = torch.from_numpy(q_np).cuda()
    m.knn_tensor(src)                                     # same size once: the timed call below grows nothing
    m.counters()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        q = torch.zeros_like(src)                         # zeros until the side stream has passed the sleep
        torch.cuda._sleep(400_000_000)                    # ~0.2 s at 1.98 GHz
        q.copy_(src)
        t0 = time.perf_counter()
        idx, d2 = m.knn_tensor(q)
        dt = time.perf_counter() - t0
        pending = not side.query()
        total = d2.double().sum()                         # a reduction on the side stream reads the lists
        found = (idx >= 0).sum()
    side.synchronize()
    assert pending
    assert dt < 0.05, dt
    assert math.isclose(total.item(), float(hd.astype(np.float64).sum()), rel_tol=1e-12)   # (summation orders differ)
    assert found.item() == int((hi != 0xFFFFFFFF).sum())
    assert np.array_equal(idx.cpu().numpy().view(np.uint32), hi)
    m.close()


def test_map_build_and_add_from_tensors_equal_host_arrays():
    case = synth.make_case("mb", 3000, 120000, 3, 3, varied_map_cov=True)
    rng = np.random.default_rng(7)
    n = case.map_xyz.shape[0]
    ids = rng.permutation(n).astype(np.int32)
    add = (case.map_xyz[rng.integers(0, n, 80000)] + rng.normal(0, 0.3, (80000, 3))).astype(F)   # above the 65536 bounce size
    add_ny = rng.uniform(0.0005, 0.01, 80000).astype(F)
    small = (case.map_xyz[rng.integers(0, n, 2000)] + rng.normal(0, 0.3, (2000, 3))).astype(F)
    small_ids = np.arange(2000, dtype=np.int32) + 10_000_000
    host = plugin.MeasurementModel(case.n_lidar, params=case.params)
    dev = plugin.MeasurementModel(case.n_lidar, params=case.params)
    host.map_build(case.map_xyz, case.map_normal_y, ids)
    host.map_add_points(add, add_ny)
    host.map_add_points(small, np.full(2000, 0.003, F), small_ids)
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dev.map_build_tensor(cuda(case.map_xyz), cuda(case.map_normal_y), cuda(ids))
    dev.map_add_points_tensor(cuda(add), cuda(add_ny))
    dev.map_add_points_tensor(cuda(small), cuda(np.full(2000, 0.003, F)), cuda(small_ids))
    y70 = float(np.quantile(np.concatenate([case.map_xyz[:, 1], add[:, 1], small[:, 1]]), 0.7))
    for m in (host, dev):                                # most slots dead: the commit compacts
        m.map_delete_boxes([[-1e9, -1e9, -1e9, 1e9, y70, 1e9]])
    a, b = host.map_download(), dev.map_download()
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    assert host.counters().map_compactions == dev.counters().map_compactions == 1
    for m in (host, dev):
        m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    ga, gb = host.h_share_model(case.x_prop, True), dev.h_share_model(case.x_prop, True)
    assert ga[0] == gb[0] and np.array_equal(ga[1], gb[1]) and np.array_equal(ga[2], gb[2])
    xa, Pa = case.x_prop.copy(), case.P_prop.copy()
    xb, Pb = case.x_prop.copy(), case.P_prop.copy()
    host.update_iterated_dyn_share_modified(xa, Pa, case.max_iter)
    dev.update_iterated_dyn_share_modified(xb, Pb, case.max_iter)
    assert np.array_equal(synth.state_to_vec(xa, case.n_lidar), synth.state_to_vec(xb, case.n_lidar)) and np.array_equal(Pa, Pb)
    # the empty build is malio_map_build's empty build
    dev.map_build_tensor(torch.empty((0, 3), device="cuda"), torch.empty(0, device="cuda"))
    assert dev.map_info() == (0, 0)
    host.close()
    dev.close()


def test_knn_shares_the_scan_buffers():
    case = synth.case_C1()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    m = H.make_model(case, snap)
    m.h_share_model(case.x_prop, True)
    m.knn_tensor(torch.from_numpy(case.map_xyz[:100]).cuda())
    with pytest.raises(capi.MalioError) as e:
        m.h_share_model(case.x_prop, True)
    assert e.value.status == capi.ERR_STATE
    m.close()


def test_argument_errors_launch_nothing():
    case = synth.case_C1()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    m = plugin.MeasurementModel(1)
    lib, h = m.lib, m._h
    n = 64
    dq = torch.from_numpy(case.map_xyz[:n]).cuda()
    di = torch.empty((n, capi.K), dtype=torch.int32, device="cuda")
    dd = torch.empty((n, capi.K), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    # no map yet
    c0 = m.counters()
    assert lib.malio_knn_device(h, dq.data_ptr(), n, di.data_ptr(), dd.data_ptr(), stream) == capi.ERR_STATE
    assert lib.malio_map_add_points_device(h, dq.data_ptr(), dd.data_ptr(), None, n, stream) == capi.ERR_STATE
    m.upload_map(snap)
    c0 = m.counters()
    hq = np.ascontiguousarray(case.map_xyz[:n])
    pq = torch.from_numpy(hq).pin_memory()
    bad = {"host": hq.ctypes.data, "pinned": pq.data_ptr(), "null": None, "misaligned": dq.data_ptr() + 2}
    for what, p in bad.items():
        assert lib.malio_knn_device(h, p, n, di.data_ptr(), dd.data_ptr(), stream) == capi.ERR_INVALID_ARG, what
        assert lib.malio_knn_device(h, dq.data_ptr(), n, p, dd.data_ptr(), stream) == capi.ERR_INVALID_ARG, what
        assert lib.malio_knn_device(h, dq.data_ptr(), n, di.data_ptr(), p, stream) == capi.ERR_INVALID_ARG, what
        assert lib.malio_map_build_device(h, p, dd.data_ptr(), None, n, stream) == capi.ERR_INVALID_ARG, what
        assert lib.malio_map_add_points_device(h, dq.data_ptr(), p, None, n, stream) == capi.ERR_INVALID_ARG, what
    assert lib.malio_map_build_device(h, dq.data_ptr(), dd.data_ptr(), hq.ctypes.data, n, stream) == capi.ERR_INVALID_ARG
    if torch.cuda.device_count() > 1:
        other = torch.from_numpy(hq).to("cuda:1")
        assert lib.malio_knn_device(h, other.data_ptr(), n, di.data_ptr(), dd.data_ptr(), stream) == capi.ERR_INVALID_ARG
        assert lib.malio_map_build_device(h, other.data_ptr(), dd.data_ptr(), None, n, stream) == capi.ERR_INVALID_ARG
    assert lib.malio_knn_device(h, None, 0, None, None, stream) == capi.OK
    c1 = m.counters()
    assert c1.kernel_launches == c0.kernel_launches and c1.knn_launches == c0.knn_launches
    # the map is still the snapshot: nothing was built
    assert lib.malio_map_info(h, None, None) == capi.ERR_STATE
    # the torch wrappers refuse before the call
    for t in (dq.cpu(), dq.double(), dq.t(), dq[:, :2].contiguous(), torch.empty((n, 6), device="cuda")[:, ::2],
              torch.empty((n, 3), device="cuda:1" if torch.cuda.device_count() > 1 else "cpu")):
        with pytest.raises(ValueError):
            m.knn_tensor(t)
    m.close()


def _understated_chain():
    # the construction of test_gpu_more.py::test_traversal_fault_stays_with_its_handle: every left leaf is closer to the query
    # than the spine points seen so far, so the traversal stack grows with the real depth, not the declared one
    from test_gpu_more import _chain_snapshot
    pts = []
    for k in range(60):
        pts.append((2.0 * k, 0.0, 0.0))
        pts.append((2.0 * k + 1, 1000.0, 0.0))
    deep = _chain_snapshot(np.array(pts, F))
    return deep, plugin.MapSnapshot(deep.nodes, deep.node_cov, deep.node_ids, 8)


def test_deferred_fault_reaches_the_next_call_and_stays_with_its_handle():
    deep, understated = _understated_chain()
    q_np = np.array([[120.0, 0.0, 0.0], [120.5, 0.25, 0.0]], F)
    case = synth.case_C1()
    snap_b = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    a = plugin.MeasurementModel(1, knn_cell_size=-1.0)
    b = plugin.MeasurementModel(1, knn_cell_size=-1.0)
    b.upload_map(snap_b)
    a.upload_map(understated)
    q = torch.from_numpy(q_np).cuda()
    a.knn_tensor(q)                                      # enqueued: the guard fires on the device after the call returned
    qb = case.map_xyz[::97] + F(0.05)
    _same_as_host(b, qb)                                 # the other handle is untouched, even while A's report is pending
    with pytest.raises(capi.MalioError) as e:
        a.counters()                                     # the next call on A reports the fault instead of running
    assert e.value.status == capi.ERR_TREE_TOO_DEEP
    with pytest.raises(capi.MalioError) as e:
        a.knn_tensor(q)                                  # and the fault stays with the map, as for malio_knn
    assert e.value.status == capi.ERR_TREE_TOO_DEEP
    with pytest.raises(capi.MalioError) as e:
        a.Nearest_Search(q_np)
    assert e.value.status == capi.ERR_TREE_TOO_DEEP
    _same_as_host(b, qb)
    a.upload_map(deep)                                   # the true depth clears it
    idx, d2 = _same_as_host(a, q_np)
    o_idx, o_d2, _, _ = po.knn_snapshot(deep.nodes, deep.node_cov, q_np)
    assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)) and np.array_equal(d2, o_d2)
    a.counters()
    a.close()
    b.close()
