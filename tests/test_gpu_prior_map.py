"""Localization in a prior map on the device (malio_prior_map_*), against the restated lasermap_fov_segment
(tests/prior_map_ref.py):
  - the live set after every window call is prior ∩ cube, by id, along a scripted drive (±x, ±y, z, diagonals, staying put
    without enqueueing work, a jump past the cube, a cube without a prior point), with points on the cube faces, tiles across
    the faces, a prior at ±1e5 m, an empty prior and a load that replaces the previous one;
  - k-NN on the window equals a brute-force search over prior ∩ cube (ties in slot order) and the real ikd-Tree's distances;
  - malio_ieskf_update on the window is bit-identical to the same update on a handle built with malio_map_build from the
    window's points in slot order;
  - scans rendered from a corridor prior of 4 km localize through a sliding window, without any map insert;
  - refusals leave the prior and the window as they were, the device load's stream order and pointer checks, identical slots
    from two runs, and device bytes that stay flat over 100 slides."""
import ctypes as C
from dataclasses import replace

import numpy as np
import pytest
import torch

import np_mapops as nm
import prior_map_ref as R
import pyoracle as po
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
CUBE, DET = 40.0, 5.0          # thr 7.5 m, mov_dist 11.25 m (R.DRIVE); a tile of 25 m straddles most faces


def _prior(rng, n, half=80.0, offset=0.0):
    xyz = np.column_stack([rng.uniform(-half, half, n), rng.uniform(-half, half, n), rng.uniform(-20, 20, n)])
    return (xyz + [offset, offset, 0.0]).astype(F)


def _face_points(cube):
    """Points on the six faces of a cube, one ulp either side, and on its corners."""
    c = np.asarray(cube, F)
    mid = [F((np.float64(c[a]) + np.float64(c[3 + a])) / 2) for a in range(3)]
    pts = []
    for a in range(3):
        for v in (c[a], c[3 + a]):
            for w in (np.nextafter(v, F(-np.inf)), v, np.nextafter(v, F(np.inf))):
                p = list(mid); p[a] = w; pts.append(p)
    pts += [list(c[:3]), list(c[3:])]
    return np.array(pts, F)


def _ids(m):
    return np.sort(m.map_download()["ids"]) if m.map_info()[0] else np.zeros(0, np.int32)


def _drive(m, prior, offset, want_slots=False):
    """Runs DRIVE on m and on the restatement; checks the live set after every call.  Returns the slot-order ids per step."""
    w = R.Window(prior, CUBE, DET)
    out = []
    moves = 0
    for k, d in enumerate(R.DRIVE):
        pos = R.drive_pos(w, d, (offset, offset, 0.0))
        before = set(w.live().tolist()) if w.cube is not None else set()
        c0 = m.counters().kernel_launches
        init, moved, slabs = w.step(pos)
        rep = m.prior_map_window(pos, CUBE, DET)
        moves += moved
        live = w.live()
        assert rep["initialized"] == init and rep["moved"] == moved, k
        assert np.array_equal(rep["cube"], w.cube), k
        assert np.array_equal(rep["boxes"], slabs), k
        assert rep["n_live"] == len(live), (k, rep["n_live"], len(live))
        if moved:
            assert rep["n_killed"] == len(before - set(live.tolist())), k
            assert rep["n_entered"] == len(set(live.tolist()) - before), k
        if not init and not moved:
            assert m.counters().kernel_launches == c0, k        # nothing enqueued
        assert np.array_equal(_ids(m), np.sort(live)), k
        if want_slots:
            out.append(m.map_download()["ids"].copy())
    assert moves >= 12
    return out


@pytest.mark.parametrize("offset", [0.0, 1e5, -1e5])
def test_live_set_along_a_scripted_drive(offset):
    rng = np.random.default_rng(11)
    prior = _prior(rng, 30000, offset=offset)
    prior = np.concatenate([prior, _face_points(R.init_cube((offset, offset, 0.0), CUBE))])
    m = plugin.MeasurementModel(1)
    m.prior_map_load(prior)
    assert m.prior_map_info()["n_points"] == len(prior)
    _drive(m, prior, offset)
    m.close()


def test_empty_prior_empty_cube_and_a_replacing_load():
    rng = np.random.default_rng(12)
    m = plugin.MeasurementModel(1)
    lib, h = m.lib, m._h
    rep = capi.WindowReport()
    pos = np.zeros(3)
    assert lib.malio_prior_map_window(h, capi.ptr(pos), CUBE, DET, C.byref(rep)) == capi.ERR_STATE
    q = torch.from_numpy(rng.uniform(-10, 10, (100, 3)).astype(F)).cuda()
    m.prior_map_load(np.zeros((0, 3), F))                             # n = 0
    r = m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
    assert r["initialized"] and r["n_live"] == 0 and m.map_info()[0] == 0
    idx, d2 = m.knn_tensor(q)
    assert torch.all(idx == -1) and torch.all(torch.isinf(d2))
    prior = _prior(rng, 5000)
    m.prior_map_load(prior)                                           # replaces the empty prior, ends the window
    r = m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
    assert r["initialized"] and np.array_equal(_ids(m), np.flatnonzero(R.in_box(prior, R.init_cube((0, 0, 0), CUBE))))
    r = m.prior_map_window((500.0, 0.0, 0.0), CUBE, DET)              # far away: nothing moves (the reference's rule)
    assert not r["moved"]
    m.prior_map_load(prior + F(1000.0))                               # a prior without a point in the cube
    r = m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
    assert r["initialized"] and r["n_live"] == 0
    idx, d2 = m.knn_tensor(q)
    assert torch.all(idx == -1)
    # malio_map_build ends the window: the next call builds it afresh
    m.prior_map_load(prior)
    m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
    m.map_build(prior[:10], np.full(10, 0.001, F))
    r = m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
    assert r["initialized"]
    m.prior_map_clear()
    assert lib.malio_prior_map_window(h, capi.ptr(pos), CUBE, DET, C.byref(rep)) == capi.ERR_STATE
    m.close()


def test_knn_on_the_window_equals_brute_force_and_the_reference_tree():
    rng = np.random.default_rng(13)
    prior = _prior(rng, 40000)
    # exact duplicates: distance ties, broken by slot order on the device and by the brute force alike
    prior = np.concatenate([prior, prior[:300]])
    m = plugin.MeasurementModel(1)
    m.prior_map_load(prior)
    w = R.Window(prior, CUBE, DET)
    tree = po.RefTree(box_length=0.5) if po.ref_available() else None
    before = None
    for k, d in enumerate(R.DRIVE[:11]):
        pos = R.drive_pos(w, d)
        init, moved, slabs = w.step(pos)
        m.prior_map_window(pos, CUBE, DET)
        live = w.live()
        mp = m.map_download()
        q = np.concatenate([prior[live[rng.integers(0, len(live), 1500)]] + rng.normal(0, 0.5, (1500, 3)),
                            rng.uniform(w.cube[:3] - 5, w.cube[3:] + 5, (500, 3))]).astype(F)
        idx, d2 = m.knn_tensor(torch.from_numpy(q).cuda())
        ri, rd, _ = nm.knn_bruteforce(mp["xyz"], mp["slots"], q)
        assert np.array_equal(idx.cpu().numpy().view(np.uint32), ri), k
        assert d2.cpu().numpy().tobytes() == rd.tobytes(), k
        if tree is not None:
            if init:
                tree.build(prior[live], np.full(len(live), 0.001, F), live.astype(np.int32))
            elif moved:
                tree.delete_boxes(slabs)
                enter = np.setdiff1d(live, before)
                tree.add_points(prior[enter], np.full(len(enter), 0.001, F), enter.astype(np.int32), downsample=False)
            tree.wait_rebuild()
            if k in (0, 3, 6, 10):
                _, td, _, found = tree.knn(q)
                full = found == capi.K
                assert np.array_equal(td[full], d2.cpu().numpy()[full]), k
        before = live
    if tree is not None:
        tree.close()
    m.close()


def test_ieskf_update_on_the_window_is_bit_identical_to_a_built_map():
    case = synth.case_C1()
    a = plugin.MeasurementModel(case.n_lidar, params=case.params)
    a.prior_map_load(case.map_xyz, case.map_normal_y)
    r = a.prior_map_window(case.x_prop, 60.0, 10.0)
    assert r["initialized"] and 0 < r["n_live"] < len(case.map_xyz)
    mp = a.map_download()
    b = plugin.MeasurementModel(case.n_lidar, params=case.params)
    b.map_build(mp["xyz"], mp["normal_y"], mp["ids"])
    res = []
    for m in (a, b):
        m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
        x, P = case.x_prop.copy(), case.P_prop.copy()
        rep = m.update_iterated_dyn_share_modified(x, P, case.max_iter)
        assert rep.n_eff_last > 0
        res.append((synth.state_to_vec(x, case.n_lidar).tobytes(), P.tobytes(), rep.passes))
    assert res[0] == res[1]
    a.close(); b.close()


def _corridor(rng, length=4000.0, per_site=12000):
    half = length / 2 + 100.0
    sites = np.arange(-length / 2, length / 2 + 1, 50.0)
    return np.concatenate([synth.sample_surfaces(per_site, (x, 0.0), 40.0, half, rng) for x in sites]).astype(F), half


def test_localization_through_a_sliding_window_over_a_corridor():
    """A 4 km corridor (ground and the street grid's walls); 21 scans 20 m apart rendered from the prior at known poses.  Per
    scan: the window (a 200 m cube) at the predicted pose, then the IESKF update, no map insert.  Every scan point's neighbours
    lie inside the cube, so each estimate must equal, bit for bit, the estimate against the whole corridor built as one map
    (malio_map_build widens its cells for it; it does not refuse a few km).  Against the truth: the prediction is off by 0.1 m and
    0.5 deg; in this scene the update lands within 0.1 m and 0.25 deg of the truth, window or whole map alike, and the error does
    not grow along the drive (each scan is localized against the fixed prior, nothing accumulates)."""
    rng = np.random.default_rng(14)
    prior, half = _corridor(rng)
    base = synth.make_case("corridor", 6000, 1000, 1, 4)
    m = plugin.MeasurementModel(1, params=base.params)
    m.prior_map_load_tensor(torch.from_numpy(prior).cuda(), torch.full((len(prior),), 0.001, device="cuda"))
    assert m.prior_map_info()["n_points"] == len(prior)
    full = plugin.MeasurementModel(1, params=base.params)
    full.map_build(prior, np.full(len(prior), 0.001, F))
    extq = [np.array(base.x_true.ext[0].q[:])]
    extt = [np.array(base.x_true.ext[0].t[:])]
    rot = np.array(base.x_true.rot[:])
    slides = 0
    live_max = 0
    rs = np.random.default_rng(15)
    for k in range(21):
        pos = np.array([20.0 * k, 0.0, 1.8])
        xt = synth.make_state(pos, rot, extq, extt)
        pw = synth.sample_surfaces(6000, pos[:2], 40.0, half, rs) + rs.normal(0, 0.02, (6000, 3))
        case = synth.with_scan(replace(base, x_true=xt), pw, seed=k)
        xp = synth.make_state(pos + synth.rand_unit(rs) * 0.1, synth.q_mul(rot, synth.q_exp(synth.rand_unit(rs) * np.deg2rad(0.5))),
                              extq, extt)
        r = m.prior_map_window(xp, 200.0, 30.0)
        slides += r["moved"]
        live_max = max(live_max, r["n_live"])
        res = []
        for h in (m, full):
            h.upload_scan(case.pts, case.table, case.table_off, None)
            x, P = xp.copy(), synth.init_P(case.n_dof)
            rep = h.update_iterated_dyn_share_modified(x, P, 4)
            assert rep.n_eff_last > 1000, k
            res.append((synth.state_to_vec(x, 1).tobytes(), P.tobytes()))
        assert res[0] == res[1], k
        v = np.frombuffer(res[0][0], np.float64)   # pos, rot (w, x, y, z), ...
        err = np.linalg.norm(v[:3] - pos)
        dq = synth.q_mul(synth.q_conj(v[3:7]), rot)
        ang = np.rad2deg(2 * np.arcsin(min(1.0, np.linalg.norm(dq[1:]))))
        assert err < 0.1 and ang < 0.25, (k, err, ang)
    assert slides >= 2
    assert live_max < len(prior) // 5          # the window holds a small part of the corridor
    m.close(); full.close()


def test_refusals_keep_the_prior_and_the_window():
    rng = np.random.default_rng(16)
    prior = _prior(rng, 5000)
    m = plugin.MeasurementModel(1)
    m.prior_map_load(prior)
    m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
    ids0 = _ids(m)
    info0 = m.prior_map_info()
    for bad, status in ((np.nan, capi.ERR_INVALID_ARG), (np.inf, capi.ERR_INVALID_ARG), (1e8, capi.ERR_CAPACITY), (-1e8, capi.ERR_CAPACITY)):
        p = prior.copy()
        p[1234, 1] = bad
        with pytest.raises(capi.MalioError) as e:
            m.prior_map_load(p)
        assert e.value.status == status
        assert m.prior_map_info()["n_points"] == info0["n_points"]
        r = m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
        assert not r["initialized"] and not r["moved"]
        assert np.array_equal(_ids(m), ids0)
    for args in (((np.nan, 0, 0), CUBE, DET), ((0, 0, 0), 0.0, DET), ((0, 0, 0), np.inf, DET), ((0, 0, 0), CUBE, -1.0)):
        with pytest.raises(capi.MalioError) as e:
            m.prior_map_window(*args)
        assert e.value.status == capi.ERR_INVALID_ARG
    assert not m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)["initialized"]
    m.close()


def test_device_load_stream_order_and_pointer_refusals():
    rng = np.random.default_rng(17)
    prior = _prior(rng, 20000)
    m = plugin.MeasurementModel(1)
    src = torch.from_numpy(prior).cuda()
    ny = torch.full((len(prior),), 0.001, device="cuda")
    ids = torch.arange(len(prior), dtype=torch.int32, device="cuda") * 3
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        xyz = torch.zeros_like(src)                      # zeros until the side stream has passed the sleep
        torch.cuda._sleep(200_000_000)
        xyz.copy_(src)
        m.prior_map_load_tensor(xyz, ny, ids)
        xyz.zero_()                                      # after the call in stream order: the load has read the points
    side.synchronize()
    r = m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)
    want = np.flatnonzero(R.in_box(prior, R.init_cube((0, 0, 0), CUBE)))
    assert r["n_live"] == len(want) and np.array_equal(_ids(m), np.sort(want * 3))
    lib, h = m.lib, m._h
    stream = torch.cuda.current_stream().cuda_stream
    c0 = m.counters()
    n = 64
    hq = np.ascontiguousarray(prior[:n])
    pq = torch.from_numpy(hq).pin_memory()
    bad = {"host": hq.ctypes.data, "pinned": pq.data_ptr(), "null": None, "misaligned": src.data_ptr() + 2}
    for what, p in bad.items():
        assert lib.malio_prior_map_load_device(h, p, ny.data_ptr(), None, n, stream) == capi.ERR_INVALID_ARG, what
        assert lib.malio_prior_map_load_device(h, src.data_ptr(), p, None, n, stream) == capi.ERR_INVALID_ARG, what
        if p is not None:
            assert lib.malio_prior_map_load_device(h, src.data_ptr(), ny.data_ptr(), p, n, stream) == capi.ERR_INVALID_ARG, what
    if torch.cuda.device_count() > 1:
        other = torch.from_numpy(hq).to("cuda:1")
        assert lib.malio_prior_map_load_device(h, other.data_ptr(), ny.data_ptr(), None, n, stream) == capi.ERR_INVALID_ARG
    c1 = m.counters()
    assert c1.kernel_launches == c0.kernel_launches
    assert m.prior_map_info()["n_points"] == len(prior)
    assert not m.prior_map_window((0.0, 0.0, 0.0), CUBE, DET)["initialized"]
    for t in (src.cpu(), src.double(), src[:, :2].contiguous()):
        with pytest.raises(ValueError):
            m.prior_map_load_tensor(t, ny)
    m.close()


def test_two_runs_give_identical_slots():
    rng = np.random.default_rng(18)
    prior = _prior(rng, 30000)
    runs = []
    for _ in range(2):
        m = plugin.MeasurementModel(1)
        m.prior_map_load(prior)
        runs.append(_drive(m, prior, 0.0, want_slots=True))
        m.close()
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


def test_device_bytes_stay_flat_over_100_slides():
    rng = np.random.default_rng(19)
    prior = _prior(rng, 100000, half=120.0)
    m = plugin.MeasurementModel(1)
    m.prior_map_load(prior)
    w = R.Window(prior, CUBE, DET)
    sizes = []
    moves = 0
    for k in range(111):
        pos = R.drive_pos(w, (0, 0, 0) if k == 0 else ((-15, 0, 0) if (k // 4) % 2 else (15, 0, 0)))   # four slides each way
        w.step(pos)
        r = m.prior_map_window(pos, CUBE, DET)
        moves += r["moved"]
        if k >= 10:
            sizes.append(m.prior_map_info()["device_bytes"])
    assert moves >= 100
    assert len(set(sizes)) == 1, sizes[:3]
    assert np.array_equal(_ids(m), np.sort(w.live()))
    m.close()
