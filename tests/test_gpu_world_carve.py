"""Clearing moving objects out of the voxel map on the device (malio_world_voxel_accumulate_carve and the kept download /
save), exactly against tests/carve_ref.py:
  - (hit, miss) of every voxel after every scan of a 20-scan street drive, L = 1 and L = 3, with plain accumulate calls mixed
    in, a table regrowth in the middle and a clearing save; the centroids byte-identical to a handle that only accumulates;
  - the kept download and the kept PCD against the unfiltered download minus the rule's voxels; the kept file as a prior holds
    no point of the car's trail; two runs give the same bytes;
  - every refusal leaves centroids, counters and entry count as they were; the device-memory contract of the two downloads;
    device bytes flat over 300 carved scans.
Clouds are planted through malio_undistort with control points that end before the scan (every point keeps its raw
coordinates) and registered with the scan's state, as tests/test_gpu_world_voxel.py does."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import carve_ref as CR
import world_ref as W
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
Q_ID = np.array([1.0, 0.0, 0.0, 0.0])


def _plant(m, slot, xyz):
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    ctrl_t = np.array([-10.0, -9.0, -8.0, -7.0])
    m.undistort(slot, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), ctrl_t, np.tile(np.eye(4), (4, 1, 1)), np.zeros(0), -1)


def _origins(state, L):
    """Each slot's origin: body_to_world of (0, 0, 0), no upload so far (identity temporal compensation)."""
    tc = np.zeros(max(L - 1, 1), capi.RIGID)
    tc["q"][:, 0] = 1.0
    return np.concatenate([W.register_world(state, tc, np.zeros((1, 3), F), l, 0.0)[:, :3] for l in range(L)])


def _same(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.shape, b.shape)
    assert a.tobytes() == b.tobytes(), what


def _cent(m, keep=None):
    return m.voxel_map_tensor(keep).cpu().numpy()


def _evid(m):
    return m.voxel_map_evidence_tensor().cpu().numpy().view(np.uint32)


CARVE = dict(max_range=60.0, end_margin=0.5)
PLAIN = (4, 9)         # scans folded with the plain accumulate
GROW = 10              # a scan with 70 000 more points: the table regrows
CLEAR = 14             # a clearing kept save after this scan


def _drive(L, tmp_path, check=True):
    st = synth.Street()
    leaf = 0.5
    m, m2 = plugin.MeasurementModel(L), plugin.MeasurementModel(L)
    ref = CR.CarveMapRef()
    tags = np.arange(L, dtype=F)
    rng = np.random.default_rng(L)
    out = []
    for k in range(20):
        sc = synth.street_scan(st, k, L=L, spin=(16, 128), cone=300)
        body = list(sc["body"])
        if k == GROW:
            body[0] = np.concatenate([body[0], rng.uniform([-5, -9, -2], [60, 9, 12], (70000, 3)).astype(F)])
        for mm in (m, m2):
            for l in range(L):
                _plant(mm, l, body[l])
        s = sc["state"]
        d = m.publish_frame_world(s, True, tags)
        cap0 = m.voxel_map_info()["capacity"]
        if k in PLAIN:
            n = m.voxel_map_accumulate(s, tags, leaf)
            assert n == ref.accumulate(d, leaf)
        else:
            n = m.voxel_map_accumulate(s, tags, leaf, carve=CARVE)
            assert n == ref.accumulate_carve(d, [b.shape[0] for b in body], _origins(s, L), leaf, **CARVE)
        assert m2.voxel_map_accumulate(s, tags, leaf) == n
        if k == GROW:
            assert m.voxel_map_info()["capacity"] > cap0
        if check:
            c = _cent(m)
            _same(c, _cent(m2), ("accumulate", k))
            _same(c, ref.centroids(), ("restatement", k))
            _same(_evid(m), ref.evidence(), ("evidence", k))
        if k == CLEAR:
            mask = ref.kept_mask(2, 1.0)
            kept = _cent(m, dict(min_miss=2, max_miss_per_hit=1.0))
            _same(kept, ref.centroids()[mask], "kept before the clear")
            p = tmp_path / f"kept_{L}.pcd"
            m.voxel_map_save(str(p), clear=True, keep=dict(min_miss=2, max_miss_per_hit=1.0))
            _same(plugin.read_pcd(str(p)), kept, "kept file")
            out.append(p.read_bytes())
            m2.voxel_map_save(str(tmp_path / "plain.pcd"), clear=True)
            ref.clear()
            assert m.voxel_map_info()["n_voxels"] == 0 and _evid(m).shape == (0, 2)
    out += [_cent(m).tobytes(), _evid(m).tobytes(), _cent(m, True).tobytes()]
    m.close()
    m2.close()
    return out


@pytest.mark.parametrize("L", [1, 3])
def test_counters_equal_the_restatement_over_a_drive(L, tmp_path):
    _drive(L, tmp_path)


def test_two_runs_give_identical_bytes(tmp_path):
    assert _drive(3, tmp_path, check=False) == _drive(3, tmp_path, check=False)


RECENT = 9   # as tests/test_world_carve_cpu.py: the trail the car left in the last 9 scans may stay


def _in_boxes(p, boxes, grow=0.0):
    inside = np.zeros(p.shape[0], bool)
    for lo, hi in boxes:
        inside |= np.all((p >= lo - grow) & (p < hi + grow), axis=1)
    return inside


def test_kept_map_as_a_prior_has_no_trail(tmp_path):
    st = synth.Street()
    leaf = 0.5
    m = plugin.MeasurementModel(1)
    ref = CR.CarveMapRef()
    for k in range(20):
        sc = synth.street_scan(st, k)
        _plant(m, 0, sc["body"][0])
        d = m.publish_frame_world(sc["state"], True, np.zeros(1, F))
        assert m.voxel_map_accumulate(sc["state"], np.zeros(1, F), leaf, carve=True) == ref.accumulate_carve(
            d, [d.shape[0]], _origins(sc["state"], 1), leaf, plugin.CARVE_MAX_RANGE, plugin.CARVE_END_MARGIN)
    full, kept = _cent(m), _cent(m, True)
    mask = ref.kept_mask(plugin.KEEP_MIN_MISS, plugin.KEEP_MAX_MISS_PER_HIT)
    _same(kept, full[mask], "kept = unfiltered minus the rule's voxels")
    pk, pf = tmp_path / "kept.pcd", tmp_path / "full.pcd"
    m.voxel_map_save(str(pk), clear=False, keep=True)
    m.voxel_map_save(str(pf), clear=False)
    _same(plugin.read_pcd(str(pk)), kept, "kept file")
    # the car's trail: its boxes before the last RECENT scans, away from its later boxes and above the ground's voxel layer
    early = [st.car(k) for k in range(20 - RECENT)]
    late = [st.car(k) for k in range(20 - RECENT, 20)]
    counts = []
    for p in (pf, pk):
        pts = plugin.read_pcd(str(p))
        m.prior_map_load(pts[:, :3])
        assert m.prior_map_info()["n_points"] == pts.shape[0]
        xyz = pts[:, :3].astype(np.float64)
        trail = _in_boxes(xyz, early) & ~_in_boxes(xyz, late, grow=leaf) & (xyz[:, 2] >= st.car_z0 + leaf)
        counts.append(int(trail.sum()))
    assert counts[0] > 20 and counts[1] == 0, counts
    m.close()


def _snapshot(m):
    return _cent(m).tobytes(), _evid(m).tobytes(), m.voxel_map_info()["n_voxels"]


def test_refusals_leave_the_map_unchanged(tmp_path):
    L = 1
    m = plugin.MeasurementModel(L)
    lib, h = m.lib, m._h
    leaf = 0.001
    s = synth.make_state([0.0, 0.0, 0.0], Q_ID, [Q_ID], [np.zeros(3)])
    rng = np.random.default_rng(9)
    for k in range(3):
        _plant(m, 0, rng.normal(0, 0.05, (3000, 3)))
        m.voxel_map_accumulate(s, [0.0], leaf, carve=dict(max_range=50.0, end_margin=0.0))
    before = _snapshot(m)
    assert before[2] > 0 and _evid(m)[:, 1].max() > 0
    ps, tag, n = s.pass_state(), np.zeros(1, F), C.c_uint64(0)

    def carve(a, lf=leaf, state=ps):
        return lib.malio_world_voxel_accumulate_carve(h, C.byref(state), capi.ptr(tag), lf, None if a is None else C.byref(a),
                                                      C.byref(n))
    assert carve(None) == capi.ERR_INVALID_ARG
    for mr, em in ((float("nan"), 0.0), (0.0, 0.0), (-1.0, 0.0), (float("inf"), 0.0), (10.0, -1.0), (10.0, float("nan")),
                   (10.0, float("inf"))):
        assert carve(capi.CarveArgs(mr, em)) == capi.ERR_INVALID_ARG, (mr, em)
    assert carve(capi.CarveArgs(10.0, 0.0), lf=0.002) == capi.ERR_INVALID_ARG            # the map's leaf is 0.001
    assert carve(capi.CarveArgs(70.0, 0.0)) == capi.ERR_CAPACITY                         # 70 m / 1 mm > 65536 cells
    far = synth.make_state([3.0e6, 0.0, 0.0], Q_ID, [Q_ID], [np.zeros(3)])               # origin outside int, points inside
    _plant(m, 0, np.array([[-3.0e6 + 0.01, 0.0, 0.0]] * 10, F))
    assert m.publish_frame_world(far, True, tag)[:, 0].max() < 1.0
    assert carve(capi.CarveArgs(10.0, 0.0), state=far.pass_state()) == capi.ERR_CAPACITY
    _plant(m, 0, np.array([[3.0e6, 0.0, 0.0]], F))                                       # an end outside int
    assert carve(capi.CarveArgs(10.0, 0.0)) == capi.ERR_CAPACITY
    keep = capi.CarveKeep(1, float("nan"))
    p = tmp_path / "x.pcd"
    assert lib.malio_world_voxel_save_pcd_kept(h, os.fsencode(str(p)), C.byref(keep), 1) == capi.ERR_INVALID_ARG
    bad = tmp_path / "missing_dir" / "x.pcd"                                             # a failed save does not clear
    assert lib.malio_world_voxel_save_pcd_kept(h, os.fsencode(str(bad)), C.byref(capi.CarveKeep(1, 0.5)), 1) == capi.ERR_INVALID_ARG
    assert not p.exists() and not bad.exists()
    assert _snapshot(m) == before
    m.close()


def test_downloads_follow_the_device_memory_contract():
    L = 1
    m = plugin.MeasurementModel(L)
    lib, h = m.lib, m._h
    s = synth.make_state([0.0, 0.0, 1.0], Q_ID, [Q_ID], [np.zeros(3)])
    rng = np.random.default_rng(3)
    for k in range(4):
        _plant(m, 0, rng.normal(0, 6, (40000, 3)))
        n = m.voxel_map_accumulate(s, [1.0], 0.2, carve=True)
    ev, kept = _evid(m), _cent(m, dict(min_miss=1, max_miss_per_hit=0.5))
    assert 0 < kept.shape[0] < n
    k = C.c_uint64(0)
    keep = capi.CarveKeep(1, 0.5)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        be = torch.empty((n, 2), dtype=torch.int32, device="cuda")
        bk = torch.empty((n, 4), device="cuda")
        torch.cuda._sleep(200_000_000)
        be.fill_(-7)
        bk.fill_(-7.0)                                     # behind the sleep: the downloads must come after it
        assert lib.malio_world_voxel_evidence_device(h, be.data_ptr(), n, C.byref(k), side.cuda_stream) == capi.OK and k.value == n
        assert lib.malio_world_voxel_download_kept_device(h, C.byref(keep), bk.data_ptr(), n, C.byref(k), side.cuda_stream) == capi.OK
        tot = bk[: k.value].double().sum()
    side.synchronize()
    assert k.value == kept.shape[0]
    _same(be.cpu().numpy().view(np.uint32), ev, "evidence, side stream")
    _same(bk[: k.value].cpu().numpy(), kept, "kept, side stream")
    assert np.all(bk[k.value:].cpu().numpy() == -7.0)
    np.testing.assert_allclose(float(tot), kept.astype(np.float64).sum(), rtol=1e-9)
    st = torch.cuda.current_stream().cuda_stream
    assert lib.malio_world_voxel_evidence_device(h, None, 0, C.byref(k), st) == capi.OK and k.value == n
    assert lib.malio_world_voxel_download_kept_device(h, C.byref(keep), None, 0, C.byref(k), st) == capi.OK and k.value == kept.shape[0]
    assert lib.malio_world_voxel_evidence_device(h, None, 5, C.byref(k), st) == capi.ERR_INVALID_ARG
    assert lib.malio_world_voxel_download_kept_device(h, None, bk.data_ptr(), n, C.byref(k), st) == capi.ERR_INVALID_ARG
    part = torch.full((n, 2), -3, dtype=torch.int32, device="cuda")
    assert lib.malio_world_voxel_evidence_device(h, part.data_ptr(), n // 3, C.byref(k), st) == capi.OK and k.value == n
    got = part.cpu().numpy()
    _same(got[: n // 3].view(np.uint32), ev[: n // 3], "cap rows")
    assert np.all(got[n // 3:] == -3)
    hp = np.zeros(n * 4, F)
    pin = torch.empty(n * 4).pin_memory()
    c0 = m.counters().kernel_launches
    for what, p in {"host": hp.ctypes.data, "pinned": pin.data_ptr(), "misaligned 4": be.data_ptr() + 4}.items():
        assert lib.malio_world_voxel_evidence_device(h, p, n, C.byref(k), st) == capi.ERR_INVALID_ARG, what
    for what, p in {"host": hp.ctypes.data, "pinned": pin.data_ptr(), "misaligned 8": bk.data_ptr() + 8}.items():
        assert lib.malio_world_voxel_download_kept_device(h, C.byref(keep), p, n, C.byref(k), st) == capi.ERR_INVALID_ARG, what
    assert m.counters().kernel_launches == c0
    _same(_evid(m), ev, "after the refusals")
    m.close()


def test_never_carved_map_has_zero_evidence_and_keeps_everything():
    m = plugin.MeasurementModel(1)
    s = synth.make_state([0.0, 0.0, 0.0], Q_ID, [Q_ID], [np.zeros(3)])
    _plant(m, 0, np.random.default_rng(1).normal(0, 3, (5000, 3)))
    b0 = m.voxel_map_info()["device_bytes"]
    n = m.voxel_map_accumulate(s, [0.0], 0.3)
    assert np.all(_evid(m) == 0) and _evid(m).shape == (n, 2)
    _same(_cent(m, True), _cent(m), "kept = all")
    info = m.voxel_map_info()
    m.voxel_map_accumulate(s, [0.0], 0.3, carve=True)
    assert m.voxel_map_info()["device_bytes"] >= info["device_bytes"] + 12 * info["capacity"] and b0 >= 0
    m.close()


def test_device_bytes_flat_over_300_carved_scans():
    m = plugin.MeasurementModel(1)
    rng = np.random.default_rng(13)
    raw = np.concatenate([rng.uniform(-30, 30, (10000, 2)), rng.uniform(-1, 2, (10000, 1))], axis=1).astype(F)
    _plant(m, 0, raw)
    hist = []
    for k in range(300):
        s = synth.make_state([2.0 * (k % 10), 1.0 * (k % 3), 0.0], Q_ID, [Q_ID], [np.zeros(3)])
        m.voxel_map_accumulate(s, [1.0], 0.2, carve=True)
        hist.append(m.voxel_map_info())
    assert hist[30] == hist[-1]
    ev = _evid(m)
    assert ev[:, 0].max() > 20 and ev[:, 1].max() > 0
    m.close()
