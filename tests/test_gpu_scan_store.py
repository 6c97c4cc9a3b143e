"""The scan store and the voxel map's rebuild on the device (malio_scan_store_*, malio_world_voxel_rebuild), exactly against the
per-scan accumulate calls and tests/scan_store_ref.py:
  - a 20-scan street drive, L = 1 and L = 3 (L = 3 after an upload with a temporal compensation, so that the stored one is
    read), plain and carved scans mixed: clear and rebuild gives the session's centroids, evidence and voxel count;
  - a store of more than one chunk and more than one block gives the bytes of rebuilding it scan by scan;
  - a drifted trajectory rebuilt with the true states equals a handle that accumulated the true states (plain, carved, and
    seeded then carved); another leaf equals a session at that leaf;
  - get / put, the .npz file, register_device against malio_world_register; refusals leave the map as it was; two runs give
    the same bytes."""
import ctypes as C

import numpy as np
import pytest
import torch

import carve_ref as CR
import scan_store_ref as SR
import world_voxel_ref as V
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
Q_ID = np.array([1.0, 0.0, 0.0, 0.0])
CARVE = dict(max_range=60.0, end_margin=0.5)
PLAIN = (4, 5, 9)   # scans folded with the plain accumulate, the others carved


def _plant(m, slot, xyz):
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    ctrl_t = np.array([-10.0, -9.0, -8.0, -7.0])
    m.undistort(slot, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), ctrl_t, np.tile(np.eye(4), (4, 1, 1)), np.zeros(0), -1)


def _model(L):
    """A handle; for L > 1 its last scan upload carries a temporal compensation that is not the identity."""
    m = plugin.MeasurementModel(L)
    if L > 1:
        case = synth.make_case("store-tc", 200, 5000, L, 3)
        tc = np.zeros(L - 1, capi.RIGID)
        for i in range(L - 1):
            q = np.array([1.0, 0.01 * (i + 1), -0.02, 0.015])
            tc[i]["q"], tc[i]["t"] = q / np.linalg.norm(q), (0.05 * (i + 1), -0.03, 0.02)
        m.upload_scan(case.pts, case.table, case.table_off, tc)
    return m


def _same(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.shape, b.shape)
    assert a.tobytes() == b.tobytes(), what


def _cent(m):
    return m.voxel_map_tensor().cpu().numpy()


def _evid(m):
    return m.voxel_map_evidence_tensor().cpu().numpy().view(np.uint32)


def _snapshot(m):
    return _cent(m).tobytes(), _evid(m).tobytes(), m.voxel_map_info()["n_voxels"]


def _drifted(s, k):
    """s with a drift that grows along the drive: position and a yaw about z."""
    d = capi.PassState()
    C.memmove(C.byref(d), C.byref(s), C.sizeof(capi.PassState))
    a = 0.002 * k
    qz = np.array([np.cos(a / 2), 0.0, 0.0, np.sin(a / 2)])
    q = np.array(s.rot[:])
    w0, x0, y0, z0 = qz
    w1, x1, y1, z1 = q
    d.rot[:] = [w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1, w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1,
                w0 * y1 - x0 * z1 + y0 * w1 + z0 * x1, w0 * z1 + x0 * y1 - y0 * x1 + z0 * w1]
    d.pos[:] = np.array(s.pos[:]) + np.array([0.02, 0.12, 0.06]) * k
    return d


def _runs(plan):
    """(first, count, carve) of the runs of equal modes in plan (True: carved)."""
    out, k = [], 0
    while k < len(plan):
        j = k
        while j < len(plan) and plan[j] == plan[k]:
            j += 1
        out.append((k, j - k, CARVE if plan[k] else None))
        k = j
    return out


def _drive(L, leaf=0.5, n=20, plan=None, store_states=None, check_register=False):
    """Accumulate and store n street scans on one handle (plan[k]: carved); store_states(s, k) -> the state stored for scan k
    (default: the state it was accumulated with).  Returns (handle, the true states, the scans' planted clouds, the tags)."""
    st = synth.Street()
    m = _model(L)
    tags = np.arange(L, dtype=F) + 0.25
    plan = plan if plan is not None else [k not in PLAIN for k in range(n)]
    states, clouds = [], []
    for k in range(n):
        sc = synth.street_scan(st, k, L=L, spin=(16, 128), cone=300)
        body = list(sc["body"])
        for l in range(L):
            _plant(m, l, body[l])
        s = sc["state"].pass_state() if isinstance(sc["state"], capi.State) else sc["state"]
        ss = s if store_states is None else store_states(s, k)
        info0 = m.voxel_map_info()
        assert m.scan_store_add(ss, tags, time=0.1 * k) == k + 1
        assert m.voxel_map_info() == info0   # the store grows its own bytes only
        if check_register:
            live = m.publish_frame_world(ss, True, tags)
            _same(m.scan_store_register_tensor(k).cpu().numpy(), live, ("register_device", k))
            other = _drifted(ss, 7)
            _same(m.scan_store_register_tensor(k, other).cpu().numpy(), m.publish_frame_world(other, True, tags), ("other state", k))
        m.voxel_map_accumulate(ss, tags, leaf, carve=CARVE if plan[k] else None)
        states.append(s)
        clouds.append(body)
    return m, states, clouds, tags, plan


def _scans(m, L):
    out = []
    for k in range(m.scan_store_info()["n_scans"]):
        rec, xyz = m.scan_store_get(k)
        out.append(SR.scan_of(rec, xyz, L))
    return out


def _clear(m, tmp_path):
    m.voxel_map_save(str(tmp_path / "cleared.pcd"), clear=True)
    assert m.voxel_map_info()["n_voxels"] == 0


def _rebuild_runs(m, leaf, plan, states=None):
    n = 0
    for first, count, carve in _runs(plan):
        n = m.voxel_map_rebuild(leaf, None if states is None else states[first:first + count], first, count, carve)
    return n


@pytest.mark.parametrize("L", [1, 3])
def test_rebuild_of_a_session_equals_the_session(L, tmp_path):
    m, _, _, _, plan = _drive(L, check_register=True)
    session = _snapshot(m)
    scans = _scans(m, L)
    if L > 1:   # the compensation of the upload was stored
        assert scans[0]["temporal_comp"][0]["t"][0] == 0.05
    ref = CR.CarveMapRef()
    for first, count, carve in _runs(plan):
        SR.rebuild(ref, scans[first:first + count], 0.5, carve=carve)
    _same(np.frombuffer(session[0], F).reshape(-1, 4), ref.centroids(), "session vs restatement")
    _same(np.frombuffer(session[1], np.uint32).reshape(-1, 2), ref.evidence(), "evidence vs restatement")
    _clear(m, tmp_path)
    n = _rebuild_runs(m, 0.5, plan)
    assert n == session[2]
    assert _snapshot(m) == session
    # the whole store plain, in one call, against the per-scan calls
    _clear(m, tmp_path)
    m.voxel_map_rebuild(0.5)
    one = _snapshot(m)
    _clear(m, tmp_path)
    for k in range(len(plan)):
        m.voxel_map_rebuild(0.5, first=k, count=1)
    assert _snapshot(m)[0] == one[0] and _snapshot(m)[2] == one[2]
    m.close()


def test_store_of_several_chunks_and_blocks_equals_scan_by_scan(tmp_path):
    """Scans put with random points: chunks of several scans, scans alone in a chunk, and a second block."""
    rng = np.random.default_rng(7)
    sizes = [1_500_000, 1_500_000, 1_500_000, 3_900_000, 3_900_000, 3_900_000, 1_200_000, 1_200_000]
    assert sum(sizes[:6]) <= capi.STORE_BLOCK_POINTS < sum(sizes[:7])
    a, b = plugin.MeasurementModel(3), plugin.MeasurementModel(3)
    recs = []
    for k, n in enumerate(sizes):
        rec = capi.StoredScan()
        rec.time = float(k)
        q = np.array([1.0, *rng.normal(scale=0.1, size=3)])
        rec.state.rot[:] = q / np.linalg.norm(q)
        rec.state.pos[:] = rng.uniform(-20, 20, 3)
        for l in range(3):
            rec.state.ext[l].q[:] = Q_ID
            rec.state.ext[l].t[:] = (0.1 * l, 0.0, 0.2)
            rec.slot_tag[l] = l + 0.5
        for i in range(2):
            rec.temporal_comp[i].q[:] = Q_ID
            rec.temporal_comp[i].t[:] = (0.01, 0.02 * i, 0.0)
        rec.n_points[:] = [n // 2, n // 4, n - n // 2 - n // 4]
        xyz = rng.uniform([-100, -100, -5], [100, 100, 15], (n, 3)).astype(F)
        xyz[::9973] = np.nan
        recs.append(rec)
        for mm in (a, b):
            mm.scan_store_put(rec, xyz)
    info = a.scan_store_info()
    assert info["n_scans"] == len(sizes) and info["n_points"] == sum(sizes)
    assert info["device_bytes"] == 12 * (capi.STORE_BLOCK_POINTS + capi.STORE_BLOCK_POINTS)
    n1 = a.voxel_map_rebuild(0.5)
    for k in range(len(sizes)):
        n2 = b.voxel_map_rebuild(0.5, first=k, count=1)
    assert n1 == n2
    _same(_cent(a), _cent(b), "chunked vs scan by scan")
    # corrected states for part of the range, against the per-scan calls
    states = [_drifted(r.state, 5 + k) for k, r in enumerate(recs)]
    for mm in (a, b):
        mm.voxel_map_save(str(tmp_path / "clear.pcd"), clear=True)
    a.voxel_map_rebuild(0.5, states[2:7], 2, 5)
    for k in range(2, 7):
        b.voxel_map_rebuild(0.5, [states[k]], k, 1)
    _same(_cent(a), _cent(b), "chunked vs scan by scan, given states")
    a.close()
    b.close()


def _true_session(L, states, clouds, tags, leaf, carve_all=False, seed=None):
    m = _model(L)
    if seed is not None:
        m.voxel_map_seed(seed, leaf)
    for s, body in zip(states, clouds):
        for l in range(L):
            _plant(m, l, body[l])
        m.voxel_map_accumulate(s, tags, leaf, carve=CARVE if carve_all else None)
    return m


@pytest.mark.parametrize("L", [1, 3])
def test_corrected_trajectory_gives_the_true_map(L, tmp_path):
    plan = [False] * 20
    m, truth, clouds, tags, _ = _drive(L, plan=plan, store_states=_drifted)
    drifted_n = m.voxel_map_info()["n_voxels"]
    t = _true_session(L, truth, clouds, tags, 0.5)
    true_n = t.voxel_map_info()["n_voxels"]
    assert drifted_n > true_n   # doubled walls
    scans = _scans(m, L)
    _clear(m, tmp_path)
    assert m.voxel_map_rebuild(0.5, truth) == true_n
    _same(_cent(m), _cent(t), "rebuild with the true states vs the true session")
    ref = V.VoxelMapRef()
    SR.rebuild(ref, scans, 0.5, truth)
    _same(_cent(m), ref.centroids(), "rebuild vs restatement")
    # carved
    tc = _true_session(L, truth, clouds, tags, 0.5, carve_all=True)
    _clear(m, tmp_path)
    m.voxel_map_rebuild(0.5, truth, carve=CARVE)
    assert _snapshot(m) == _snapshot(tc)
    cref = CR.CarveMapRef()
    SR.rebuild(cref, scans, 0.5, truth, carve=CARVE)
    _same(_evid(m), cref.evidence(), "carved evidence vs restatement")
    # seeded, then carved by the corrected session
    prior = _cent(t)[::3].copy()
    _clear(m, tmp_path)
    m.voxel_map_seed(prior, 0.5)
    m.voxel_map_rebuild(0.5, truth, carve=CARVE)
    ts = _true_session(L, truth, clouds, tags, 0.5, carve_all=True, seed=prior)
    assert _snapshot(m) == _snapshot(ts)
    for h in (m, t, tc, ts):
        h.close()


def test_rebuild_at_another_leaf_equals_a_session_at_it(tmp_path):
    L = 3
    m, truth, clouds, tags, plan = _drive(L, leaf=0.5)
    _clear(m, tmp_path)
    m.voxel_map_rebuild(0.1)
    t = _true_session(L, truth, clouds, tags, 0.1)
    assert _snapshot(m) == _snapshot(t)
    m.close()
    t.close()


def test_store_round_trips(tmp_path):
    L = 3
    m, _, _, _, plan = _drive(L, n=8)
    _clear(m, tmp_path)
    m.voxel_map_rebuild(0.5, carve=CARVE)
    want = _snapshot(m)
    p = tmp_path / "store.npz"
    plugin.save_scan_store(m, str(p))
    copy, loaded = plugin.MeasurementModel(L), plugin.MeasurementModel(L)
    for k in range(8):
        rec, xyz = m.scan_store_get(k)
        copy.scan_store_put(rec, xyz)
    assert plugin.load_scan_store(loaded, str(p)) == 8
    for h in (copy, loaded):
        assert h.scan_store_info()["n_points"] == m.scan_store_info()["n_points"]
        h.voxel_map_rebuild(0.5, carve=CARVE)
        assert _snapshot(h) == want
        for k in (0, 7):
            _same(h.scan_store_register_tensor(k).cpu().numpy(), m.scan_store_register_tensor(k).cpu().numpy(), ("register", k))
    recs = m.scan_store_records()
    assert [r.time for r in recs] == [0.1 * k for k in range(8)]
    scans = _scans(m, L)
    for k in (0, 5):
        _same(m.scan_store_register_tensor(k).cpu().numpy(), SR.register(scans[k]), ("register vs restatement", k))
        other = _drifted(recs[k].state, 9)
        _same(m.scan_store_register_tensor(k, other).cpu().numpy(), SR.register(scans[k], other), ("other state", k))
        body = m.scan_store_register_tensor(k, capi.PassState(rot=(C.c_double * 4)(1, 0, 0, 0), ext=recs[k].state.ext)).cpu().numpy()
        assert np.isfinite(body[:, :3]).all()
    m.scan_store_clear()
    assert m.scan_store_info() == dict(n_scans=0, n_points=0, device_bytes=0)
    for h in (m, copy, loaded):
        h.close()


def test_refusals_leave_everything_unchanged(tmp_path):
    L = 1
    m = _model(L)
    lib, h = m.lib, m._h
    n = C.c_uint64(0)
    tags = np.zeros(1, F)
    assert lib.malio_scan_store_add(h, C.byref(capi.PassState()), tags.ctypes.data, 0.0, None) == capi.ERR_STATE   # no undistort yet
    m.close()
    m, truth, _, tags, plan = _drive(L, n=6)
    lib, h = m.lib, m._h
    before = _snapshot(m)
    store = m.scan_store_info()
    bad_carve = capi.CarveArgs(-1.0, 0.5)
    far = capi.CarveArgs(1e5, 0.5)
    ok = capi.CarveArgs(60.0, 0.5)
    far_state = (capi.PassState * 6)()
    for i in range(6):
        far_state[i] = truth[i]
    far_state[4].pos[:] = (3e9 * 0.5, 0.0, 0.0)
    cases = [
        (dict(first=5, count=2), capi.ERR_INVALID_ARG),
        (dict(first=7, count=0), capi.ERR_INVALID_ARG),
        (dict(leaf=0.25), capi.ERR_INVALID_ARG),            # differs from the map's
        (dict(leaf=float("nan")), capi.ERR_INVALID_ARG),
        (dict(carve=bad_carve), capi.ERR_INVALID_ARG),
        (dict(carve=far), capi.ERR_CAPACITY),               # max_range / leaf above the cap
        (dict(states=far_state), capi.ERR_CAPACITY),         # scan 4's points outside int
        (dict(states=far_state, carve=ok), capi.ERR_CAPACITY),
    ]
    for kw, want in cases:
        a = kw.get("carve")
        rc = lib.malio_world_voxel_rebuild(h, kw.get("first", 0), kw.get("count", 6), kw.get("states"), C.c_float(kw.get("leaf", 0.5)),
                                           None if a is None else C.byref(a), C.byref(n))
        assert rc == want, kw
        assert _snapshot(m) == before, kw
    assert m.scan_store_info() == store
    # the origin alone outside int (a slot with points): carved refused, plain accepted
    # count == 0 changes nothing
    assert lib.malio_world_voxel_rebuild(h, 6, 0, None, C.c_float(0.25), None, C.byref(n)) == capi.OK and n.value == before[2]
    assert _snapshot(m) == before
    # the map still takes its leaf
    assert m.voxel_map_rebuild(0.5, first=0, count=1) >= before[2]
    # register_device: the size protocol and device-memory contract
    rows = m.scan_store_register_tensor(2)
    cnt = C.c_uint64(0)
    assert lib.malio_scan_store_register_device(h, 2, None, None, 0, C.byref(cnt), None) == capi.OK and cnt.value == rows.shape[0]
    host = np.zeros((rows.shape[0], 4), F)
    assert lib.malio_scan_store_register_device(h, 2, None, host.ctypes.data, rows.shape[0], C.byref(cnt), None) == capi.ERR_INVALID_ARG
    dev = torch.zeros(rows.shape[0] * 4 + 1, dtype=torch.float32, device="cuda")
    assert lib.malio_scan_store_register_device(h, 2, None, dev.data_ptr() + 4, rows.shape[0], C.byref(cnt), None) == capi.ERR_INVALID_ARG
    assert lib.malio_scan_store_register_device(h, 6, None, None, 0, C.byref(cnt), None) == capi.ERR_INVALID_ARG
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        part = torch.full((100, 4), -1.0, dtype=torch.float32, device="cuda")
        assert lib.malio_scan_store_register_device(h, 2, None, part.data_ptr(), 100, C.byref(cnt), side.cuda_stream) == capi.OK
        got = part.clone()   # ordered after the call on the same stream
    side.synchronize()
    assert cnt.value == rows.shape[0]
    _same(got.cpu().numpy(), rows[:100].cpu().numpy(), "first cap points on the caller's stream")
    # get: capacity
    rec = capi.StoredScan()
    small = np.zeros((1, 3), F)
    assert lib.malio_scan_store_get(h, 2, C.byref(rec), small.ctypes.data, 1, C.byref(cnt)) == capi.ERR_CAPACITY
    # put: counts beyond L, and above 2^31 - 1
    rec.n_points[:] = [1, 1, 0]
    assert lib.malio_scan_store_put(h, C.byref(rec), small.ctypes.data, None) == capi.ERR_INVALID_ARG
    rec.n_points[:] = [0x80000000, 0, 0]
    assert lib.malio_scan_store_put(h, C.byref(rec), small.ctypes.data, None) == capi.ERR_INVALID_ARG
    assert m.scan_store_info() == store
    m.close()


def test_two_runs_give_identical_bytes(tmp_path):
    def run():
        m, truth, _, _, plan = _drive(3, n=10)
        _clear(m, tmp_path)
        m.voxel_map_rebuild(0.5, [_drifted(s, 2) for s in truth], carve=CARVE)
        out = _snapshot(m)
        m.close()
        return out
    assert run() == run()
