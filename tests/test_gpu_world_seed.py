"""Keeping a saved map current on the device (malio_world_voxel_seed*, malio_world_voxel_changes_device and
malio_world_voxel_save_changes_pcd), exactly against tests/world_seed_ref.py:
  - the seed's centroids, keys and evidence; then a 20-scan carved session on the seeded map (L = 1 and L = 3, plain
    accumulate calls mixed in): centroids, evidence, the kept download, removed and added after every few scans;
  - a seed larger than MALIO_SEED_CHUNK against the one-shot restatement; host and device entries give the same bytes;
  - the saved kept file read back and seeded; two sessions end to end, session 2 tracked in session 1's kept map;
  - refusals, the device-memory contracts, empty change sets, clearing saves, never-seeded maps and device memory."""
import ctypes as C
from dataclasses import replace

import numpy as np
import pytest
import torch

import world_ref as W
import world_seed_ref as SR
import world_voxel_ref as V
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
Q_ID = np.array([1.0, 0.0, 0.0, 0.0])
LEAF = 0.5
KEEP = dict(min_miss=plugin.KEEP_MIN_MISS, max_miss_per_hit=plugin.KEEP_MAX_MISS_PER_HIT)
GONE = 2
NEW = ((12.0, -6.4, 0.0), (16.0, -4.6, 1.4))


def _plant(m, slot, xyz):
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    ctrl_t = np.array([-10.0, -9.0, -8.0, -7.0])
    m.undistort(slot, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), ctrl_t, np.tile(np.eye(4), (4, 1, 1)), np.zeros(0), -1)


def _origins(state, L):
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


def _changes(m, keep=True):
    r, a = m.voxel_map_changes(keep)
    return r.cpu().numpy(), a.cpu().numpy()


def _session1_kept(n=20):
    """Session 1 on the default street, restated on the host (bit-exact with the device): the kept map and the restatement."""
    ref = SR.SeedMapRef()
    for k in range(n):
        s = synth.street_scan(synth.Street(), k)
        cloud = W.register_world(s["state"], None, s["body"][0], 0, 0.0)
        org = W.register_world(s["state"], None, np.zeros((1, 3), F), 0, 0.0)[:, :3]
        ref.accumulate_carve(cloud, [cloud.shape[0]], org, LEAF, plugin.CARVE_MAX_RANGE, plugin.CARVE_END_MARGIN)
    mask = ref.kept_mask(**{"min_miss": KEEP["min_miss"], "max_miss_per_hit": KEEP["max_miss_per_hit"]})
    return ref.centroids()[mask], ref.keys()[mask]


CARVE = dict(max_range=60.0, end_margin=0.5)
PLAIN = (4, 9)


@pytest.mark.parametrize("L", [1, 3])
def test_seeded_session_equals_the_restatement(L):
    seedc, _ = _session1_kept(10)
    m = plugin.MeasurementModel(L)
    ref = SR.SeedMapRef()
    assert m.voxel_map_seed(seedc, LEAF, 3) == ref.seed(seedc, LEAF, 3)
    _same(_cent(m), ref.centroids(), "seed centroids")
    _same(_evid(m), ref.evidence(), "seed evidence")
    st = synth.Street(gone=(GONE,), extra=(NEW,))
    tags = np.arange(L, dtype=F)
    for k in range(20):
        sc = synth.street_scan(st, k, L=L, spin=(16, 128), cone=300, seed=1)
        for l in range(L):
            _plant(m, l, sc["body"][l])
        s = sc["state"]
        d = m.publish_frame_world(s, True, tags)
        if k in PLAIN:
            assert m.voxel_map_accumulate(s, tags, LEAF) == ref.accumulate(d, LEAF)
        else:
            assert m.voxel_map_accumulate(s, tags, LEAF, carve=CARVE) == ref.accumulate_carve(
                d, [b.shape[0] for b in sc["body"]], _origins(s, L), LEAF, **CARVE)
        if k % 5 == 4 or k == 19:
            c = _cent(m)
            _same(c, ref.centroids(), ("centroids", k))
            _same(_evid(m), ref.evidence(), ("evidence", k))
            for keep in (dict(min_miss=2, max_miss_per_hit=1.0), KEEP):
                seeded, kept, removed, added = ref.change_masks(keep["min_miss"], keep["max_miss_per_hit"])
                _same(_cent(m, keep), c[kept], ("kept", k))
                rem, add = _changes(m, keep)
                _same(rem, c[removed], ("removed", k))
                _same(add, c[added], ("added", k))
    assert rem.shape[0] > 0 and add.shape[0] > 0
    m.close()


def test_chunked_seed_and_both_entries():
    """5.2 M points (more than MALIO_SEED_CHUNK = 2^22), five per voxel in input runs, so chunk boundaries fall inside runs."""
    rng = np.random.default_rng(5)
    n = 5_200_000
    centre = rng.uniform(-50, 50, (n // 5, 3)).astype(F)
    xyz = np.repeat(centre, 5, axis=0) + rng.uniform(-0.04, 0.04, (n, 3)).astype(F)
    cloud = np.concatenate([xyz, rng.uniform(0, 255, (n, 1)).astype(F)], axis=1).astype(F)
    cloud[123, 0] = np.nan
    ref = V.VoxelMapRef()
    nv = ref.accumulate_fast(cloud, 0.1)
    a, b = plugin.MeasurementModel(1), plugin.MeasurementModel(1)
    assert a.voxel_map_seed(cloud, 0.1, 1) == nv
    t = torch.from_numpy(cloud).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        t2 = t.clone()                                  # behind the sleep: the seed must read it after the copy
        assert b.voxel_map_seed_tensor(t2, 0.1, 1) == nv
    side.synchronize()
    ca = _cent(a)
    _same(ca, ref.centroids(), "host entry = one-shot restatement")
    _same(_cent(b), ca, "device entry = host entry")
    ev = _evid(a)
    assert np.all(ev[:, 0] == 1) and np.all(ev[:, 1] == 0)
    _same(_evid(b), ev, "evidence")
    a.close(); b.close()


def test_round_trip_through_the_kept_file(tmp_path):
    """A carved map saved kept, read back and seeded equals the restatement seeding the file's centroids.  Re-keyed: how many
    centroids fall into another voxel than the one they average (a float sum / count on a voxel face)."""
    seedc, keys = _session1_kept(20)
    m = plugin.MeasurementModel(1)
    ref = SR.SeedMapRef()
    for k in range(20):
        s = synth.street_scan(synth.Street(), k)
        _plant(m, 0, s["body"][0])
        m.voxel_map_accumulate(s["state"], [0.0], LEAF, carve=True)
    p = tmp_path / "kept.pcd"
    m.voxel_map_save(str(p), clear=True, keep=True)
    pts = plugin.read_pcd(str(p))
    _same(pts, seedc, "kept file = restated kept map")
    assert m.voxel_map_seed(pts, LEAF) == ref.seed(pts, LEAF, plugin.SEED_HITS)
    _same(_cent(m), ref.centroids(), "re-seeded")
    _same(_evid(m), ref.evidence(), "re-seeded evidence")
    rekeyed = int(np.any(V.voxel_index(pts[:, :3], LEAF)[0] != keys, axis=1).sum())
    assert rekeyed < pts.shape[0] // 100, rekeyed
    assert m.voxel_map_info()["n_voxels"] <= pts.shape[0]
    m.close()


def _in_box(p, lo, hi, grow=0.0):
    return np.all((p >= np.asarray(lo) - grow) & (p < np.asarray(hi) + grow), axis=1)


def test_two_sessions_end_to_end(tmp_path):
    """Session 1 maps the street with carving and saves the kept file.  Session 2 drives the street with parked box GONE gone
    and box NEW added: it loads the file as the prior, seeds the voxel map from it, and tracks each scan with the prior
    window and the IESKF update from the previous estimate moved by the drive's step; it carves with the tracked states.
    Thresholds from the restatement's two-session run (tests/test_world_seed_cpu.py, truth states): 68 % of the gone box's
    voxels removed, 84 % of the new box's added, 0.8 % of the static voxels removed."""
    m1 = plugin.MeasurementModel(1)
    for k in range(20):
        s = synth.street_scan(synth.Street(), k)
        _plant(m1, 0, s["body"][0])
        m1.voxel_map_accumulate(s["state"], [0.0], LEAF, carve=True)
    f1 = tmp_path / "session1.pcd"
    m1.voxel_map_save(str(f1), clear=False, keep=True)
    m1.close()
    prior = plugin.read_pcd(str(f1))
    base = synth.make_case("street", 2000, 1000, 1, 4)
    m = plugin.MeasurementModel(1, params=base.params)
    m.prior_map_load(prior[:, :3])
    assert 0 < m.voxel_map_seed(prior, LEAF) <= prior.shape[0]
    st = synth.Street(gone=(GONE,), extra=(NEW,))
    est = None
    errs = []
    for k in range(20):
        sc = synth.street_scan(st, k, seed=1)
        xt = sc["state"]
        pw = sc["body"][0].astype(np.float64) + st.ego(k)
        case = synth.with_scan(replace(base, x_true=xt), pw, seed=k)
        pos = st.ego(k) if est is None else est + (st.ego(k) - st.ego(k - 1))
        x = synth.make_state(pos, Q_ID, [Q_ID], [np.zeros(3)])
        m.prior_map_window(x, 200.0, 80.0)
        m.upload_scan(case.pts, case.table, case.table_off, None)
        P = synth.init_P(case.n_dof)
        m.update_iterated_dyn_share_modified(x, P, 4)
        est = np.array(x.pos[:])
        errs.append(float(np.linalg.norm(est - st.ego(k))))
        _plant(m, 0, case.pts["xyz"])
        m.voxel_map_accumulate(x, [0.0], LEAF, carve=True)
    assert max(errs) < LEAF, [round(e, 3) for e in errs]       # tracked within a voxel of the prior at every scan
    c = _cent(m)
    rem, add = _changes(m)
    lo, hi = synth.Street().parked()[GONE]
    gone_seed = _in_box(prior[:, :3], lo, hi) & (prior[:, 2] >= LEAF)
    gone_removed = _in_box(rem[:, :3], lo, hi) & (rem[:, 2] >= LEAF)
    assert gone_seed.sum() >= 20 and gone_removed.sum() >= 0.5 * gone_seed.sum(), (gone_seed.sum(), gone_removed.sum())
    new_all = _in_box(c[:, :3], *NEW, grow=0.1) & (c[:, 2] >= LEAF)
    new_added = _in_box(add[:, :3], *NEW, grow=0.1) & (add[:, 2] >= LEAF)
    assert new_all.sum() >= 20 and new_added.sum() >= 0.7 * new_all.sum(), (new_all.sum(), new_added.sum())
    static = ~np.zeros(prior.shape[0], bool)
    for b in synth.Street().parked():
        static &= ~_in_box(prior[:, :3], *b, grow=LEAF)
    static &= np.abs(prior[:, 1] + 2.5) > 2.0                 # away from the moving car's lane
    rem_static = ~np.zeros(rem.shape[0], bool)
    for b in synth.Street().parked():
        rem_static &= ~_in_box(rem[:, :3], *b, grow=LEAF)
    rem_static &= np.abs(rem[:, 1] + 2.5) > 2.0
    assert rem_static.sum() <= 0.02 * static.sum(), (rem_static.sum(), static.sum())
    f2, fr, fa = tmp_path / "session2.pcd", tmp_path / "removed.pcd", tmp_path / "added.pcd"
    nr, na = m.voxel_map_save_changes(str(fr), str(fa))
    assert (nr, na) == (rem.shape[0], add.shape[0])
    _same(plugin.read_pcd(str(fr)), rem, "removed file")
    _same(plugin.read_pcd(str(fa)), add, "added file")
    m.voxel_map_save(str(f2), clear=True, keep=True)
    kept2 = plugin.read_pcd(str(f2))
    m3 = plugin.MeasurementModel(1)
    m3.prior_map_load(kept2[:, :3])
    assert m3.prior_map_info()["n_points"] == kept2.shape[0]
    in_gone = _in_box(kept2[:, :3], lo, hi) & (kept2[:, 2] >= LEAF)
    assert in_gone.sum() <= gone_seed.sum() - gone_removed.sum()
    assert (_in_box(kept2[:, :3], *NEW, grow=0.1) & (kept2[:, 2] >= LEAF)).sum() >= new_added.sum() > 0
    m.close(); m3.close()


def test_refusals_and_the_seed_contract(tmp_path):
    m = plugin.MeasurementModel(1)
    lib, h = m.lib, m._h
    n = C.c_uint64(0)
    pts = np.random.default_rng(2).uniform(-5, 5, (1000, 4)).astype(F)
    for args in ((None, 1000, 0.2), (capi.ptr(pts), 0, 0.2), (capi.ptr(pts), 1000, 0.0), (capi.ptr(pts), 1000, float("nan")),
                 (capi.ptr(pts), 1000, float("inf")), (capi.ptr(pts), 1000, -1.0)):
        assert lib.malio_world_voxel_seed(h, args[0], args[1], args[2], 1, C.byref(n)) == capi.ERR_INVALID_ARG, args
    assert m.voxel_map_info()["n_voxels"] == 0
    # a point outside int in the second chunk: the first chunk was folded, the map is empty again with its leaf unset
    big = np.random.default_rng(3).uniform(-5, 5, (SR.SEED_CHUNK + 10, 4)).astype(F)
    big[SR.SEED_CHUNK + 5, 0] = 3.0e6
    assert lib.malio_world_voxel_seed(h, capi.ptr(big), big.shape[0], 0.001, 2, C.byref(n)) == capi.ERR_CAPACITY
    info = m.voxel_map_info()
    assert info["n_voxels"] == 0 and _cent(m).shape == (0, 4)
    assert m.voxel_map_seed(pts, 0.3, 4) > 0                 # another leaf: the refused seed fixed none
    before = (_cent(m).tobytes(), _evid(m).tobytes())
    assert np.all(_evid(m) == [4, 0])
    assert lib.malio_world_voxel_seed(h, capi.ptr(pts), 1000, 0.3, 1, C.byref(n)) == capi.ERR_STATE
    # the first carve keeps the seeded counters: a scan far away hits nothing seeded
    s = synth.make_state([100.0, 0.0, 0.0], Q_ID, [Q_ID], [np.zeros(3)])
    _plant(m, 0, np.random.default_rng(4).uniform(-1, 1, (500, 3)))
    m.voxel_map_accumulate(s, [0.0], 0.3, carve=True)
    ev = _evid(m)
    seeded_rows = _cent(m)[:, 0] < 50.0
    assert np.all(ev[seeded_rows] == [4, 0]) and np.all(ev[~seeded_rows][:, 0] == 1)
    # a map an empty accumulate fixed the leaf of is not empty
    m2 = plugin.MeasurementModel(1)
    _plant(m2, 0, np.zeros((0, 3), F))
    m2.voxel_map_accumulate(s, [0.0], 0.3)
    assert m2.lib.malio_world_voxel_seed(m2._h, capi.ptr(pts), 1000, 0.3, 1, C.byref(n)) == capi.ERR_STATE
    assert m2.lib.malio_world_voxel_save_changes_pcd(m2._h, C.byref(plugin.carve_keep()), None, None, None, None) == capi.ERR_STATE
    m2.close()
    # device entry: pointer and alignment
    t = torch.from_numpy(pts).cuda()
    m3 = plugin.MeasurementModel(1)
    pin = torch.from_numpy(pts).pin_memory()
    st = torch.cuda.current_stream().cuda_stream
    c0 = m3.counters().kernel_launches
    flat = torch.zeros(4 * 1001, device="cuda")
    for what, p in {"host": pts.ctypes.data, "pinned": pin.data_ptr(), "misaligned": flat.data_ptr() + 4}.items():
        assert m3.lib.malio_world_voxel_seed_device(m3._h, p, 1000, 0.3, 1, C.byref(n), st) == capi.ERR_INVALID_ARG, what
    assert m3.counters().kernel_launches == c0 and m3.voxel_map_info()["n_voxels"] == 0
    assert m3.voxel_map_seed_tensor(t, 0.3, 4) == SR.SeedMapRef().seed(pts, 0.3, 4)
    _same(_evid(m3), np.frombuffer(before[1], np.uint32).reshape(-1, 2), "device entry evidence")
    m3.close()
    m.close()


def test_changes_contract_empty_sets_and_clearing_saves(tmp_path):
    m = plugin.MeasurementModel(1)
    lib, h = m.lib, m._h
    s = synth.make_state([0.0, 0.0, 1.0], Q_ID, [Q_ID], [np.zeros(3)])
    rng = np.random.default_rng(7)
    # never seeded: removed empty, added = the kept download
    for k in range(3):
        _plant(m, 0, rng.normal(0, 6, (20000, 3)))
        m.voxel_map_accumulate(s, [1.0], 0.2, carve=True)
    rem, add = _changes(m)
    assert rem.shape == (0, 4)
    _same(add, _cent(m, True), "never seeded: added = kept")
    fr, fa = tmp_path / "r.pcd", tmp_path / "a.pcd"
    assert m.voxel_map_save_changes(str(fr), str(fa)) == (0, add.shape[0])
    assert not fr.exists() and fa.exists()
    # a clearing save resets the seeded set
    m.voxel_map_save(str(tmp_path / "x.pcd"), clear=True)
    seedc = rng.uniform(-6, 6, (30000, 4)).astype(F)
    nv = m.voxel_map_seed(seedc, 0.2, 1)
    rem, add = _changes(m)
    assert rem.shape == (0, 4) and add.shape == (0, 4)      # never carved: everything kept, nothing new
    assert m.voxel_map_save_changes(str(tmp_path / "r2.pcd"), str(tmp_path / "a2.pcd")) == (0, 0)
    assert not (tmp_path / "r2.pcd").exists() and not (tmp_path / "a2.pcd").exists()
    for k in range(4):
        _plant(m, 0, rng.normal(0, 6, (20000, 3)))
        m.voxel_map_accumulate(s, [1.0], 0.2, carve=True)
    keep = capi.CarveKeep(1, 0.5)
    rem, add = _changes(m, keep)
    assert rem.shape[0] > 0 and add.shape[0] > 0
    n_all = m.voxel_map_info()["n_voxels"]
    # size protocol and device-memory contract
    nr, na = C.c_uint64(0), C.c_uint64(0)
    st = torch.cuda.current_stream().cuda_stream
    assert lib.malio_world_voxel_changes_device(h, C.byref(keep), None, 0, C.byref(nr), None, 0, C.byref(na), st) == capi.OK
    assert (nr.value, na.value) == (rem.shape[0], add.shape[0])
    assert lib.malio_world_voxel_changes_device(h, None, None, 0, C.byref(nr), None, 0, C.byref(na), st) == capi.ERR_INVALID_ARG
    assert lib.malio_world_voxel_changes_device(h, C.byref(keep), None, 5, C.byref(nr), None, 0, C.byref(na), st) == capi.ERR_INVALID_ARG
    br = torch.full((n_all, 4), -7.0, device="cuda")
    ba = torch.full((n_all, 4), -7.0, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        br.fill_(-5.0)
        assert lib.malio_world_voxel_changes_device(h, C.byref(keep), br.data_ptr(), 3, C.byref(nr), ba.data_ptr(), n_all,
                                                    C.byref(na), side.cuda_stream) == capi.OK
    side.synchronize()
    _same(br[:3].cpu().numpy(), rem[:3], "cap rows")
    assert np.all(br[3:].cpu().numpy() == -5.0)
    _same(ba[: na.value].cpu().numpy(), add, "added, side stream")
    hp = np.zeros(n_all * 4, F)
    pin = torch.empty(n_all * 4).pin_memory()
    for what, p in {"host": hp.ctypes.data, "pinned": pin.data_ptr(), "misaligned": ba.data_ptr() + 8}.items():
        assert lib.malio_world_voxel_changes_device(h, C.byref(keep), p, n_all, C.byref(nr), None, 0, C.byref(na), st) == capi.ERR_INVALID_ARG, what
        assert lib.malio_world_voxel_changes_device(h, C.byref(keep), None, 0, C.byref(nr), p, n_all, C.byref(na), st) == capi.ERR_INVALID_ARG, what
    # the kept map is the partition
    kept = _cent(m, keep)
    assert kept.shape[0] == nv - rem.shape[0] + add.shape[0]
    key = lambda a: {r.tobytes() for r in a}
    assert key(kept) >= key(add) and not (key(kept) & key(rem))
    # a clearing save resets the seeded set: afterwards removed is empty and added = kept
    m.voxel_map_save(str(tmp_path / "y.pcd"), clear=True)
    _plant(m, 0, rng.normal(0, 6, (20000, 3)))
    m.voxel_map_accumulate(s, [1.0], 0.2, carve=True)
    rem, add = _changes(m)
    assert rem.shape == (0, 4)
    _same(add, _cent(m, True), "after a clearing save")
    m.close()


def test_device_bytes_after_a_10m_point_seed():
    n = 10_000_000
    rng = np.random.default_rng(11)
    cloud = np.concatenate([rng.uniform(-200, 200, (n, 2)), rng.uniform(0, 20, (n, 1)), np.zeros((n, 1))], axis=1).astype(F)
    m = plugin.MeasurementModel(1)
    nv = m.voxel_map_seed(cloud, 0.2, 2)
    info = m.voxel_map_info()
    hc = 1 << 17
    while hc < 2 * n:
        hc *= 2
    chunk = 1 << 22
    scratch = (chunk + chunk // 8 + 1024) * 48                 # sort area and run rows of a chunk
    bound = info["capacity"] * (32 + 12) + hc * 4 + scratch + (64 << 20)   # entries, counters, hash, scratch, CUB storage
    assert nv <= info["capacity"] and info["device_bytes"] <= bound, (info, bound)
    assert info["device_bytes"] < info["capacity"] * 44 + hc * 4 + n * 24   # no point-sized scratch left behind
    m.close()
