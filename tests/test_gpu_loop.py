"""Loop closure over the scan store on the device (malio_scan_store_match) and end to end with malio_pose_graph_optimize:
  - exactness: small stored scans (L = 1 and L = 3 with a stored temporal compensation), one and three levels: pose, info,
    inliers, rms and per-level steps byte-equal to tests/loop_ref.py;
  - recovery: ray-cast scans of an aperiodic scene, guesses offset within the basin, recovered to a stated tolerance;
  - end to end: a ray-cast drive around a block back to its start, the stored states drifted by a random walk; close_loops
    brings the loop's nodes to within 0.1 m and 0.3 degrees of the truth, and the map where the loop closes, rebuilt under its
    states, matches the true-state rebuild (voxel count within 5 %, overlap > 0.7) where the drifted one does not (doubled
    walls: more than 8 % more voxels, overlap < 0.55);
  - degeneracy: a corridor gives a small eig_min and close_loops rejects the edge;
  - stability: two runs give the same bytes, refusals change nothing, the handle's device bytes stay."""
import ctypes as C
import math

import numpy as np
import pytest

import loop_ref as LR
import scan_store_ref as SR
from malio_b200 import capi, plugin, synth
from test_gpu_place import raycast
from test_gpu_relocalize import make_scene, q_yaw, sample_scene, scan_of  # noqa: F401

pytestmark = pytest.mark.gpu
F = np.float32


def _state(q, p, extq=None, extt=None):
    s = capi.PassState()
    s.rot[:], s.pos[:] = [float(v) for v in q], [float(v) for v in p]
    for l in range(capi.MAX_LIDAR):
        s.ext[l].q[:] = [1.0, 0.0, 0.0, 0.0] if extq is None else [float(v) for v in extq[l % len(extq)]]
        if extt is not None:
            s.ext[l].t[:] = [float(v) for v in extt[l % len(extt)]]
    return s


def _put(m, L, state, body_pts, tc=None):
    """Store world points seen from `state` as one scan: the LiDAR-frame points of each slot (round robin)."""
    rec = capi.StoredScan()
    rec.state = state
    if tc is not None:
        for i in range(L - 1):
            rec.temporal_comp[i].q[:] = list(tc[i]["q"])
            rec.temporal_comp[i].t[:] = list(tc[i]["t"])
    else:
        for i in range(L - 1):
            rec.temporal_comp[i].q[:] = [1.0, 0.0, 0.0, 0.0]
    parts = []
    for l in range(L):
        rec.slot_tag[l] = l
        parts.append(body_pts[l])
        rec.n_points[l] = body_pts[l].shape[0]
    m.scan_store_put(rec, np.concatenate(parts).astype(F))
    return rec


def _sensor(pw, L, state, tc):
    """World points -> per-slot LiDAR-frame float32 points for state (the inverse of the registration)."""
    extq = [np.array(state.ext[l].q[:]) for l in range(L)]
    extt = [np.array(state.ext[l].t[:]) for l in range(L)]
    lidar = np.arange(len(pw)) % L
    x = synth.world_to_sensor(pw, lidar, np.array(state.pos[:]), np.array(state.rot[:]), extq, extt, tc).astype(F)
    return [x[lidar == l] for l in range(L)]


def _store(m, L, items, tc=None):
    scans = []
    for state, pw in items:
        body = _sensor(pw, L, state, tc)
        rec = _put(m, L, state, body, tc)
        scans.append(SR.scan_of(rec, np.concatenate(body), L))
    return scans


def _same(got, want, what):
    assert np.asarray(got).tobytes() == np.asarray(want).tobytes(), what


def _check_exact(got, want):
    _same(np.array(got["rot"]), want["rot"], "rot")
    _same(np.array(got["pos"]), want["pos"], "pos")
    _same(got["info"], want["info"], "info")
    _same(np.array(got["rel_rot"]), want["rel_rot"], "rel_rot")
    _same(np.array(got["rel_pos"]), want["rel_pos"], "rel_pos")
    assert got["n_inliers"] == want["n_inliers"] and got["n_points"] == want["n_points"]
    assert got["rms"] == want["rms"] and got["fitness"] == want["fitness"]
    assert got["iterations"] == want["iterations"] and got["converged"] == want["converged"]
    assert got["target_voxels"] == want["target_voxels"] and got["target_points"] == want["target_points"]
    assert abs(got["eig_min"] - want["eig_min"]) <= 1e-8 * max(1.0, abs(want["eig_min"]))


def _small_case(seed, L):
    rng = np.random.default_rng(seed)
    scene = make_scene(rng, 40.0, 6)
    extq = [synth.q_exp(synth.rand_unit(rng) * 0.1) for _ in range(L)]
    extt = [rng.normal(0, 0.2, 3) for _ in range(L)]
    tc = None
    if L > 1:
        tc = np.zeros(L - 1, capi.RIGID)
        for i in range(L - 1):
            tc[i]["q"], tc[i]["t"] = synth.q_exp(synth.rand_unit(rng) * 0.03), rng.normal(0, 0.05, 3)
    items = []
    for k in range(4):
        pos = np.array([2.0 * k, 0.5 * k, 1.8])
        st = _state(q_yaw(0.05 * k), pos, extq, extt)
        items.append((st, sample_scene(scene, rng, 3.0, center=pos, radius=15.0)))
    return items, tc


@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("levels", [1, 3])
def test_match_is_bit_identical_to_the_restatement(L, levels):
    items, tc = _small_case(10 + L, L)
    m = plugin.MeasurementModel(L)
    scans = _store(m, L, items, tc)
    leaf = (2.0, 1.0, 0.5)[3 - levels:]
    gate = (1.0, 0.5, 0.3)[3 - levels:]
    a = plugin.match_args(0, 3, leaf=leaf, gate=gate, max_iter=8, eps_rot=1e-7, eps_pos=1e-6, min_points=4, planarity=0.2, sigma=0.05)
    guess = _state(LR.q_mul(list(items[3][0].rot), list(q_yaw(0.02))), np.array(items[3][0].pos[:]) + [0.3, -0.2, 0.1],
                   [list(items[3][0].ext[l].q) for l in range(3)], [list(items[3][0].ext[l].t) for l in range(3)])
    for g in (None, guess):
        want = LR.match(scans, 3, 1, a, guess=g)
        kw = {f: getattr(a, f) for f in ("max_iter", "eps_rot", "eps_pos", "min_points", "planarity", "sigma")}
        got = m.scan_store_match(3, 1, g, target_first=0, target_count=3, leaf=leaf, gate=gate, **kw)
        _check_exact(got, want)
        assert want["n_inliers"] > 100
    m.close()


def _recovery_case(seed=3):
    rng = np.random.default_rng(seed)
    scene = make_scene(rng, 80.0, 25)
    pos = [np.array([0.0, 0.0, 1.8]), np.array([3.0, 1.0, 1.8]), np.array([1.0, 2.0, 1.8])]
    items = []
    for k, p in enumerate(pos):
        st = _state(q_yaw(0.3 * k), p)
        items.append((st, raycast(scene, p, 0.3 * k, np.array([1.0, 0, 0, 0]), rng, beams=32, az=720, tmax=60.0)))
    return items


BASIN = [(0.5, 2.0), (1.0, 3.0), (2.0, 5.0)]   # (metres, degrees) offsets of the guess recovered


@pytest.mark.parametrize("offset", BASIN)
def test_recovery_from_offset_guesses(offset):
    items = _recovery_case()
    m = plugin.MeasurementModel(1)
    _store(m, 1, items)
    rng = np.random.default_rng(int(offset[0] * 10))
    truth = items[2][0]
    for trial in range(4):
        d = rng.normal(size=3)
        d[2] *= 0.3
        d *= offset[0] / np.linalg.norm(d)
        yaw = math.radians(offset[1]) * (1 if trial % 2 else -1)
        g = _state(LR.q_mul(list(q_yaw(yaw)), list(truth.rot)), np.array(truth.pos[:]) + d)
        r = m.scan_store_match(2, 0, g, target_first=0, target_count=2)
        assert np.abs(r["pos"] - np.array(truth.pos[:])).max() < 0.05, (offset, trial, r["pos"], r["fitness"])
        dq = LR.q_mul([truth.rot[0], -truth.rot[1], -truth.rot[2], -truth.rot[3]], list(r["rot"]))
        assert 2 * math.degrees(math.asin(min(1.0, np.linalg.norm(dq[1:])))) < 0.2
        assert plugin.accept_edge(r), r
    m.close()


def test_runs_repeat_refusals_change_nothing_and_device_bytes_stay():
    items = _recovery_case()
    m = plugin.MeasurementModel(1)
    _store(m, 1, items)
    recs = [bytes(r) for r in m.scan_store_records()]
    store = m.scan_store_info()
    r1 = m.scan_store_match(2, 0, target_first=0, target_count=2)
    r2 = m.scan_store_match(2, 0, target_first=0, target_count=2)
    for k in r1:
        _same(np.asarray(r1[k]), np.asarray(r2[k]), k)
    assert r1["device_bytes"] > 0
    assert m.scan_store_info() == store and [bytes(r) for r in m.scan_store_records()] == recs
    lib, h = m.lib, m._h
    rep = capi.MatchReport()

    def raw(source=2, anchor=0, guess=None, **kw):
        a = plugin.match_args(**{"target_first": 0, "target_count": 2, **kw})
        return lib.malio_scan_store_match(h, source, anchor, None if guess is None else C.byref(guess), C.byref(a), C.byref(rep))

    bad = [dict(source=3), dict(anchor=3), dict(target_count=0), dict(target_first=2, target_count=2), dict(anchor=2),
           dict(leaf=(0.0,), gate=(1.0,)), dict(leaf=(1.0,), gate=(float("nan"),)), dict(leaf=(1.0,), gate=(-1.0,)),
           dict(sigma=0.0), dict(planarity=float("inf")), dict(max_iter=0),
           dict(guess=_state([float("nan"), 0, 0, 0], [0, 0, 0]))]
    for kw in bad:
        assert raw(**kw) == capi.ERR_INVALID_ARG, kw
    a = plugin.match_args(0, 2)
    a.n_levels = 0
    assert lib.malio_scan_store_match(h, 2, 0, None, C.byref(a), C.byref(rep)) == capi.ERR_INVALID_ARG
    a.n_levels = capi.MATCH_MAX_LEVELS + 1
    assert lib.malio_scan_store_match(h, 2, 0, None, C.byref(a), C.byref(rep)) == capi.ERR_INVALID_ARG
    assert raw(leaf=(1e-6,), gate=(1.0,)) == capi.ERR_CAPACITY   # keys beyond 2^20 at a micrometre leaf
    assert m.scan_store_info() == store and [bytes(r) for r in m.scan_store_records()] == recs
    r3 = m.scan_store_match(2, 0, target_first=0, target_count=2)
    _same(r3["info"], r1["info"], "after refusals")
    m.close()


LIFT = np.array([0.0, 0.0, 0.25])   # the drive's world moved up by half a leaf: the ground lies inside a voxel layer, not on a face


def _block_drive(seed=5, n=48, radius=25.0):
    """A ray-cast drive around a block back to its start: n poses on a circle, the last near the first.  The world is lifted by
    LIFT, so that the ground (z = 0 in the ray cast) does not sit on a face of the 0.5 m voxel grid, where its range noise
    would split it over two voxel layers under the true states only."""
    rng = np.random.default_rng(seed)
    scene = make_scene(rng, 90.0, 30)
    scene["c"][0] = (0.0, 0.0)
    scene["size"][0] = (20.0, 20.0)
    items = []
    for k in range(n):
        t = 2 * math.pi * k / (n - 2)
        p = np.array([radius * math.cos(t), radius * math.sin(t), 1.8])
        pw = raycast(scene, p, t + math.pi / 2, np.array([1.0, 0, 0, 0]), rng, beams=24, az=600, tmax=50.0)
        items.append((_state(q_yaw(t + math.pi / 2), p + LIFT), pw + LIFT))
    return items


def _voxel_keys(m, leaf):
    """The voxel keys of the map's centroids (a centroid lies in its voxel)."""
    c = m.voxel_map_tensor().cpu().numpy()[:, :3].astype(np.float64)
    return set(map(tuple, np.floor(c / leaf).astype(np.int64)))


def _angle_deg(a, b):
    dq = LR.q_mul([a.rot[0], -a.rot[1], -a.rot[2], -a.rot[3]], list(b.rot))
    return 2 * math.degrees(math.asin(min(1.0, np.linalg.norm(dq[1:]))))


def test_close_loops_then_rebuild_corrects_a_drifted_drive(tmp_path):
    items = _block_drive()
    n = len(items)
    rng = np.random.default_rng(9)
    true = [s for s, _ in items]
    drift, walk_p, walk_y = [], np.zeros(3), 0.0
    for k, s in enumerate(true):
        if k:
            walk_p = walk_p + rng.normal(scale=[0.03, 0.03, 0.005])
            walk_y += rng.normal(scale=0.002)
        q = LR.q_mul(list(q_yaw(walk_y)), list(s.rot))
        drift.append(_state(q, np.array(LR.q_rot(list(q_yaw(walk_y)), list(s.pos[:]))) + walk_p))
    m = plugin.MeasurementModel(1)
    for (s, pw), d in zip(items, drift):
        body = _sensor(pw, 1, s, None)
        _put(m, 1, d, body)
    res = plugin.close_loops(m, radius=8.0, min_gap=20, stride=1, half_window=4)
    assert len(res["edges"]) >= 3, [(r["anchor"], r["source"], r["fitness"], r["rms"], r["eig_min"]) for r in res["reports"]]
    err_before = max(np.linalg.norm(np.array(d.pos[:]) - np.array(t.pos[:])) for d, t in zip(drift, true))
    # the trajectory's frame is node 0's: compare relative to it
    err_after = max(np.linalg.norm(np.array(c.pos[:]) - np.array(t.pos[:])) for c, t in zip(res["states"], true))
    print(f"close_loops: {len(res['edges'])} edges of {len(res['reports'])} candidates, max position error "
          f"{err_before:.3f} -> {err_after:.3f} m")
    print("edges (anchor, source, fitness, rms, eig_min):",
          [(e["a"], e["b"], round(e["fitness"], 3), round(e["rms"], 4), f"{e['eig_min']:.3g}") for e in res["edges"]])
    # a loop at the end of the drive fixes the end; the middle keeps part of the random walk's excursion
    loop_nodes = sorted({e["b"] for e in res["edges"]})
    err_loop = max(np.linalg.norm(np.array(res["states"][k].pos[:]) - np.array(true[k].pos[:])) for k in loop_nodes)
    before_loop = max(np.linalg.norm(np.array(drift[k].pos[:]) - np.array(true[k].pos[:])) for k in loop_nodes)
    rot_loop = max(_angle_deg(true[k], res["states"][k]) for k in loop_nodes)
    rot_before = max(_angle_deg(true[k], drift[k]) for k in loop_nodes)
    print(f"loop nodes {loop_nodes}: position error {before_loop:.3f} -> {err_loop:.3f} m, heading {rot_before:.2f} -> {rot_loop:.2f} deg")
    assert err_loop < 0.1 and rot_loop < 0.3 and err_after < 0.7 * err_before
    assert before_loop > 0.5 and rot_before > 1.0   # the drift the closure undoes
    # The map where the loop closes: the first and last scans of the drive rebuilt under each trajectory.  The drifted states
    # double its walls (more voxels, a small overlap with the true-state map); the closed states bring both back.
    leaf, region = 0.5, [(0, 5), (n - 6, 6)]
    maps = {}
    for name, states in (("true", true), ("drifted", drift), ("closed", res["states"])):
        if m.voxel_map_info()["n_voxels"]:
            m.voxel_map_save(str(tmp_path / "map.pcd"), clear=True)
        for first, count in region:
            m.voxel_map_rebuild(leaf, states=states[first:first + count], first=first, count=count)
        maps[name] = _voxel_keys(m, leaf)
    t = maps["true"]
    grow = {k: len(v) / len(t) - 1.0 for k, v in maps.items()}
    jac = {k: len(v & t) / len(v | t) for k, v in maps.items()}
    print("loop region voxels:", {k: len(v) for k, v in maps.items()}, "growth", grow, "overlap with the true map", jac)
    assert grow["drifted"] > 0.08 and abs(grow["closed"]) < 0.05
    assert jac["drifted"] < 0.55 and jac["closed"] > 0.7
    m.close()


def test_a_corridor_is_degenerate_and_rejected():
    rng = np.random.default_rng(4)
    scene = dict(half=200.0, c=np.array([[0.0, 6.0], [0.0, -6.0]]), size=np.array([[400.0, 1.0], [400.0, 1.0]]),
                 h=np.array([6.0, 6.0]), yaw=np.zeros(2))
    items = []
    for k in range(3):
        p = np.array([4.0 * k, 0.0, 1.8])
        items.append((_state(q_yaw(0.0), p), raycast(scene, p, 0.0, np.array([1.0, 0, 0, 0]), rng, beams=24, az=600, tmax=40.0)))
    m = plugin.MeasurementModel(1)
    _store(m, 1, items)
    r = m.scan_store_match(2, 0, target_first=0, target_count=2)
    good = _recovery_case()
    m2 = plugin.MeasurementModel(1)
    _store(m2, 1, good)
    g = m2.scan_store_match(2, 0, target_first=0, target_count=2)
    print(f"eig_min corridor {r['eig_min']:.3g} ({plugin.constraint(r):.3g} per inlier), street {g['eig_min']:.3g} "
          f"({plugin.constraint(g):.3g} per inlier)")
    assert plugin.constraint(r) < plugin.ACCEPT_CONSTRAINT < plugin.constraint(g)
    assert plugin.constraint(r) < 0.2 * plugin.constraint(g)
    assert not plugin.accept_edge(r)
    res = plugin.close_loops(m, radius=10.0, min_gap=2, half_window=0)
    assert res["reports"] and not res["edges"]
    m.close()
    m2.close()
