"""Relocalization in a loaded prior map on the device (malio_relocalize), against the numpy restatement (tests/reloc_ref.py):
  - exactness: yaw index, offset, score, n_points, rotation and position equal the exhaustive search on 32 seeded instances
    (lattices that are not powers of two, half_z = 0, n_yaw = 1, a prior at +-1e5 m, a box reaching past the prior, 2-3 LiDARs
    with temporal compensation, a 90-degree symmetric scene, a ground-only prior, an empty prior);
  - recovery: scans rendered from an aperiodic scene of buildings at random poses are found within one yaw step and one lattice
    step, and the window plus two IESKF updates from there land within 0.1 m and 0.25 degrees of the truth;
  - nothing else changes: the device map, the prior's info, the counters other than launches and bytes, and the next IESKF
    update are those of a handle that never relocalized;
  - refusals leave a later call giving the fresh-handle answer, two runs give identical reports, device_bytes within the limits."""
import ctypes as C
import math

import numpy as np
import pytest

import reloc_ref as RR
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
MAX_PYRAMID_BYTES, MAX_INDEX_BYTES = 2 << 30, 4 << 30   # MALIO_RELOC_MAX_PYRAMID_BYTES / _INDEX_BYTES


# ------------------------------------------------------------------ an aperiodic scene: buildings of random place, size and heading
def make_scene(rng, half, n_build):
    """Ground z = 0 over [-half, half]^2 and n_build boxes: centre, footprint 6-30 m a side, height 5-40 m, heading uniform."""
    return dict(half=half, c=rng.uniform(-half, half, (n_build, 2)), size=rng.uniform(6, 30, (n_build, 2)),
                h=rng.uniform(5, 40, n_build), yaw=rng.uniform(0, 2 * np.pi, n_build))


def sample_scene(scene, rng, density, center=None, radius=None):
    """Uniform points on the ground and on the buildings' walls and roofs, `density` per m^2 (float64 [n, 3]); with center /
    radius only those within radius (horizontal) of center."""
    half = scene["half"]
    parts = []
    if center is None:
        gx0, gx1, gy0, gy1 = -half, half, -half, half
    else:
        gx0, gx1 = max(-half, center[0] - radius), min(half, center[0] + radius)
        gy0, gy1 = max(-half, center[1] - radius), min(half, center[1] + radius)
    n = rng.poisson(density * max(gx1 - gx0, 0) * max(gy1 - gy0, 0))
    parts.append(np.column_stack([rng.uniform(gx0, gx1, n), rng.uniform(gy0, gy1, n), np.zeros(n)]))
    for (cx, cy), (sx, sy), h, yaw in zip(scene["c"], scene["size"], scene["h"], scene["yaw"]):
        if center is not None and math.hypot(cx - center[0], cy - center[1]) > radius + 30:
            continue
        R = np.array([[math.cos(yaw), -math.sin(yaw)], [math.sin(yaw), math.cos(yaw)]])
        faces = []   # (origin, u, v) in the building frame, u / v spans
        for sgn in (-1, 1):
            faces.append(((sgn * sx / 2, -sy / 2, 0), (0, sy, 0), (0, 0, h)))
            faces.append(((-sx / 2, sgn * sy / 2, 0), (sx, 0, 0), (0, 0, h)))
        faces.append(((-sx / 2, -sy / 2, h), (sx, 0, 0), (0, sy, 0)))
        for o, u, v in faces:
            o, u, v = np.array(o), np.array(u), np.array(v)
            k = rng.poisson(density * np.linalg.norm(u) * np.linalg.norm(v))
            p = o + rng.random((k, 1)) * u + rng.random((k, 1)) * v
            p[:, :2] = p[:, :2] @ R.T + (cx, cy)
            parts.append(p)
    p = np.concatenate(parts)
    if center is not None:
        p = p[np.hypot(p[:, 0] - center[0], p[:, 1] - center[1]) <= radius]
    return p


def q_yaw(psi):
    return np.array([math.cos(psi / 2), 0.0, 0.0, math.sin(psi / 2)])


def _extrinsics(rng, L):
    extq = [synth.q_exp(synth.rand_unit(rng) * 0.2) for _ in range(L)]
    extt = [rng.normal(0, 0.3, 3) for _ in range(L)]
    tc = None
    if L > 1:
        tc = np.zeros(L - 1, capi.RIGID)
        for l in range(1, L):
            tc[l - 1]["q"] = synth.q_exp(synth.rand_unit(rng) * 0.05)
            tc[l - 1]["t"] = rng.normal(0, 0.1, 3)
    return extq, extt, tc


def scan_of(pw, rng, pos, rot, extq, extt, tc):
    """World points -> scan records seen from (pos, rot), LiDARs round-robin, with pose tables of two entries each."""
    L = len(extq)
    lidar = np.arange(len(pw)) % L
    pts = np.zeros(len(pw), capi.SCAN_PT)
    pts["xyz"] = synth.world_to_sensor(pw, lidar, pos, rot, extq, extt, tc).astype(F)
    pts["lidar"] = lidar
    table, table_off = synth.make_tables(L, 2, rng)
    pts["table_idx"] = rng.integers(0, 2, len(pw))
    return pts, table, table_off


# ------------------------------------------------------------------ exactness against the exhaustive search
def _instance(seed, kind="scene", L=1, hxy=3, hz=1, n_yaw=12, res=1.0, offset=0.0, past=False):
    rng = np.random.default_rng(1000 + seed)
    extq, extt, tc = _extrinsics(rng, L)
    tilt = synth.q_exp(np.array([rng.normal(0, 0.05), rng.normal(0, 0.05), 0.0]))
    truth = np.array([rng.uniform(-5, 5), rng.uniform(-5, 5), 1.8])
    if kind == "scene":
        scene = make_scene(rng, 30.0, 6)
        prior = sample_scene(scene, rng, 2.0)
        pw = sample_scene(scene, rng, 1.0, truth[:2], 25.0)
        pw = pw[rng.permutation(len(pw))[:400]]
        if past:                                   # the prior ends at x = 0, the guess sits near that edge
            prior = prior[prior[:, 0] < 0]
            truth[0] = -2.0
    elif kind == "ground":                         # a plane with a point in every voxel: every xy offset (and yaw) ties
        g = np.arange(-60.0, 60.0, 0.25)
        gx, gy = np.meshgrid(g, g, indexing="ij")
        prior = np.column_stack([gx.ravel(), gy.ravel(), np.full(gx.size, 0.3)])
        pw = np.column_stack([rng.uniform(-20, 20, 300) + truth[0], rng.uniform(-20, 20, 300) + truth[1], np.full(300, 0.3)])
    elif kind == "empty":
        prior = np.zeros((0, 3))
        pw = rng.uniform(-20, 20, (300, 3))
    else:
        raise ValueError(kind)
    truth[:2] += offset
    prior = prior + np.array([offset, offset, 0.0])
    pw = pw + np.array([offset, offset, 0.0])
    psi = rng.uniform(0, 2 * np.pi)
    rot_true = synth.q_mul(q_yaw(psi), tilt)
    pts, table, table_off = scan_of(pw, rng, truth, rot_true, extq, extt, tc)
    guess = synth.make_state(truth + rng.uniform(-0.8, 0.8, 3) * res * np.array([hxy, hxy, hz]), tilt, extq, extt)
    yaw_lo = float(rng.uniform(-np.pi, np.pi))
    return dict(prior=prior.astype(F), pts=pts, table=table, table_off=table_off, tc=tc, guess=guess, L=L,
                args=dict(res=res, half_xy=hxy, half_z=hz, n_yaw=n_yaw, yaw_lo=yaw_lo, yaw_step=2 * np.pi / n_yaw))


def _symmetric(seed, n_yaw):
    """A scan invariant under 90-degree turns about the guess (points at voxel centres, exact in float), the prior its own points:
    yaws 0, 90, 180 and 270 degrees score the same, exactly."""
    rng = np.random.default_rng(2000 + seed)
    p = rng.integers(-15, 15, (60, 3)).astype(np.float64) + 0.5
    p[:, 2] = np.abs(p[:, 2])
    pw = np.concatenate([p, np.column_stack([-p[:, 1], p[:, 0], p[:, 2]]), np.column_stack([-p[:, 0], -p[:, 1], p[:, 2]]),
                         np.column_stack([p[:, 1], -p[:, 0], p[:, 2]])])
    extq, extt, tc = [np.array([1.0, 0, 0, 0])], [np.zeros(3)], None
    pts, table, table_off = scan_of(pw, rng, np.zeros(3), np.array([1.0, 0, 0, 0]), extq, extt, tc)
    guess = synth.make_state(np.zeros(3), np.array([1.0, 0, 0, 0]), extq, extt)
    return dict(prior=pw.astype(F), pts=pts, table=table, table_off=table_off, tc=tc, guess=guess, L=1,
                args=dict(res=1.0, half_xy=3, half_z=1, n_yaw=n_yaw, yaw_lo=0.0, yaw_step=2 * np.pi / n_yaw))


INSTANCES = (
    [("scene", dict(seed=s, L=1 + s % 3, hxy=(1, 2, 3, 5, 6, 4)[s % 6], hz=(0, 1, 2)[s % 3], n_yaw=(1, 7, 12, 24)[s % 4],
                    res=(0.5, 0.8, 1.0, 1.7)[s % 4])) for s in range(14)]
    + [("scene", dict(seed=20 + s, hxy=4, hz=0, n_yaw=1, res=0.9)) for s in range(2)]
    + [("scene", dict(seed=30 + s, L=2, hxy=20, hz=1, n_yaw=36, res=1.0, offset=(1e5, -1e5)[s % 2])) for s in range(4)]
    + [("scene", dict(seed=40 + s, L=3, hxy=10, hz=1, n_yaw=6, res=2.0, past=True)) for s in range(3)]
    + [("sym", dict(seed=50 + s, n_yaw=(8, 4, 12)[s])) for s in range(3)]
    + [("scene", dict(seed=60 + s, kind="ground", hxy=6, hz=1, n_yaw=6, res=1.0)) for s in range(2)]
    + [("scene", dict(seed=70 + s, kind="ground", hxy=5, hz=2, n_yaw=3, res=0.7, offset=1e5)) for s in range(1)]
    + [("scene", dict(seed=80 + s, kind="empty", L=1 + s, hxy=2, hz=1, n_yaw=5)) for s in range(2)]
)


def _model(case):
    m = plugin.MeasurementModel(case["L"])
    m.prior_map_load(case["prior"])
    m.upload_scan(case["pts"], case["table"], case["table_off"], case["tc"])
    return m


def _check_exact(case, r):
    a = case["args"]
    want = RR.relocalize(case["guess"], case["tc"], case["pts"], case["prior"], a["res"], a["half_xy"], a["half_z"], a["n_yaw"],
                         a["yaw_lo"], a["yaw_step"])
    got = (r["yaw_index"], r["offset"], r["score"], r["n_points"])
    assert got == (want["yaw_index"], want["offset"], want["score"], want["n_points"]), (got, want["score"])
    assert r["n_candidates"] == want["n_candidates"]
    assert r["rot"].tobytes() == want["rot"].tobytes() and r["pos"].tobytes() == want["pos"].tobytes()
    assert r["nodes_bounded"] >= r["leaves_scored"] >= (1 if want["score"] else 0)
    return want


def test_exact_against_the_exhaustive_search():
    assert len(INSTANCES) >= 30
    ratios = []
    for kind, kw in INSTANCES:
        case = _symmetric(**kw) if kind == "sym" else _instance(**kw)
        m = _model(case)
        r = m.relocalize(case["guess"], **case["args"])
        want = _check_exact(case, r)
        sc = want["scores"]
        if kind == "sym":                          # the exact yaw ties resolve to the smallest k
            q = case["args"]["n_yaw"] // 4
            assert r["yaw_index"] == 0 and all(sc[k].max() == sc.max() for k in (q, 2 * q, 3 * q)), kw
        if kw.get("kind") == "ground":             # every xy offset ties: the first one wins
            assert r["offset"][:2] == (-kw["hxy"], -kw["hxy"]) and r["yaw_index"] == 0 and r["score"] == case["pts"].shape[0], kw
        if kw.get("kind") == "empty":
            assert r["score"] == 0 and r["yaw_index"] == 0 and r["offset"] == (-kw["hxy"], -kw["hxy"], -kw["hz"])
        if kind == "scene" and kw.get("kind", "scene") == "scene" and r["n_candidates"] >= 100000:
            ratios.append(r["nodes_bounded"] / r["n_candidates"])
        m.close()
    # on lattices of 10^5 candidates and more the bound prunes most of them (below that, the inner nodes are as many as the leaves)
    print("nodes_bounded / n_candidates on the structured instances:", np.round(ratios, 4).tolist())
    assert len(ratios) == 4 and max(ratios) < 0.25, ratios


# ------------------------------------------------------------------ recovery from a guess without heading
def _recovery_scene():
    rng = np.random.default_rng(5)
    scene = make_scene(rng, 200.0, 90)
    return scene, sample_scene(scene, rng, 3.0).astype(F)


def _angle_deg(q1, q2):
    dq = synth.q_mul(synth.q_conj(q1), q2)
    return np.rad2deg(2 * np.arcsin(min(1.0, np.linalg.norm(dq[1:]))))


def test_recovery_from_a_guess_without_heading():
    scene, prior = _recovery_scene()
    res, hxy, hz, n_yaw = 1.0, 20, 2, 360
    params = capi.default_params(1)
    m = plugin.MeasurementModel(1, params=params)
    rng = np.random.default_rng(6)
    extq, extt = [synth.q_exp([0.0, 0.05, 0.0])], [np.array([0.1, 0.0, 0.2])]
    for trial in range(6):
        truth = np.array([rng.uniform(-100, 100), rng.uniform(-100, 100), 1.8])
        tilt = synth.q_exp(np.array([rng.normal(0, 0.03), rng.normal(0, 0.03), 0.0]))
        psi = rng.uniform(0, 2 * np.pi)
        rot = synth.q_mul(q_yaw(psi), tilt)
        pw = sample_scene(scene, rng, 2.0, truth[:2], 50.0)
        pw = pw[rng.permutation(len(pw))[:8000]] + rng.normal(0, 0.02, (min(len(pw), 8000), 3))
        pts, table, table_off = scan_of(pw, rng, truth, rot, extq, extt, None)
        guess = synth.make_state(truth + rng.uniform(-0.8, 0.8, 3) * res * np.array([hxy, hxy, hz]), tilt, extq, extt)
        m.prior_map_load(prior)
        m.upload_scan(pts, table, table_off, None)
        r = m.relocalize(guess, res, hxy, hz, n_yaw=n_yaw)
        dyaw = (r["yaw_index"] * 2 * np.pi / n_yaw - psi + np.pi) % (2 * np.pi) - np.pi
        assert abs(dyaw) <= 2 * np.pi / n_yaw + 1e-9, (trial, np.rad2deg(dyaw), r["score"], r["n_points"])
        assert np.all(np.abs(r["pos"] - truth) <= res + 1e-9), (trial, r["pos"] - truth, r["score"], r["n_points"])
        # the window at the result, then the IESKF update
        x = r["state"]
        m.prior_map_window(x, 200.0, 30.0)
        m.upload_scan(pts, table, table_off, None)
        # One update (4 iterations) from up to a lattice step and a yaw step off does not always reach the corridor test's bound
        # (0.075 - 0.131 m measured); a second update on the same scan, from the first one's estimate, does.
        errs = []
        for _ in range(2):
            P = synth.init_P(23)
            rep = m.update_iterated_dyn_share_modified(x, P, 4)
            errs.append((np.linalg.norm(np.array(x.pos[:]) - truth), _angle_deg(np.array(x.rot[:]), rot)))
        print(f"trial {trial}: score {r['score']}/{r['n_points']} nodes {r['nodes_bounded']}/{r['n_candidates']} "
              f"reloc err {np.abs(r['pos'] - truth).max():.2f} m {np.rad2deg(abs(dyaw)):.2f} deg; after one update "
              f"{errs[0][0]:.3f} m {errs[0][1]:.3f} deg, after two {errs[1][0]:.3f} m {errs[1][1]:.3f} deg (n_eff {rep.n_eff_last})")
        assert errs[1][0] < 0.1 and errs[1][1] < 0.25, (trial, errs)
    m.close()


# ------------------------------------------------------------------ nothing else changes
CHANGING = {"kernel_launches", "h2d_bytes", "d2h_bytes"}


def test_nothing_else_changes():
    case = _instance(3, L=2, hxy=5, hz=1, n_yaw=24, res=1.0)
    runs = []
    for relocalize in (False, True):
        m = plugin.MeasurementModel(2)
        m.prior_map_load(case["prior"])
        m.prior_map_window(case["guess"], 60.0, 10.0)
        m.upload_scan(case["pts"], case["table"], case["table_off"], case["tc"])
        info0, c0, map0 = m.prior_map_info(), m.counters(), m.map_download()
        if relocalize:
            m.relocalize(case["guess"], **case["args"])
        info1, c1, map1 = m.prior_map_info(), m.counters(), m.map_download()
        assert info1 == info0
        for f, _ in capi.Counters._fields_:
            if f in CHANGING:
                assert getattr(c1, f) >= getattr(c0, f), f
            else:
                assert getattr(c1, f) == getattr(c0, f), f
        for k in map0:
            assert np.array_equal(map0[k], map1[k]), k
        x, P = case["guess"].copy(), synth.init_P(17 + 6 * 2)
        rep = m.update_iterated_dyn_share_modified(x, P, 4)
        runs.append((synth.state_to_vec(x, 2).tobytes(), P.tobytes(), rep.passes, {k: v.tobytes() for k, v in map1.items()}, info1))
        m.close()
    assert runs[0] == runs[1]


# ------------------------------------------------------------------ refusals and determinism
def _raw(m, s, a):
    rep = capi.RelocReport()
    rc = m.lib.malio_relocalize(m._h, C.byref(s), C.byref(a), C.byref(rep))
    return rc, rep


def _args(res=1.0, half_xy=5, half_z=1, n_yaw=12, yaw_lo=0.3, yaw_step=2 * np.pi / 12):
    a = capi.RelocArgs()
    a.res, a.half_xy, a.half_z, a.n_yaw, a.yaw_lo, a.yaw_step = res, half_xy, half_z, n_yaw, yaw_lo, yaw_step
    return a


def _key(r):
    return {k: (v.tobytes() if isinstance(v, np.ndarray) else v) for k, v in r.items() if k != "state"}


def test_refusals_leave_a_later_call_as_on_a_fresh_handle_and_runs_repeat():
    case = _instance(7, L=2, hxy=5, hz=1, n_yaw=12, res=1.0)
    s = case["guess"].pass_state()
    fresh = _model(case)
    want = _key(fresh.relocalize(case["guess"], **case["args"]))
    assert _key(fresh.relocalize(case["guess"], **case["args"])) == want        # two runs: identical, nodes_bounded included
    assert want["device_bytes"] <= MAX_PYRAMID_BYTES + MAX_INDEX_BYTES and want["device_bytes"] > 0
    fresh.close()
    m = plugin.MeasurementModel(2)
    a = _args()
    assert _raw(m, s, a)[0] == capi.ERR_STATE                                    # no prior
    m.prior_map_load(case["prior"])
    assert _raw(m, s, a)[0] == capi.ERR_STATE                                    # no scan
    m.upload_scan(case["pts"], case["table"], case["table_off"], case["tc"])
    lib, h = m.lib, m._h
    rep = capi.RelocReport()
    assert lib.malio_relocalize(h, None, C.byref(a), C.byref(rep)) == capi.ERR_INVALID_ARG
    assert lib.malio_relocalize(h, C.byref(s), None, C.byref(rep)) == capi.ERR_INVALID_ARG
    assert lib.malio_relocalize(h, C.byref(s), C.byref(a), None) == capi.ERR_INVALID_ARG
    bad_args = [_args(n_yaw=0), _args(res=0.0), _args(res=-1.0), _args(res=np.nan), _args(res=np.inf), _args(yaw_lo=np.nan),
                _args(yaw_step=np.inf)]
    for b in bad_args:
        assert _raw(m, s, b)[0] == capi.ERR_INVALID_ARG
    for f, i in (("pos", 0), ("rot", 3)):
        sb = case["guess"].pass_state()
        getattr(sb, f)[i] = np.nan
        assert _raw(m, sb, a)[0] == capi.ERR_INVALID_ARG
    for b in (_args(n_yaw=1 << 20, half_xy=100),                                 # > 2^32 candidates
              _args(res=1e-3, half_xy=2, n_yaw=2),                               # the pyramid's box: > 2 GB
              _args(res=1e-8, half_xy=1, n_yaw=1)):                              # voxel indices beyond 2^30
        rc, _ = _raw(m, s, b)
        assert rc == capi.ERR_CAPACITY, (b.res, b.n_yaw, rc)
    c0 = m.counters()
    got = _key(m.relocalize(case["guess"], **case["args"]))
    assert got == want
    c1 = m.counters()
    assert c1.kernel_launches > c0.kernel_launches and c1.d2h_bytes > c0.d2h_bytes
    m.close()


def test_a_communicator_is_refused():
    case = _instance(8, L=1, hxy=2, hz=0, n_yaw=4)
    m = _model(case)
    try:
        m.comm_init(plugin.MeasurementModel.nccl_unique_id(), 0, 1)
    except capi.MalioError:
        m.close()
        pytest.skip("NCCL is not available")
    rc, _ = _raw(m, case["guess"].pass_state(), _args(half_xy=2, half_z=0, n_yaw=4))
    assert rc == capi.ERR_STATE
    m.close()
