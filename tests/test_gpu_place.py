"""Relocalization without a position guess on the device (malio_place_db_build, malio_relocalize_global), against the numpy
restatement (tests/place_ref.py):
  - the database: positions, z_s, nibbles and ring keys bit-identical on seeded priors (a scene of buildings, the scene 1e5 m
    from the origin, points on column faces, a single column, an empty prior, the level cap on and off);
  - the query descriptor with 1-3 LiDARs and temporal compensation; the stage-1 and stage-2 lists, ties included (a prior holding
    two identical copies of a block); stage 3 equal to malio_relocalize called by hand on every candidate;
  - recovery: 20 ray-cast scans (a spinning pattern, occlusion included) at random free poses of an aperiodic 500 m scene, with
    random yaw and the true tilt, found within one lattice step and one yaw step; after the window and two IESKF updates the
    median error is within 0.1 m and 0.25 degrees and every scan within 0.5 m and 0.5 degrees;
  - nothing else changes, refusals leave a later call as on a fresh handle, two runs repeat, device bytes within the limits."""
import ctypes as C
import math

import numpy as np
import pytest

import place_ref as PR
from malio_b200 import capi, plugin, synth
from test_gpu_relocalize import _extrinsics, make_scene, q_yaw, sample_scene, scan_of

pytestmark = pytest.mark.gpu
F = np.float32
MAX_GRID_BYTES, MAX_DB_BYTES = 4 << 30, 8 << 30   # MALIO_PLACE_MAX_GRID_BYTES / _DB_BYTES
SMALL = dict(r_max=20.0, n_ring=5, n_sector=12)


def _db_args(fov=None, **kw):
    a = dict(SMALL)
    a.update(kw)
    if fov is not None:
        a["fov_up"] = math.radians(fov)
    return plugin.MeasurementModel.place_args(1.8, **a)


def _check_db(m, prior, args):
    rep = m.place_db_build(args=args)
    want = PR.database(prior, args)
    got = m.place_db_download(args.n_ring, args.n_sector)
    assert rep["n_positions"] == len(want["cols"]) == m.place_db_info()["n_positions"]
    assert np.array_equal(got["cols"].astype(np.int64), want["cols"])
    assert got["z_s"].tobytes() == want["z_s"].tobytes()
    assert np.array_equal(got["nibbles"], PR.pack(want["levels"]))
    assert np.array_equal(got["ring_keys"].astype(np.int64), want["ring_keys"])
    assert rep["device_bytes"] <= MAX_DB_BYTES and rep["scratch_bytes"] <= MAX_GRID_BYTES + (1 << 24)
    return rep, want


def _priors():
    rng = np.random.default_rng(11)
    scene = make_scene(rng, 40.0, 8)
    base = sample_scene(scene, rng, 1.0)
    faces = rng.integers(-30, 30, (3000, 3)).astype(np.float64)            # every coordinate on a column face
    faces[:, 2] = rng.uniform(-1, 12, 3000)
    single = np.column_stack([np.full(7, 4.25), np.full(7, 6.5), np.linspace(0.0, 9.0, 7)])
    return [("scene", base, None, 2), ("scene-cap", base, 15.0, 2), ("scene-open", base, 15.0, 0),
            ("far", base + np.array([1e5, -1e5, 0.0]), 20.0, 3), ("faces", faces, None, 2), ("single", single, None, 2),
            ("empty", np.zeros((0, 3)), None, 2)]


def test_database_is_bit_identical_to_the_restatement():
    m = plugin.MeasurementModel(1)
    for name, prior, fov, block in _priors():
        prior = prior.astype(F)
        m.prior_map_load(prior)
        rep, want = _check_db(m, prior, _db_args(fov, block_level=block))
        if name == "empty":
            assert rep["n_positions"] == 0
        elif name == "single":
            assert rep["n_positions"] == 1 and want["levels"].sum() == 0
        else:
            assert rep["n_positions"] > 50 and want["levels"].max() >= 3, name
        if name == "scene-cap":
            assert want["levels"].max() < 15
        if name == "scene-open":                   # without occlusion the rings behind a wall keep their values
            assert want["levels"].sum() > prev["levels"].sum()
        prev = want
        print(name, rep)
    m.close()


# ------------------------------------------------------------------ query and ranking
def _instance(seed, L, twin=False):
    rng = np.random.default_rng(300 + seed)
    extq, extt, tc = _extrinsics(rng, L)
    scene = make_scene(rng, 30.0, 6)
    prior = sample_scene(scene, rng, 1.5)
    if twin:                                       # two identical copies of the block: identical descriptors, stage ties
        prior = np.concatenate([prior, prior + np.array([90.0, 0.0, 0.0])])
    tilt = synth.q_exp(np.array([rng.normal(0, 0.05), rng.normal(0, 0.05), 0.0]))
    truth = np.array([rng.uniform(-10, 10), rng.uniform(-10, 10), 1.8])
    rot = synth.q_mul(q_yaw(rng.uniform(0, 2 * np.pi)), tilt)
    pw = sample_scene(scene, rng, 1.0, truth[:2], 22.0)
    pts, table, table_off = scan_of(pw[rng.permutation(len(pw))[:3000]], rng, truth, rot, extq, extt, tc)
    guess = synth.make_state(rng.normal(0, 50, 3), synth.q_mul(q_yaw(rng.uniform(0, 6.3)), tilt), extq, extt)
    return dict(prior=prior.astype(F), pts=pts, table=table, table_off=table_off, tc=tc, guess=guess, L=L)


def _model(case, args):
    m = plugin.MeasurementModel(case["L"])
    m.prior_map_load(case["prior"])
    m.place_db_build(args=args)
    m.upload_scan(case["pts"], case["table"], case["table_off"], case["tc"])
    return m


@pytest.mark.parametrize("seed,L,twin", [(0, 1, False), (1, 2, False), (2, 3, False), (3, 1, True), (4, 2, True)])
def test_query_and_candidates_equal_the_restatement(seed, L, twin):
    case = _instance(seed, L, twin)
    args = _db_args(25.0)
    m = _model(case, args)
    k1, k2 = 48, 6
    r = m.relocalize_global(case["guess"], k1=k1, k2=k2, res=1.0, half_xy=2, half_z=1)
    q, qk = PR.query(case["guess"], case["tc"], case["pts"], args)
    nb = args.n_ring * args.n_sector
    assert np.array_equal(r["query"][:nb].astype(np.int64), q) and not r["query"][nb:].any()
    db = PR.database(case["prior"], args)
    surv, d1 = PR.stage1(qk, db["ring_keys"], k1)
    assert np.array_equal(r["stage1"], surv) and np.array_equal(r["stage1_d1"], d1)
    p2, d2, sh = PR.stage2(q, db["levels"], surv, args, k2)
    got = [(c["position"], c["d2"], c["shift"]) for c in r["cand"]]
    assert got == list(zip(p2.tolist(), d2.tolist(), sh.tolist()))
    if twin:
        assert len(set(d1.tolist())) < len(d1) and len(set(r["stage1_d1"].tolist())) < k1
    # stage 3: malio_relocalize by hand on every candidate, the best by score, ties to the lower rank
    n_yaw, yaw_lo = PR.verify_args(args.n_sector, math.radians(1.0))
    assert (r["verify"]["n_yaw"], r["verify"]["yaw_lo"]) == (n_yaw, yaw_lo)
    best = None
    for k, c in enumerate(r["cand"]):
        g = PR.verification_guess(case["guess"], db["cols"][c["position"]], db["z_s"][c["position"]], c["shift"], args)
        assert np.array(g.rot[:]).tobytes() == c["guess_rot"].tobytes() and np.array(g.pos[:]).tobytes() == c["guess_pos"].tobytes()
        h = m.relocalize(g, 1.0, 2, 1, n_yaw=n_yaw, yaw_lo=yaw_lo, yaw_step=math.radians(1.0))
        assert (h["score"], h["n_points"]) == (c["score"], c["n_points"])
        assert h["rot"].tobytes() == c["rot"].tobytes() and h["pos"].tobytes() == c["pos"].tobytes()
        if best is None or h["score"] > best[1]["score"]:
            best = (k, h)
    assert r["best_rank"] == best[0] and r["score"] == best[1]["score"] and r["pos"].tobytes() == best[1]["pos"].tobytes()
    assert r["rot"].tobytes() == best[1]["rot"].tobytes()
    m.close()


# ------------------------------------------------------------------ recovery from ray-cast scans
def _boxes_hit(o, d, scene, tmax):
    """Nearest hit parameter of rays o + t d (d unit, [n, 3]) with the ground z = 0 and the scene's turned boxes; inf for none."""
    t = np.full(len(d), np.inf)
    g = d[:, 2] < -1e-9
    t[g] = -o[2] / d[g, 2]
    near = np.hypot(scene["c"][:, 0] - o[0], scene["c"][:, 1] - o[1]) < tmax + 25
    for (cx, cy), (sx, sy), h, yaw in zip(scene["c"][near], scene["size"][near], scene["h"][near], scene["yaw"][near]):
        c, s = math.cos(yaw), math.sin(yaw)
        ox, oy = (o[0] - cx) * c + (o[1] - cy) * s, -(o[0] - cx) * s + (o[1] - cy) * c
        dx, dy = d[:, 0] * c + d[:, 1] * s, -d[:, 0] * s + d[:, 1] * c
        lo, hi = np.full(len(d), -np.inf), np.full(len(d), np.inf)
        with np.errstate(divide="ignore", invalid="ignore"):
            for oo, dd, a, b in ((ox, dx, -sx / 2, sx / 2), (oy, dy, -sy / 2, sy / 2), (o[2], d[:, 2], 0.0, h)):
                t1, t2 = (a - oo) / dd, (b - oo) / dd
                lo = np.maximum(lo, np.minimum(t1, t2))
                hi = np.minimum(hi, np.maximum(t1, t2))
        hit = (lo <= hi) & (lo > 0)
        t = np.where(hit & (lo < t), lo, t)
    t[t > tmax] = np.inf
    return t


def raycast(scene, origin, psi, tilt, rng, beams=32, az=900, fov=22.5, tmax=100.0):
    """A spinning pattern from origin: `beams` elevations in [-fov, fov] degrees, `az` azimuths, turned by the sensor's yaw and
    tilt; world hit points (float64 [n, 3]) with 2 cm range noise."""
    el = np.deg2rad(np.linspace(-fov, fov, beams))
    a = np.linspace(0, 2 * np.pi, az, endpoint=False) + rng.uniform(0, 2 * np.pi / az)
    E, A = np.meshgrid(el, a, indexing="ij")
    d = np.column_stack([(np.cos(E) * np.cos(A)).ravel(), (np.cos(E) * np.sin(A)).ravel(), np.sin(E).ravel()])
    d = d @ synth.q_to_R(synth.q_mul(q_yaw(psi), tilt)).T
    t = _boxes_hit(origin, d, scene, tmax)
    ok = np.isfinite(t)
    t = t[ok] + rng.normal(0, 0.02, ok.sum())
    return origin + d[ok] * t[:, None]


def _free(scene, p, margin=3.0):
    for (cx, cy), (sx, sy), yaw in zip(scene["c"], scene["size"], scene["yaw"]):
        c, s = math.cos(yaw), math.sin(yaw)
        x, y = (p[0] - cx) * c + (p[1] - cy) * s, -(p[0] - cx) * s + (p[1] - cy) * c
        if abs(x) < sx / 2 + margin and abs(y) < sy / 2 + margin:
            return False
    return True


def _angle_deg(q1, q2):
    dq = synth.q_mul(synth.q_conj(q1), q2)
    return np.rad2deg(2 * np.arcsin(min(1.0, np.linalg.norm(dq[1:]))))


def test_recovery_from_ray_cast_scans_without_a_guess():
    rng = np.random.default_rng(21)
    scene = make_scene(rng, 250.0, 140)
    prior = sample_scene(scene, rng, 3.0).astype(F)
    params = capi.default_params(1)
    m = plugin.MeasurementModel(1, params=params)
    m.prior_map_load(prior)
    db = m.place_db_build(1.8, fov_up=math.radians(22.5))
    print("database", db)
    extq, extt = [synth.q_exp([0.0, 0.05, 0.0])], [np.array([0.1, 0.0, 0.2])]
    found, lines, refined = 0, [], []
    for trial in range(20):
        while True:
            o = np.array([rng.uniform(-200, 200), rng.uniform(-200, 200), 1.8])
            if _free(scene, o):
                break
        tilt = synth.q_exp(np.array([rng.normal(0, 0.03), rng.normal(0, 0.03), 0.0]))
        psi = rng.uniform(0, 2 * np.pi)
        rot = synth.q_mul(q_yaw(psi), tilt)
        truth = o - synth.q_to_R(rot) @ extt[0]               # the state whose slot-0 origin sits at o
        pw = raycast(scene, o, psi, tilt, rng)
        pts, table, table_off = scan_of(pw, rng, truth, rot, extq, extt, None)
        guess = synth.make_state(np.zeros(3), tilt, extq, extt)
        if trial:                                  # a fresh window for this scan: reload the prior (which drops the database)
            m.prior_map_load(prior)
            assert m.place_db_info()["n_positions"] == 0
            assert m.place_db_build(1.8, fov_up=math.radians(22.5)) == db
        m.upload_scan(pts, table, table_off, None)
        r = m.relocalize_global(guess)
        ang = _angle_deg(r["rot"], rot)
        dpos = np.abs(r["pos"] - truth)
        ranks = [k for k, c in enumerate(r["cand"]) if np.hypot(*(np.array(c["col"]) + 0.5 - o[:2])) <= 2.0]
        lines.append(f"trial {trial}: score {r['score']}/{r['n_points']} rank {r['best_rank']} (near truth: {ranks}) "
                     f"err {dpos.max():.2f} m {ang:.2f} deg, rank {r['ms_rank']:.1f} ms verify {r['ms_verify']:.1f} ms")
        print(lines[-1], flush=True)
        assert ang <= 1.0 + 1e-6 and np.all(dpos[:2] <= 0.5 + 1e-9), lines[-1]
        found += 1
        x = r["state"]
        m.prior_map_window(x, 200.0, 30.0)
        m.upload_scan(pts, table, table_off, None)
        errs = []
        for _ in range(2):
            P = synth.init_P(23)
            rep = m.update_iterated_dyn_share_modified(x, P, 4)
            errs.append((np.linalg.norm(np.array(x.pos[:]) - truth), _angle_deg(np.array(x.rot[:]), rot)))
        print(f"  after one update {errs[0][0]:.3f} m {errs[0][1]:.3f} deg, after two {errs[1][0]:.3f} m {errs[1][1]:.3f} deg "
              f"(n_eff {rep.n_eff_last})", flush=True)
        refined.append(errs[1])
    # On these ray-cast scans two IESKF updates from the verified pose (within 0.5 m and 1 degree) do not always reach the
    # corridor test's 0.1 m / 0.25 degrees: measured on one H100, median 0.080 m / 0.195 deg, worst 0.345 m / 0.448 deg; more
    # updates keep shrinking the error.  The bound checked: the median within 0.1 m / 0.25 deg, every scan within 0.5 m / 0.5 deg.
    refined = np.array(refined)
    print("after two updates: median", np.median(refined, axis=0), "max", refined.max(axis=0))
    assert np.median(refined[:, 0]) < 0.1 and np.median(refined[:, 1]) < 0.25, refined
    assert refined[:, 0].max() < 0.5 and refined[:, 1].max() < 0.5, refined
    assert found == 20
    m.close()


# ------------------------------------------------------------------ nothing else changes
CHANGING = {"kernel_launches", "h2d_bytes", "d2h_bytes"}


def test_nothing_else_changes():
    case = _instance(5, 2)
    guess = synth.make_state(np.array([1.0, -2.0, 1.8]), case["guess"].rot[:], [np.array(e.q[:]) for e in case["guess"].ext[:2]],
                             [np.array(e.t[:]) for e in case["guess"].ext[:2]])
    runs = []
    for place in (False, True):
        m = plugin.MeasurementModel(2)
        m.prior_map_load(case["prior"])
        m.prior_map_window(guess, 60.0, 10.0)
        m.upload_scan(case["pts"], case["table"], case["table_off"], case["tc"])
        info0, c0, map0 = m.prior_map_info(), m.counters(), m.map_download()
        if place:
            m.place_db_build(args=_db_args(25.0))
            m.relocalize_global(case["guess"], k1=32, k2=4, res=1.0, half_xy=2, half_z=1)
        info1, c1, map1 = m.prior_map_info(), m.counters(), m.map_download()
        assert info1 == info0
        for f, _ in capi.Counters._fields_:
            if f in CHANGING:
                assert getattr(c1, f) >= getattr(c0, f), f
            else:
                assert getattr(c1, f) == getattr(c0, f), f
        for k in map0:
            assert np.array_equal(map0[k], map1[k]), k
        x, P = guess.copy(), synth.init_P(17 + 6 * 2)
        rep = m.update_iterated_dyn_share_modified(x, P, 4)
        runs.append((synth.state_to_vec(x, 2).tobytes(), P.tobytes(), rep.passes, {k: v.tobytes() for k, v in map1.items()}, info1))
        m.close()
    assert runs[0] == runs[1]


# ------------------------------------------------------------------ refusals and determinism
def _key(r):
    out = {}
    for k, v in r.items():
        if k in ("state", "ms_rank", "ms_verify"):
            continue
        if k == "cand":
            v = [{kk: (vv.tobytes() if isinstance(vv, np.ndarray) else vv) for kk, vv in c.items()} for c in v]
        out[k] = v.tobytes() if isinstance(v, np.ndarray) else v
    return out


def _graw(m, s, k1=32, k2=4, yaw_step=math.radians(1.0), res=1.0, half_xy=2, half_z=1):
    a = capi.GlobalArgs()
    a.k1, a.k2, a.yaw_step, a.res, a.half_xy, a.half_z = k1, k2, yaw_step, res, half_xy, half_z
    return m.lib.malio_relocalize_global(m._h, C.byref(s), C.byref(a), C.byref(capi.GlobalReport()))


def test_refusals_leave_a_later_call_as_on_a_fresh_handle_and_runs_repeat():
    case = _instance(6, 2)
    args = _db_args(25.0)
    kw = dict(k1=32, k2=4, res=1.0, half_xy=2, half_z=1)
    fresh = _model(case, args)
    want_db = fresh.place_db_download(args.n_ring, args.n_sector)
    want = _key(fresh.relocalize_global(case["guess"], **kw))
    assert _key(fresh.relocalize_global(case["guess"], **kw)) == want
    assert 0 < want["device_bytes"] <= MAX_GRID_BYTES + MAX_DB_BYTES + (6 << 30)
    fresh.close()
    s = case["guess"].pass_state()
    m = plugin.MeasurementModel(2)
    rep = capi.PlaceDbReport()
    assert m.lib.malio_place_db_build(m._h, C.byref(args), C.byref(rep)) == capi.ERR_STATE          # no prior
    assert _graw(m, s) == capi.ERR_STATE
    m.prior_map_load(case["prior"])
    assert _graw(m, s) == capi.ERR_STATE                                                             # no database
    bad = [dict(cell=0.0), dict(cell=np.nan), dict(step=1.5), dict(step=0.0), dict(r_max=-1.0), dict(n_ring=0), dict(n_sector=10),
           dict(n_sector=0), dict(n_ring=64, n_sector=128), dict(dz=0.0), dict(fov_up=np.nan), dict(r_max=300.0)]
    for b in bad:
        a = _db_args(**b)
        assert m.lib.malio_place_db_build(m._h, C.byref(a), C.byref(rep)) == capi.ERR_INVALID_ARG, b
    for b in (dict(cell=1e-3, step=2e-3, r_max=0.1), dict(cell=1e-6, step=1e-6, r_max=1e-5)):                 # grid bytes / column indices
        a = _db_args(**b)
        far = case["prior"] + np.array([2e3, 0, 0], F) if b["cell"] < 1e-5 else case["prior"]
        m.prior_map_load(far)
        assert m.lib.malio_place_db_build(m._h, C.byref(a), C.byref(rep)) == capi.ERR_CAPACITY, b
        assert m.place_db_info()["n_positions"] == 0
    m.prior_map_load(case["prior"])
    m.place_db_build(args=args)
    assert _graw(m, s) == capi.ERR_STATE                                                             # no scan
    m.upload_scan(case["pts"], case["table"], case["table_off"], case["tc"])
    lib, h = m.lib, m._h
    ga = capi.GlobalArgs()
    assert lib.malio_relocalize_global(h, None, C.byref(ga), C.byref(capi.GlobalReport())) == capi.ERR_INVALID_ARG
    for b in (dict(k1=0), dict(k2=0), dict(k1=4, k2=8), dict(k1=2000), dict(k2=40, k1=64), dict(yaw_step=0.0), dict(yaw_step=np.nan),
              dict(res=0.0)):
        assert _graw(m, s, **b) == capi.ERR_INVALID_ARG, b
    got_db = m.place_db_download(args.n_ring, args.n_sector)
    assert all(np.array_equal(got_db[k], want_db[k]) for k in want_db)
    assert _key(m.relocalize_global(case["guess"], **kw)) == want
    info = m.place_db_info()
    m.prior_map_clear()
    assert m.place_db_info() == dict(n_positions=0, device_bytes=0) and info["n_positions"] > 0
    assert _graw(m, s) == capi.ERR_STATE
    m.close()
