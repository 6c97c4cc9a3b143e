"""Localization past the edge of a saved map (malio_prior_map_extend, the session layer), against the restatement
(tests/prior_extend_ref.py) fed with the device's own classes and world points (malio_map_incremental on the same state):
  - after every window and extend call of a scripted run (load, window, scans with extend, slides away from the extension and
    back, a reload, a malio_map_build in between) the window's live points equal (prior ∪ session) ∩ cube in xyz bits,
    normal_y, ids and slot order, and the session download equals the restated session;
  - with an empty session the window's reports, slot orders and launches are those of a run that never extends;
  - a drive of 450 m past the edge of a corridor prior keeps its planes with extend and loses them without;
  - refusals: no window, no pass, a bad filter_size_map, NULL state."""
import ctypes as C
from dataclasses import replace

import numpy as np
import pytest

import prior_extend_ref as E
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
DS = 0.5


def _corridor(rng, x0, x1, per_site=8000, half=None):
    """Ground and street-grid walls along x in [x0, x1] (sites every 50 m); the full scene's half extent is `half`."""
    sites = np.arange(x0, x1 + 1, 50.0)
    return np.concatenate([synth.sample_surfaces(per_site, (x, 0.0), 40.0, half, rng) for x in sites]).astype(F)


class Drive:
    """Scans rendered at known poses from the full scene (prior half + unmapped half)."""

    def __init__(self, length=1200.0, seed=21):
        rng = np.random.default_rng(seed)
        self.half = length / 2 + 100.0
        self.base = synth.make_case("corridor", 6000, 1000, 1, 4)
        self.extq = [np.array(self.base.x_true.ext[0].q[:])]
        self.extt = [np.array(self.base.x_true.ext[0].t[:])]
        self.rot = np.array(self.base.x_true.rot[:])
        self.rs = np.random.default_rng(seed + 1)

    def scan(self, pos, k):
        xt = synth.make_state(pos, self.rot, self.extq, self.extt)
        pw = synth.sample_surfaces(6000, pos[:2], 40.0, self.half, self.rs) + self.rs.normal(0, 0.02, (6000, 3))
        return synth.with_scan(replace(self.base, x_true=xt), pw, seed=k)

    def state(self, pos, rot=None):
        return synth.make_state(pos, self.rot if rot is None else rot, self.extq, self.extt)


def _check_window(m, W, k):
    mp = m.map_download() if m.map_info()[0] else dict(xyz=np.zeros((0, 3), F), normal_y=np.zeros(0, F), ids=np.zeros(0, np.int32))
    assert mp["xyz"].tobytes() == W.xyz.tobytes(), k
    assert mp["normal_y"].tobytes() == W.ny.tobytes(), k
    assert np.array_equal(mp["ids"], W.ids), k
    s = m.prior_map_session()
    assert s[:, :3].tobytes() == W.sxyz.tobytes(), k
    assert np.all(s[:, 3] == E.SESSION_NY), k


def _update(m, case, x):
    m.upload_scan(case.pts, case.table, case.table_off, None)
    P = synth.init_P(case.n_dof)
    return m.update_iterated_dyn_share_modified(x, P, 4)


def test_window_holds_prior_and_session_in_the_cube_after_every_call():
    d = Drive(length=600.0)
    prior = _corridor(np.random.default_rng(22), -400.0, 0.0, half=d.half)    # the prior ends near x = 40 (walls, ground)
    ids = np.arange(len(prior), dtype=np.int32) * 2
    m = plugin.MeasurementModel(1, params=d.base.params)
    m.prior_map_load(prior, np.full(len(prior), 0.001, F), ids)
    CUBE, DET = 160.0, 20.0       # thr 30 m, mov_dist 36 m
    W = E.SessionWindow(prior, np.full(len(prior), 0.001, F), ids, CUBE, DET)
    xs = [-40.0, -20.0, 0.0, 20.0, 40.0, 60.0, 80.0, 100.0, 120.0, 140.0, 160.0, 120.0, 80.0, 40.0, 0.0, -40.0, -80.0, -120.0,
          -80.0, -40.0, 0.0, 40.0, 80.0, 120.0, 160.0]
    moves, inserted = 0, 0
    for k, x in enumerate(xs):
        pos = np.array([x, 0.0, 1.8])
        if k == 14:                                   # a malio_map_build ends the window, not the session
            m.map_build(prior[:10], np.full(10, 0.001, F))
            W.end()
        if k == 18:                                   # a reload starts an empty session
            m.prior_map_load(prior, np.full(len(prior), 0.001, F), ids)
            W = E.SessionWindow(prior, np.full(len(prior), 0.001, F), ids, CUBE, DET)
        xs_ = d.state(pos)
        init, moved, slabs, n_in = W.step(plugin.pos_lid(xs_))
        r = m.prior_map_window(xs_, CUBE, DET)
        assert (r["initialized"], r["moved"]) == (init, moved), k
        assert np.array_equal(r["cube"], W.cube), k
        if init or moved:
            assert r["n_entered"] == n_in, k
        moves += moved
        _check_window(m, W, k)
        case = d.scan(pos, k)
        x_est = d.state(pos)
        rep = _update(m, case, x_est)
        if rep.n_eff_last == 0:
            continue                                  # no pass to extend from (the IESKF found nothing to hold on to)
        cls, world = m.map_incremental(x_est, DS, True)
        want = W.extend(cls, world, DS)
        got = m.prior_map_extend(x_est, DS)
        assert got == want, (k, got, want)
        inserted += got["n_inserted"]
        _check_window(m, W, k)
    assert moves >= 8 and inserted > 1000
    m.close()


def test_an_empty_session_changes_no_window_call():
    """Two handles drive inside the prior; one calls extend after every scan with 1 km voxels, each of which holds prior points
    of the window wherever the scans reach (a copy of the scene 0.3 m lower fills the voxels below the ground, which the scans'
    noise reaches), so nothing is admitted and its session stays empty.  Window reports, slot orders and the launches of every window
    call match those of the handle that never extends."""
    d = Drive(length=600.0)
    prior = _corridor(np.random.default_rng(23), -300.0, 300.0, per_site=12000, half=d.half)
    prior = np.concatenate([prior, prior - F([0.0, 0.0, 0.3])])
    hs = [plugin.MeasurementModel(1, params=d.base.params) for _ in range(2)]
    for m in hs:
        m.prior_map_load(prior, np.full(len(prior), 0.001, F))
    reps = [[], []]
    for k, x in enumerate([-100.0, -80.0, -60.0, -40.0, -20.0, 0.0, -40.0, -80.0]):
        pos = np.array([x, 0.0, 1.8])
        case = d.scan(pos, k)
        for j, m in enumerate(hs):
            c0 = m.counters().kernel_launches
            r = m.prior_map_window(d.state(pos), 160.0, 20.0)
            reps[j].append((r, m.counters().kernel_launches - c0, m.map_download()["ids"].copy()))
            x_est = d.state(pos)
            _update(m, case, x_est)
            if j == 1:
                e = m.prior_map_extend(x_est, 1000.0)
                assert e["n_candidates"] > 0 and e["n_session"] == 0
    for (ra, la, ia), (rb, lb, ib) in zip(*reps):
        assert la == lb
        assert np.array_equal(ia, ib)
        for key in ra:
            assert np.array_equal(ra[key], rb[key]), key
    for m in hs:
        m.close()


def _err(x, pos, rot):
    v = synth.state_to_vec(x, 1)
    dq = synth.q_mul(synth.q_conj(v[3:7]), rot)
    return float(np.linalg.norm(v[:3] - pos)), float(np.rad2deg(2 * np.arcsin(min(1.0, np.linalg.norm(dq[1:])))))


def _drive_past_the_edge(extend, xs, d, prior, stats):
    m = plugin.MeasurementModel(1, params=d.base.params)
    m.prior_map_load(prior, np.full(len(prior), 0.001, F))
    x = d.state(np.array([xs[0], 0.0, 1.8]))
    prev = np.array([xs[0], 0.0, 1.8])
    out = []
    far_ids = None
    for k, xv in enumerate(xs):
        pos = np.array([xv, 0.0, 1.8])
        v = synth.state_to_vec(x, 1)
        xp = synth.make_state(v[:3] + (pos - prev), v[3:7], d.extq, d.extt)      # previous estimate + the true motion
        prev = pos
        r = m.prior_map_window(xp, 200.0, 30.0)
        stats["slides"] += r["moved"]
        case = d.scan(pos, k)
        x = xp
        rep = _update(m, case, x)
        e, a = _err(x, pos, d.rot)
        out.append((xv, int(rep.n_eff_last), e, a))
        if extend and rep.n_eff_last > 0:
            m.prior_map_extend(x, DS)
        if extend and xv == max(xs):
            far_ids = set(m.map_download()["ids"].tolist())
        if extend and k == len(xs) - 1:
            stats["back_ids"] = m.map_download()["ids"]
            stats["far_ids"] = far_ids
            stats["session"] = len(m.prior_map_session())
        if not extend and rep.n_eff_last == 0:
            break
    m.close()
    return out


def test_localization_continues_past_the_edge_of_the_prior():
    """A corridor of 1.2 km (ground and the street grid's walls); only its western half (x <= 0) is the prior.  Scans 20 m
    apart drive from x = -100 to x = 460 (460 m past the prior's last wall site, several slides of a 200 m cube in unmapped
    ground) and back to x = -100; each prediction is the previous estimate plus the true motion.
    With extend every scan keeps at least 1000 effective points and the pose stays within 2 m and 1 deg of the truth: past the
    edge the session is mapped from the estimates themselves, so the error walks (an H100 run: at worst 0.71 m and 0.17 deg,
    at least 3557 effective points, 214 600 session points, 21 slides).  Without extend the same drive finds no effective point
    within 150 m of the edge (that run lost it at x = 100).  On the way back the session
    points inserted near the edge, which the window had dropped at the far end, are live again."""
    d = Drive(length=1200.0)
    prior = _corridor(np.random.default_rng(24), -700.0, 0.0, per_site=12000, half=d.half)
    out_x = list(np.arange(-100.0, 461.0, 20.0))
    xs = out_x + out_x[-2::-1]
    st = dict(slides=0)
    with_ext = _drive_past_the_edge(True, xs, d, prior, st)
    print("extend drive (x, n_eff, err m, err deg):", [(float(a), b, round(c, 4), round(e, 4)) for a, b, c, e in with_ext])
    print("max err m / deg:", max(r[2] for r in with_ext), max(r[3] for r in with_ext), "min n_eff:", min(r[1] for r in with_ext),
          "session:", st["session"], "slides:", st["slides"])
    for xv, n_eff, e, a in with_ext:
        assert n_eff > 1000, (xv, n_eff)
        assert e < 2.0 and a < 1.0, (xv, e, a)
    assert st["slides"] >= 8
    back = set(st["back_ids"].tolist())
    sess_back = {i for i in back if i < 0}
    assert sess_back and not (sess_back <= st["far_ids"])     # session points the far window had dropped are live again
    st2 = dict(slides=0)
    without = _drive_past_the_edge(False, xs, d, prior, st2)
    lost = [xv for xv, n_eff, _, _ in without if n_eff == 0]
    print("without extend, lost at x =", lost[:1])
    assert lost and lost[0] <= 150.0, without[-5:]


def test_refusals():
    d = Drive(length=600.0)
    prior = _corridor(np.random.default_rng(25), -200.0, 0.0, per_site=4000, half=d.half)
    m = plugin.MeasurementModel(1, params=d.base.params)
    lib, h = m.lib, m._h
    pos = np.array([-20.0, 0.0, 1.8])
    x = d.state(pos)
    ps = x.pass_state()
    rep = capi.ExtendReport()
    assert lib.malio_prior_map_extend(h, C.byref(ps), C.c_double(DS), C.byref(rep)) == capi.ERR_STATE      # no prior
    m.prior_map_load(prior, np.full(len(prior), 0.001, F))
    assert lib.malio_prior_map_extend(h, C.byref(ps), C.c_double(DS), C.byref(rep)) == capi.ERR_STATE      # no window
    m.prior_map_window(x, 160.0, 20.0)
    assert lib.malio_prior_map_extend(h, C.byref(ps), C.c_double(DS), None) == capi.ERR_STATE              # no pass
    case = d.scan(pos, 0)
    _update(m, case, x)
    ps = x.pass_state()
    for bad in (0.0, -0.5, float("nan"), float("inf")):
        assert lib.malio_prior_map_extend(h, C.byref(ps), C.c_double(bad), C.byref(rep)) == capi.ERR_INVALID_ARG, bad
    assert lib.malio_prior_map_extend(h, None, C.c_double(DS), C.byref(rep)) == capi.ERR_INVALID_ARG
    assert m.prior_map_session().shape == (0, 4)
    m.map_build(prior[:10], np.full(10, 0.001, F))                                                          # window ended
    assert lib.malio_prior_map_extend(h, C.byref(ps), C.c_double(DS), C.byref(rep)) == capi.ERR_STATE
    m.prior_map_window(x, 160.0, 20.0)
    m.upload_scan(case.pts, case.table, case.table_off, None)
    assert lib.malio_prior_map_extend(h, C.byref(ps), C.c_double(DS), C.byref(rep)) == capi.ERR_STATE      # scan without a pass
    m.prior_map_clear()
    n = C.c_uint64(7)
    assert lib.malio_prior_map_session_download(h, None, 0, C.byref(n)) == capi.ERR_STATE
    m.close()


def test_slides_do_not_grow_scratch_with_the_session():
    """A slide tests every session point (the session has no tile index), but its output scratch is sized by the points that
    enter, not by the session: two handles with the same prior and the same slides, one holding a session of ~60 k points
    outside the cube, grow their device bytes over the slides by the same amount up to the block counts (8 B per 1024 session
    points), far below the 25 B per session point a candidate-sized scratch would take."""
    base = synth.make_case("ground scans", 1000, 1000, 1, 3)
    gx, gy = np.meshgrid(np.arange(-180.0, 0.0, 0.5), np.arange(-100.0, 100.0, 0.5), indexing="ij")
    prior = np.column_stack([gx.ravel(), gy.ravel(), np.zeros(gx.size)]).astype(F)
    rng = np.random.default_rng(26)
    hs = []
    for _ in range(2):
        h = plugin.MeasurementModel(1, params=base.params)
        h.prior_map_load(prior, np.full(len(prior), 0.001, F))
        h.prior_map_window(np.array([-90.0, 0.0, 0.0]), 200.0, 20.0)
        hs.append(h)
    n_sess = 0
    for k in range(3):                                   # far outside the cube: the session grows, the window does not
        pw = np.column_stack([rng.uniform(0, 80, 60000) + 1000.0 + 100.0 * k, rng.uniform(-50, 50, 60000), rng.uniform(0.05, 0.45, 60000)])
        x = synth.make_state((1040.0 + 100.0 * k, 0.0, 1.8), (1.0, 0.0, 0.0, 0.0), [(1.0, 0.0, 0.0, 0.0)], [(0.0, 0.0, 0.0)])
        c = synth.with_scan(replace(base, x_true=x), pw, seed=k)
        hs[1].upload_scan(c.pts, c.table, c.table_off, None)
        hs[1].h_share_model(x, True)
        n_sess = hs[1].prior_map_extend(x, DS)["n_session"]
    assert n_sess > 40000
    before = [h.prior_map_info()["device_bytes"] for h in hs]
    cubes = [h.prior_map_window(np.array([-90.0, 0.0, 0.0]), 200.0, 20.0)["cube"] for h in hs]
    for rep in range(6):
        for j, h in enumerate(hs):
            c = cubes[j]
            r = h.prior_map_window(np.array([(c[0] + 15.0) if rep % 2 else (c[3] - 15.0), 0.0, 0.0]), 200.0, 20.0)
            assert r["moved"]
            cubes[j] = r["cube"]
    grow = [h.prior_map_info()["device_bytes"] - b for h, b in zip(hs, before)]
    assert grow[1] - grow[0] <= 2 * (n_sess // 1024 + 256) * 5 + 16384, (grow, n_sess)
    for h in hs:
        h.close()
