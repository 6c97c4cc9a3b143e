"""Both relocalization searches at the argument shapes and scan contents the exactness tests of test_gpu_relocalize.py and
test_gpu_place.py never reach, against the numpy restatements (tests/reloc_ref.py, tests/place_ref.py):
  - malio_relocalize: pyramids where z still splits after x and y stopped (dz > dxy), half_xy = 0 and half_xy = half_z = 0 (the
    top level is the leaf level), 2049 / 4100 / 65 537 yaws (top-level chunks and the register kernel's grid-y loop), NaN, inf
    and overflowing scan points, a scan with no finite point, scans of 1 / 31 / 33 / 257 points, points on voxel faces at an
    inexact res, and a ground-only prior whose 13 122 candidates all tie;
  - the place database bit-identical at the defaults, 4 / 8 / 16 sectors (the 45-degree boundary), lattices of step 2 and 3
    cells starting at a negative column that is not a multiple of the step, 32 x 128 = MALIO_PLACE_MAX_BINS bins, a stencil of
    MALIO_PLACE_MAX_RADIUS_CELLS, block levels 1 and 15, and ring caps down to level 1;
  - the query and stages 1-2: scan points on column half-boundaries, non-finite points and points beyond the stencil,
    k1 = MALIO_PLACE_MAX_K1 with more and fewer positions, k2 = MALIO_PLACE_MAX_K2, and a prior symmetric under quarter turns
    whose stage-2 shifts tie.
The instance builders are shared with test_reloc_edges_cpu.py, which shows that each of them tells a planted mistake apart."""
import math

import numpy as np
import pytest

import place_ref as PR
import reloc_ref as RR
import world_ref
from malio_b200 import capi, plugin, synth
from test_gpu_place import _check_db
from test_gpu_relocalize import _instance as _reloc_instance
from test_gpu_relocalize import make_scene, q_yaw, sample_scene, scan_of

pytestmark = pytest.mark.gpu
F = np.float32
ID_Q = np.array([1.0, 0.0, 0.0, 0.0])
CHUNK = 2048                                       # top-level yaws per chunk in malio_reloc.cu


# ================================================================== malio_relocalize instances
def _truncate(case, n):
    case = dict(case)
    case["pts"] = case["pts"][:n].copy()
    return case


def z_deeper(hxy, hz):
    """The building scene with a lattice deeper in z than in x / y."""
    return _reloc_instance(900 + 10 * hxy + hz, hxy=hxy, hz=hz, n_yaw=6, res=1.0)


def zero_lattice(n_yaw):
    return _reloc_instance(920 + n_yaw, hxy=0, hz=0, n_yaw=n_yaw, res=1.0)


def many_yaws(n_yaw):
    """n_yaw yaws over a small lattice (or a single offset for the largest count) on a short scan."""
    if n_yaw > 1 << 16:
        return _truncate(_reloc_instance(930, hxy=0, hz=0, n_yaw=n_yaw, res=1.0), 60)
    return _truncate(_reloc_instance(931 + n_yaw % 7, hxy=1, hz=1, n_yaw=n_yaw, res=1.0), 100)


# yaws in [0.3, 0.8] rad after an untilted guess with unrotated extrinsics: a point at (+-3e38, +-3e38, z) leaves float range
# under every candidate (one coordinate grows by cos + sin >= 1.25)
OVERFLOW = np.array([[3e38, 3e38, 1.0], [-3e38, 3e38, 2.0], [3e38, -3e38, 0.0], [-3e38, -3e38, -1.0], [3.3e38, 3.2e38, 5.0]])
NONFINITE = np.array([[np.nan, 1.0, 2.0], [1.0, np.inf, 0.0], [0.0, 1.0, -np.inf], [np.inf, -np.inf, np.nan], [-np.inf, 2.0, 3.0]])


def nonfinite(seed, kind="mixed"):
    """kind 'mixed': a scan of the building scene with NaN / inf points and finite points that overflow in body_to_world;
    'none': the same scan holding only such points; 'clean': only its finite points."""
    rng = np.random.default_rng(940 + seed)
    scene = make_scene(rng, 30.0, 6)
    prior = sample_scene(scene, rng, 2.0)
    truth = np.array([rng.uniform(-5, 5), rng.uniform(-5, 5), 1.8])
    extq, extt = [ID_Q], [rng.normal(0, 0.3, 3)]
    pw = sample_scene(scene, rng, 1.0, truth[:2], 25.0)
    pw = pw[rng.permutation(len(pw))[:300]]
    pts, table, table_off = scan_of(pw, rng, truth, q_yaw(rng.uniform(0.3, 0.8)), extq, extt, None)
    bad = np.concatenate([NONFINITE, OVERFLOW, NONFINITE[::-1], OVERFLOW[::-1]])
    if kind == "mixed":
        at = np.sort(rng.choice(len(pts), len(bad), replace=False))
        pts["xyz"][at] = bad.astype(F)
    elif kind == "none":
        pts = pts[:len(bad)].copy()
        pts["xyz"] = bad.astype(F)
    guess = synth.make_state(truth + rng.uniform(-2, 2, 3) * np.array([1, 1, 0.5]), ID_Q, extq, extt)
    return dict(prior=prior.astype(F), pts=pts, table=table, table_off=table_off, tc=None, guess=guess, L=1,
                args=dict(res=1.0, half_xy=3, half_z=1, n_yaw=6, yaw_lo=0.3, yaw_step=0.1))


def face_coords(res, lo=-1500, hi=1500):
    """The float multiples float32(k * res) (as float64) and those among them where floor(w / res) and floor(w * (1 / res))
    differ.  At res 0.1 and 0.3 no float32 multiple splits the two (1 / 0.1 is exactly 10, and for 0.3 both round the same way);
    at 0.7 some do (10.5 = 15 * 0.7: the quotient rounds to 15, the product with 1 / 0.7 to just below)."""
    w = (np.arange(lo, hi + 1) * res).astype(F).astype(np.float64)
    differ = np.floor(w / res) != np.floor(w * (1.0 / res))
    return w, w[differ]


def faces(res, seed=0):
    """Scan points at float multiples of res (identity rotation, extrinsics and position, one yaw at 0: w is the point), on the
    multiples where dividing by res and multiplying by its reciprocal disagree when there are any; the prior holds the centres
    of their voxels (by division) and some clutter."""
    rng = np.random.default_rng(960 + seed)
    allw, d = face_coords(res)
    d = d if len(d) else allw
    n = 240
    xyz = np.column_stack([rng.choice(d, n), rng.choice(d, n), rng.choice(allw[len(allw) // 2 - 20:len(allw) // 2 + 40], n)])
    pts = np.zeros(n, capi.SCAN_PT)
    pts["xyz"] = xyz.astype(F)
    table, table_off = synth.make_tables(1, 2, rng)
    pts["table_idx"] = rng.integers(0, 2, n)
    vox = np.floor(xyz / res)
    keep = rng.random(n) < 0.8
    span = np.abs(xyz).max()
    prior = np.concatenate([(vox[keep] + 0.5) * res, rng.uniform(-span, span, (100, 3))])
    guess = synth.make_state(np.zeros(3), ID_Q, [ID_Q], [np.zeros(3)])
    return dict(prior=prior.astype(F), pts=pts, table=table, table_off=table_off, tc=None, guess=guess, L=1,
                args=dict(res=res, half_xy=2, half_z=1, n_yaw=1, yaw_lo=0.0, yaw_step=1.0))


def ground_tie(seed=0):
    """A ground-only prior (one point in every voxel of z = 0) and a ground scan: every one of the 2 x 81 x 81 candidates scores
    every point."""
    rng = np.random.default_rng(980 + seed)
    g = np.arange(-110.0, 110.0) + 0.5
    gx, gy = np.meshgrid(g, g, indexing="ij")
    prior = np.column_stack([gx.ravel(), gy.ravel(), np.full(gx.size, 0.3)])
    extq, extt = [synth.q_exp(synth.rand_unit(rng) * 0.2)], [rng.normal(0, 0.3, 3)]
    tilt = synth.q_exp(np.array([rng.normal(0, 0.05), rng.normal(0, 0.05), 0.0]))
    truth = np.array([rng.uniform(-5, 5), rng.uniform(-5, 5), 1.8])
    pw = np.column_stack([rng.uniform(-20, 20, 300) + truth[0], rng.uniform(-20, 20, 300) + truth[1], np.full(300, 0.3)])
    pts, table, table_off = scan_of(pw, rng, truth, synth.q_mul(q_yaw(rng.uniform(0, 2 * np.pi)), tilt), extq, extt, None)
    guess = synth.make_state(truth + np.array([rng.uniform(-30, 30), rng.uniform(-30, 30), 0.0]), tilt, extq, extt)
    return dict(prior=prior.astype(F), pts=pts, table=table, table_off=table_off, tc=None, guess=guess, L=1,
                args=dict(res=1.0, half_xy=40, half_z=0, n_yaw=2, yaw_lo=float(rng.uniform(-np.pi, np.pi)), yaw_step=np.pi))


Z_DEEPER = [(1, 3), (2, 6), (1, 7), (0, 2)]


def reloc_cases():
    """(name, builder, argument) of every malio_relocalize instance; the builders run lazily (some restatements take seconds)."""
    out = [(f"zdeep-{hxy}-{hz}", z_deeper, (hxy, hz)) for hxy, hz in Z_DEEPER]
    out += [(f"zero-{k}", zero_lattice, (k,)) for k in (1, 12)]
    out += [(f"yaws-{k}", many_yaws, (k,)) for k in (2049, 4100, 65537)]
    out += [("nonfinite", nonfinite, (0, "mixed")), ("no-finite", nonfinite, (1, "none"))]
    out += [(f"n{n}", lambda n: _truncate(nonfinite(2, "clean"), n), (n,)) for n in (1, 31, 33, 257)]
    out += [(f"faces-{res}", faces, (res,)) for res in (0.1, 0.3, 0.7)]
    out += [("ground", ground_tie, ())]
    return out


def single_offset_scores(case):
    """RR.scores for half_xy = half_z = 0 and one LiDAR without temporal compensation, all yaws at once: world_ref.register_world's
    operations in its order, broadcast over the candidate rotations (int64[n_yaw] scores, finite points per yaw)."""
    a, ps = case["args"], case["guess"].pass_state()
    assert a["half_xy"] == a["half_z"] == 0 and case["L"] == 1 and case["tc"] is None
    body = world_ref._qrot(np.array(ps.ext[0].q[:]), case["pts"]["xyz"].astype(np.float64)) + np.array(ps.ext[0].t[:])
    qs = np.array(RR.candidate_rotations(ps.rot[:], a["yaw_lo"], a["yaw_step"], a["n_yaw"]))
    pos = np.array(ps.pos[:])
    occ = np.unique(RR.prior_voxels(case["prior"], a["res"]), axis=0)
    key = lambda v: (v[..., 0] * (1 << 21) + v[..., 1]) * (1 << 21) + v[..., 2]
    occ_keys = key(occ)
    v0, v1, v2 = body[None, :, 0], body[None, :, 1], body[None, :, 2]
    scores, n_fin = [], []
    for k0 in range(0, len(qs), 4096):
        w, x, y, z = (qs[k0:k0 + 4096, i:i + 1] for i in range(4))
        a0, a1, a2 = y * v2 - z * v1, z * v0 - x * v2, x * v1 - y * v0
        u0, u1, u2 = a0 + a0, a1 + a1, a2 + a2
        c0, c1, c2 = y * u2 - z * u1, z * u0 - x * u2, x * u1 - y * u0
        with np.errstate(invalid="ignore", over="ignore"):
            W = np.stack([(v0 + w * u0) + c0 + pos[0], (v1 + w * u1) + c1 + pos[1], (v2 + w * u2) + c2 + pos[2]], axis=-1)
            W = W.astype(F).astype(np.float64)
        fin = np.all(np.isfinite(W), axis=-1)
        vox = np.floor(np.where(fin[..., None], W, 0.0) / a["res"]).astype(np.int64)
        scores.append((np.isin(key(vox), occ_keys) & fin).sum(axis=1))
        n_fin.append(fin.sum(axis=1))
    return np.concatenate(scores), np.concatenate(n_fin), qs


def single_offset_want(case):
    sc, n_fin, qs = single_offset_scores(case)
    k = int(np.argmax(sc))
    ps = case["guess"].pass_state()
    return dict(yaw_index=k, offset=(0, 0, 0), score=int(sc[k]), n_points=int(n_fin[k]), rot=qs[k],
                pos=np.array([float(ps.pos[j]) + 0.0 * case["args"]["res"] for j in range(3)]), n_candidates=len(sc), scores=sc)


def reloc_want(case):
    a = case["args"]
    if a["n_yaw"] > 1 << 16:                       # the exhaustive restatement takes minutes here: the same arithmetic, batched
        return single_offset_want(case)
    return RR.relocalize(case["guess"], case["tc"], case["pts"], case["prior"], a["res"], a["half_xy"], a["half_z"], a["n_yaw"],
                         a["yaw_lo"], a["yaw_step"])


def _reloc_model(case):
    m = plugin.MeasurementModel(case["L"])
    m.prior_map_load(case["prior"])
    m.upload_scan(case["pts"], case["table"], case["table_off"], case["tc"])
    return m


def _registered(case, k=0):
    """World points of the scan under candidate rotation k (world_ref.register_world, the bits malio_world_register gives)."""
    a = case["args"]
    q = RR.candidate_rotations(case["guess"].rot[:], a["yaw_lo"], a["yaw_step"], k + 1)[k]
    return world_ref.register_world(RR._with_rot(case["guess"], q), case["tc"], case["pts"]["xyz"],
                                    case["pts"]["lidar"].astype(np.int64), 0.0)[:, :3]


@pytest.mark.parametrize("name,build,arg", reloc_cases(), ids=[c[0] for c in reloc_cases()])
def test_relocalize_equals_the_exhaustive_search(name, build, arg):
    case = build(*arg)
    a = case["args"]
    want = reloc_want(case)
    if name.startswith("zdeep"):
        dxy, dz = RR.ceil_log2(2 * a["half_xy"] + 1), RR.ceil_log2(2 * a["half_z"] + 1)
        assert dz > dxy, (dxy, dz)
    if name.startswith("yaws"):
        assert a["n_yaw"] > CHUNK and a["n_yaw"] % CHUNK
    if name == "yaws-65537":                       # the batched restatement is RR.scores on the first yaws
        assert a["n_yaw"] > 65535 and a["half_xy"] == a["half_z"] == 0
        head = dict(case, args=dict(a, n_yaw=300))
        assert np.array_equal(RR.scores(head["guess"], None, case["pts"], case["prior"], a["res"], 0, 0, 300, a["yaw_lo"],
                                        a["yaw_step"])[0].ravel(), want["scores"][:300])
    if name == "nonfinite":                        # the planted points: non-finite under every candidate, the rest finite
        bad = ~np.all(np.isfinite(case["pts"]["xyz"]), axis=1)
        over = np.all(np.isfinite(case["pts"]["xyz"]), axis=1) & (np.abs(case["pts"]["xyz"]).max(axis=1) > 1e38)
        assert bad.sum() == 10 and over.sum() == 10
        for k in range(a["n_yaw"]):
            fin = np.all(np.isfinite(_registered(case, k)), axis=1)
            assert not fin[bad | over].any() and fin[~(bad | over)].all()
        assert want["n_points"] == len(case["pts"]) - 20
    if name == "no-finite":
        assert want["score"] == 0 and want["n_points"] == 0 and want["yaw_index"] == 0
        assert want["offset"] == (-a["half_xy"], -a["half_xy"], -a["half_z"])
    if name.startswith("faces"):                   # w is the point itself; at 0.7 the x and y of every point split / and * (1 / res)
        w = _registered(case)
        assert w.tobytes() == case["pts"]["xyz"].tobytes()
        w = w.astype(np.float64)
        split = (np.floor(w / a["res"]) != np.floor(w * (1.0 / a["res"]))).sum()
        assert split >= 2 * len(w) if a["res"] == 0.7 else split == 0
        t = w[:, :2] / a["res"]
        assert (np.abs(t - np.round(t)) <= 1e-6 * np.maximum(1.0, np.abs(t))).all()      # within a float ulp of a face
    if name == "ground":                           # 13 122 candidates tie: the first one
        assert want["n_candidates"] == 13122 and (want["scores"] == len(case["pts"])).all()
        assert want["yaw_index"] == 0 and want["offset"] == (-40, -40, 0)
    m = _reloc_model(case)
    r = m.relocalize(case["guess"], **a)
    got = (r["yaw_index"], r["offset"], r["score"], r["n_points"], r["n_candidates"])
    assert got == (want["yaw_index"], want["offset"], want["score"], want["n_points"], want["n_candidates"]), (name, got)
    assert r["rot"].tobytes() == want["rot"].tobytes() and r["pos"].tobytes() == want["pos"].tobytes()
    assert r["nodes_bounded"] >= r["leaves_scored"]
    again = m.relocalize(case["guess"], **a)
    assert {k: (v.tobytes() if isinstance(v, np.ndarray) else v) for k, v in again.items() if k != "state"} == \
           {k: (v.tobytes() if isinstance(v, np.ndarray) else v) for k, v in r.items() if k != "state"}
    print(name, {k: r[k] for k in ("score", "n_points", "n_candidates", "nodes_bounded", "leaves_scored", "device_bytes")})
    m.close()


# ================================================================== place database instances
SMALL = dict(r_max=20.0, n_ring=5, n_sector=12)


def _pargs(**kw):
    if "fov_up_deg" in kw:
        kw["fov_up"] = math.radians(kw.pop("fov_up_deg"))
    return plugin.MeasurementModel.place_args(1.8, **kw)


def scene_prior(seed, half=15.0, n_build=3, density=0.5):
    rng = np.random.default_rng(1100 + seed)
    return sample_scene(make_scene(rng, half, n_build), rng, density).astype(F)


def lattice_x0(cell, m):
    """A box start x0 < 0 whose column floor(x0 / cell) is not a multiple of m (and, for m = 3, is 2 mod 3: there the usual
    positive-only ceiling (i + m - 1) / m under truncating division misses the first lattice column)."""
    for x0 in (-37.3, -37.6, -37.45, -37.8, -38.1):
        i = math.floor(x0 / cell)
        if i % m and (m != 3 or i % 3 == 2):
            return x0
    raise AssertionError((cell, m))


def lattice_prior(cell, m, seed=0):
    """Points in [x0, x0 + 20]^2 (x0 from lattice_x0), heights 0-12 m, the box's corner and the first lattice row and column
    occupied."""
    rng = np.random.default_rng(1200 + seed)
    x0 = lattice_x0(cell, m)
    p = np.column_stack([rng.uniform(x0, x0 + 20, 1500), rng.uniform(x0, x0 + 20, 1500), rng.uniform(0, 12, 1500)])
    first = (-(-math.floor(x0 / cell) // m) * m + 0.5) * cell     # the centre of the first lattice column
    t = np.linspace(x0 + 0.01, x0 + 19.9, 40)
    rows = np.concatenate([np.column_stack([np.full(40, first), t, rng.uniform(0, 3, 40)]),
                           np.column_stack([t, np.full(40, first), rng.uniform(0, 3, 40)])])
    return np.concatenate([[[x0, x0, 1.0]], p, rows]).astype(F)


def radius_prior(seed=0):
    """Two lattice columns (step 64 m at cell 0.25: m = 256) with points all around them within the 64 m stencil."""
    rng = np.random.default_rng(1300 + seed)
    p = np.column_stack([rng.uniform(-60, 124, 4000), rng.uniform(-60, 60, 4000), rng.uniform(-1, 15, 4000)])
    return np.concatenate([[[0.1, 0.1, 0.0], [64.1, 0.1, 0.0]], p]).astype(F)


def db_cases():
    """(name, prior builder, args)."""
    out = [("defaults", lambda: scene_prior(0, 25.0, 4, 0.05), _pargs())]
    out += [(f"sectors-{s}", lambda: scene_prior(1), _pargs(**dict(SMALL, n_sector=s))) for s in (4, 8, 16)]
    out += [(f"lattice-{c}-{m}", (lambda c=c, m=m: lattice_prior(c, m)),
             _pargs(cell=c, step=m * c, r_max=10.0, n_ring=4, n_sector=12)) for c in (0.5, 0.25) for m in (2, 3)]
    out += [("bins-4096", lambda: scene_prior(2), _pargs(r_max=20.0, n_ring=32, n_sector=128))]
    out += [("radius-256", radius_prior, _pargs(cell=0.25, step=64.0, r_max=64.0))]
    out += [(f"block-{b}", lambda: scene_prior(3), _pargs(**dict(SMALL, block_level=b))) for b in (1, 15)]
    out += [("cap-1", lambda: scene_prior(4, 20.0, 4), _pargs(r_max=40.0, n_ring=8, n_sector=12, z_lo=0.0, fov_up_deg=2.0))]
    return out


@pytest.mark.parametrize("name,prior,args", db_cases(), ids=[c[0] for c in db_cases()])
def test_database_is_bit_identical_to_the_restatement(name, prior, args):
    prior = prior()
    m = plugin.MeasurementModel(1)
    m.prior_map_load(prior)
    rep, want = _check_db(m, prior, args)
    nb = args.n_ring * args.n_sector
    assert rep["n_positions"] >= 2 and want["levels"].max() >= 1, name
    if name == "bins-4096":
        assert nb == capi_max_bins() and want["levels"][:, nb - args.n_sector:].any()
    if name == "radius-256":
        assert args.r_max / args.cell == 256 and rep["n_positions"] == 2 and rep["n_stencil"] > 200000
    if name.startswith("lattice"):
        mm = int(round(args.step / args.cell))
        ilo = int(np.floor(prior[:, 0].astype(np.float64) / args.cell).min())
        assert ilo < 0 and ilo % mm and (want["cols"] % mm == 0).all() and (want["cols"] < 0).all()
    if name == "cap-1":
        assert PR.caps(args).min() == 1 and (want["levels"] == 1).any()
    print(name, rep)
    m.close()


def capi_max_bins():
    return 4096                                    # MALIO_PLACE_MAX_BINS


# ================================================================== query and ranking instances
def query_scan(seed, prior_pts, center, radius=45.0, n=1500, snap=None, junk=True):
    """Scan records of the prior's points around `center` seen from there (identity rotation and extrinsics, so that a point's
    registered rel is its own coordinates): with `snap` (a cell) every other point moved onto a column half-boundary, with
    `junk` NaN / inf points and points beyond the 60 m stencil (near enough that stage 3's pyramid box stays within its limit)."""
    rng = np.random.default_rng(1400 + seed)
    p = prior_pts.astype(np.float64)
    p = p[np.hypot(p[:, 0] - center[0], p[:, 1] - center[1]) <= radius] - np.asarray(center)
    p = p[rng.permutation(len(p))[:n]]
    if snap is not None:
        p[::2, 0] = (np.floor(p[::2, 0] / snap) + 0.5) * snap
        p[1::2, 1] = (np.floor(p[1::2, 1] / snap) + 0.5) * snap
    if junk:
        p = np.concatenate([p, NONFINITE, [[75.0, 3.0, 2.0], [-200.0, 0.0, 9.0], [0.0, 64.0, 5.0], [0.0, -90.0, 1.0]]])
    pts = np.zeros(len(p), capi.SCAN_PT)
    pts["xyz"] = p.astype(F)
    table, table_off = synth.make_tables(1, 2, rng)
    pts["table_idx"] = rng.integers(0, 2, len(p))
    return pts, table, table_off


def quarter_prior(seed=0, n=300, half=30):
    """Points at quarter-metre offsets and their quarter turns about the centre (0.5, 0.5) of column (0, 0): (x, y) ->
    (1 - y, x) is exact in float and maps column (i, j) to (-j, i)."""
    rng = np.random.default_rng(1500 + seed)
    p = np.column_stack([rng.integers(-half, half, (n, 2)) + rng.choice([0.25, 0.75], (n, 2)), rng.uniform(-1, 14, n)])
    p = np.concatenate([[[0.25, 0.25, 0.0]], p])
    out = [p]
    for _ in range(3):
        p = np.column_stack([1.0 - p[:, 1], p[:, 0], p[:, 2]])
        out.append(p)
    return np.concatenate(out).astype(F)


def query_case(kind, n_sector=72):
    """(prior, args, scan, guess, k1, k2)."""
    guess = synth.make_state(np.array([3.0, -7.0, 1.0]), ID_Q, [ID_Q], [np.zeros(3)])
    if kind == "half":                             # cell 0.5: half-boundary columns
        prior = scene_prior(10, 25.0, 4, 0.12)
        args = _pargs(cell=0.5, n_sector=n_sector)
        center = np.array([0.3, -1.2, 1.8])
        k1, k2 = 64, 8
        pts = query_scan(10, prior, center, snap=0.5)
    elif kind in ("many", "few"):                  # k1 = 1024 over more / fewer positions, k2 = 32
        prior = scene_prior(11, 20.0, 4, 0.9) if kind == "many" else scene_prior(12, 25.0, 4, 0.1)
        args = _pargs(n_sector=n_sector)
        center = np.array([1.0, 2.0, 1.8])
        k1, k2 = 1024, 32
        pts = query_scan(11, prior, center)
    elif kind == "quarter":                        # the scan seen from column (0, 0) of a quarter-turn symmetric prior
        prior = quarter_prior()
        args = _pargs(n_sector=n_sector)
        zs = float(prior[(np.floor(prior[:, 0]) == 0) & (np.floor(prior[:, 1]) == 0), 2].min()) + 1.8
        center = np.array([0.5, 0.5, zs])
        k1, k2 = 1024, 32
        pts = query_scan(12, prior, center, junk=False)
    else:
        raise ValueError(kind)
    return dict(prior=prior, args=args, pts=pts, guess=guess, k1=k1, k2=k2)


QUERY = [(k, s) for k in ("half", "many", "few", "quarter") for s in (72, 8)]


def query_want(case):
    args = case["args"]
    pts = case["pts"][0]
    q, qk = PR.query(case["guess"], None, pts, args)
    db = PR.database(case["prior"], args)
    surv, d1 = PR.stage1(qk, db["ring_keys"], case["k1"])
    p2, d2, sh = PR.stage2(q, db["levels"], surv, args, case["k2"])
    return dict(q=q, qk=qk, db=db, surv=surv, d1=d1, p2=p2, d2=d2, sh=sh)


def quarter_position(db):
    return int(np.flatnonzero((db["cols"][:, 0] == 0) & (db["cols"][:, 1] == 0))[0])


@pytest.mark.parametrize("kind,n_sector", QUERY, ids=[f"{k}-{s}" for k, s in QUERY])
def test_query_and_ranking_equal_the_restatement(kind, n_sector):
    case = query_case(kind, n_sector)
    args, (pts, table, table_off) = case["args"], case["pts"]
    want = query_want(case)
    db = want["db"]
    n_pos = len(db["cols"])
    if kind == "half":                             # the half-boundary points: rel / cell + 0.5 an integer
        w = pts["xyz"].astype(np.float64)
        fin = np.all(np.isfinite(w), axis=1)
        assert (np.floor(w[fin, 0] / args.cell + 0.5) == w[fin, 0] / args.cell + 0.5).sum() >= (fin.sum() - 4) // 2
    if kind == "many":
        assert n_pos > case["k1"]
    if kind == "few":
        assert n_pos < case["k1"]
    m = plugin.MeasurementModel(1)
    m.prior_map_load(case["prior"])
    _check_db(m, case["prior"], args)
    m.upload_scan(pts, table, table_off, None)
    r = m.relocalize_global(case["guess"], k1=case["k1"], k2=case["k2"], res=1.0, half_xy=2, half_z=1)
    nb = args.n_ring * args.n_sector
    assert np.array_equal(r["query"][:nb].astype(np.int64), want["q"]) and not r["query"][nb:].any()
    assert r["n_stage1"] == min(case["k1"], n_pos) and r["n_candidates"] == min(case["k2"], r["n_stage1"])
    assert np.array_equal(r["stage1"], want["surv"]) and np.array_equal(r["stage1_d1"], want["d1"])
    got = [(c["position"], c["d2"], c["shift"]) for c in r["cand"]]
    assert got == list(zip(want["p2"].tolist(), want["d2"].tolist(), want["sh"].tolist()))
    if kind == "quarter":                          # the centre's descriptor repeats every Q sectors: the smallest shift wins
        Q = args.n_sector // 4
        p0 = quarter_position(db)
        ds = PR.shift_distances(want["q"], db["levels"][p0], args.n_ring, args.n_sector)
        assert all(np.array_equal(ds, np.roll(ds, Q * t)) for t in range(4))
        c0 = [c for c in r["cand"] if c["position"] == p0]
        assert len(c0) == 1 and c0[0]["shift"] < Q and c0[0]["d2"] == ds.min() == 0
    if kind == "few" and n_sector == 72:           # stage 3 by hand: malio_relocalize from every candidate's guess
        n_yaw, yaw_lo = PR.verify_args(args.n_sector, math.radians(1.0))
        best = None
        for k, c in enumerate(r["cand"]):
            g = PR.verification_guess(case["guess"], db["cols"][c["position"]], db["z_s"][c["position"]], c["shift"], args)
            assert np.array(g.rot[:]).tobytes() == c["guess_rot"].tobytes() and np.array(g.pos[:]).tobytes() == c["guess_pos"].tobytes()
            h = m.relocalize(g, 1.0, 2, 1, n_yaw=n_yaw, yaw_lo=yaw_lo, yaw_step=math.radians(1.0))
            assert (h["score"], h["n_points"]) == (c["score"], c["n_points"])
            assert h["rot"].tobytes() == c["rot"].tobytes() and h["pos"].tobytes() == c["pos"].tobytes()
            if best is None or h["score"] > best[1]["score"]:
                best = (k, h)
        assert r["best_rank"] == best[0] and r["score"] == best[1]["score"]
        assert r["pos"].tobytes() == best[1]["pos"].tobytes() and r["rot"].tobytes() == best[1]["rot"].tobytes()
    print(kind, n_sector, "positions", n_pos, "best", r["best_rank"], r["score"], r["n_points"])
    m.close()
