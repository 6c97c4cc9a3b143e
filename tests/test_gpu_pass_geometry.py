"""The measurement pass's reduction at every boundary of its launch geometry, entry by entry, against the exact sum.

The host picks the pass launch at run time from the point count (reduce_ref.launch_geometry): n_tiles tiles of 128
points, a co-resident wave of W = 4 * SMs blocks, per_block tiles per block, the FAST variant (rows in shared memory) up
to 2 tiles per block and the generic one (rows through global memory, reduce_block) above.  Each block re-derives its tile
range (block_tiles).  Here the launch is read back from MALIO_PASS_TRACE and must equal that formula, and at N = 0, 1,
127..129, T = W - 1, W, W + 1, N = 256 W, 256 W + 1 and T = 3 W, 3 W + 1 the reduced system must lie within
kappa * u * sum_i |t_i| of the extended-precision sum of the oracle's terms (tests/reduce_ref.py), for every entry: a
lost, doubled or misplaced row shows there whatever the summation order.  kappa is the longest dependent rounding chain
of the device's summation at that launch (reduce_ref.pass_kappa), fixed from the code, not from a measurement.

Scans are prefixes of one scan per LiDAR count, uploaded unsorted (tile t = caller points [128 t, 128 t + 128)), with the
LiDAR ids laid out point by point, in runs that change at a tile and at a block boundary, with whole blocks or a whole
LiDAR lifted 300 m off the map (no neighbour within the k-NN gate: never selected) and with a LiDAR whose only point is
the scan's last."""
import re
from dataclasses import replace

import numpy as np
import pytest

import helpers as H
import reduce_ref as rr
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu

TRACE = re.compile(r"\[malio\] pass trace: grid (\d+) fast (\d)")
FAR = np.array([0.0, 0.0, 300.0])
MAX_ROWS = 17 + 6 * capi.MAX_LIDAR     # malio_download_rows returns at most this many rows


SHAPES_N = ("T=W-1", "T=W", "T=W+1", "N=256W", "N=256W+1", "T=3W", "T=3W+1")


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def boundary_n(shape):
    """The boundary shapes for W = 4 x the SM count of this GPU (S = 132: 67,456 ... 202,880 points)."""
    W = 4 * sm_count()
    return {"T=W-1": 128 * (W - 1), "T=W": 128 * W, "T=W+1": 128 * (W + 1), "N=256W": 256 * W, "N=256W+1": 256 * W + 1,
            "T=3W": 128 * 3 * W, "T=3W+1": 128 * (3 * W + 1)}[shape]


RATIOS = []   # (shape, n_eff, grid, fast, kappa, observed max ratio, weight difference in u): printed at the end


# ------------------------------------------------------------------ one world per LiDAR count, prefixes of one scan
@pytest.fixture(scope="module")
def worlds():
    cache = {}

    def get(L):
        if L not in cache:
            base = synth.make_case(f"geo{L}", 64, 200000, L, 3, varied_map_cov=True)
            rng = np.random.default_rng(100 + L)
            half = base.meta["half"]
            pos = np.array(base.x_true.pos[:])
            pw = synth.sample_surfaces(boundary_n("T=3W+1"), pos[:2], min(100.0, half), half, rng)
            pw += rng.normal(0, 0.02, size=pw.shape)
            snap = plugin.build_static_snapshot(base.map_xyz, base.map_normal_y)
            cache[L] = (base, pw, snap)
        return cache[L]
    yield get
    if RATIOS:
        print("\nshape                                      n_eff  grid fast  kappa  max |dev-ref|/(u sum|t|)  |w_d/w_o-1|/u")
        for row in RATIOS:
            print("%-40s %7d %5d %4d %6d %8.2f %12.1f" % row)


def _scan(base, pw, lidar):
    """World points pw seen by LiDAR lidar[i] from the true state (synth._sensor_points with the ids given)."""
    s = base.x_true
    L = base.n_lidar
    extq = [np.array(s.ext[l].q[:]) for l in range(L)]
    extt = [np.array(s.ext[l].t[:]) for l in range(L)]
    pts = np.zeros(pw.shape[0], dtype=capi.SCAN_PT)
    pts["xyz"] = synth.world_to_sensor(pw, lidar, np.array(s.pos[:]), np.array(s.rot[:]), extq, extt,
                                       base.temporal_comp).astype(np.float32)
    pts["lidar"] = lidar.astype(np.uint16)
    sizes = np.diff(base.table_off.astype(np.int64))
    pts["table_idx"] = (np.arange(pw.shape[0]) * 7 % sizes[lidar]).astype(np.uint16)
    return pts


def layout(base, pw_all, N, kind, geo):
    """The case whose scan is the first N points of pw_all with LiDAR layout `kind` at launch geometry `geo`."""
    L = base.n_lidar
    pw = pw_all[:N].copy()
    idx = np.arange(N)
    lidar = idx % L
    pb, G, T = geo["per_block"], geo["grid"], geo["n_tiles"]
    if kind == "contiguous":
        # LiDAR 0 up to a tile boundary inside a block (or the first block boundary past a quarter), LiDAR 1 up to the
        # block boundary at half the grid, LiDAR 2 after it
        t_tile = pb * (G // 4) + (1 if pb > 1 else 0)
        t_block = pb * (G // 2)
        cuts = sorted({128 * t_tile, 128 * t_block})[: L - 1]
        lidar = np.searchsorted(np.asarray(cuts), idx, side="right")
        assert set(np.unique(lidar)) == set(range(L))
    elif kind == "dead_blocks":
        for b in (0, G // 2, G - 1):
            t0, t1 = b * pb, min((b + 1) * pb, T)
            pw[128 * t0: min(128 * t1, N)] += FAR
    elif kind == "last_only":
        # LiDAR L-1 has exactly one point, the last of the last tile, on the ground next to the vehicle
        lidar = idx % (L - 1)
        lidar[N - 1] = L - 1
        pos = np.array(base.x_true.pos[:])
        pw[N - 1] = (pos[0] + 4.0, pos[1] + 3.0, 0.0)
    elif kind == "lidar_dead":
        pw[lidar == L - 1] += FAR
    else:
        assert kind == "interleaved"
    return replace(base, name=f"L{L}-{kind}-{N}", pts=_scan(base, pw, lidar), meta=dict(base.meta, N=N))


# ------------------------------------------------------------------ oracle side, shared by the paths
_ORACLE = {}


def oracle_side(case, snap):
    key = case.name
    if key not in _ORACLE:
        orc = H.make_oracle(case, snap)
        ok = orc.h_share_model(case.x_prop, True, nthreads=8)
        so, ao = orc.stats(), orc.aux()
        hx, h, R = orc.dense()
        ref = rr.reduce_ref(hx, h, R) if ok else None
        orc.close()
        if hx.shape[0] > MAX_ROWS:   # the dense rows are only needed where the device's own rows can be read back
            hx = h = R = None
        _ORACLE[key] = dict(ok=ok, so=so, sel=ao["selected"].copy(), hx=hx, h=h, R=R, ref=ref)
    return _ORACLE[key]


def _trace(capfd):
    m = TRACE.findall(capfd.readouterr().err)
    assert m, "no pass trace on stderr (MALIO_PASS_TRACE)"
    return int(m[-1][0]), int(m[-1][1])


def _pair(hx, hv, hx_o, h_o):
    """For each oracle row the index of the closest device row (rows come in different orders); one to one."""
    A = np.column_stack([hx, hv]); B = np.column_stack([hx_o, h_o])
    pair = np.array([int(np.argmin(np.abs(A - b).max(axis=1))) for b in B], np.int64)
    assert len(set(pair.tolist())) == B.shape[0], "device and oracle rows do not pair up one to one"
    return pair


def run_shape(case, snap, geo, monkeypatch, capfd, *, fused=True, sort=False, label=""):
    """One pass on the device against the oracle and the extended-precision reference.  Returns the device stats."""
    L = case.n_lidar
    o = oracle_side(case, snap)
    monkeypatch.setenv("MALIO_PASS_TRACE", "1000000")
    if not fused:
        monkeypatch.setenv("MALIO_FUSED_PASS", "0")
    model = H.make_model(case, snap, sort_queries=sort)
    monkeypatch.delenv("MALIO_PASS_TRACE")
    monkeypatch.delenv("MALIO_FUSED_PASS", raising=False)
    try:
        capfd.readouterr()
        ok_g, HTH, HTh, st = model.h_share_model(case.x_prop, True)
        if fused:
            got = _trace(capfd)
            assert got == (geo["grid"], int(geo["fast"])), (
                f"launch (grid, fast) = {got}, expected {(geo['grid'], int(geo['fast']))} for N = {case.meta['N']} "
                f"with W = 4 x {sm_count()} SMs: the pass kernel does not run 4 blocks per SM")
        ag = model.aux(normal_y=False, nn_idx=False, nn_sqdist=False, world=False)
        so = o["so"]
        # the selection first: flags, count, the min / max the weights are scaled by
        assert np.array_equal(ag["selected"], o["sel"])
        assert st.n_eff == so.n_eff and ok_g == o["ok"]
        if not o["ok"]:
            assert not HTH.any() and not HTh.any()
        else:
            assert st.u_min == pytest.approx(so.u_min, rel=1e-12) and st.u_max == pytest.approx(so.u_max, rel=1e-12)
            assert st.tau_min == pytest.approx(so.tau_min, rel=1e-12) and st.tau_max == pytest.approx(so.tau_max, rel=1e-12)
            ref = o["ref"]
            kappa = rr.pass_kappa(geo, L)
            # the localization weight w scales every entry by w^2 (laserMapping.cpp:745-759).  It is a function of the 3 x 3
            # normal scatter each side sums in its own order, amplified by the singular-value ratio: the oracle's plain
            # left-to-right sum of 200k terms alone moves it by ~100 u.  It keeps its own bar; the system is compared at
            # the oracle's weight
            w_d, w_o = st.loc_weight, so.loc_weight
            assert w_d == pytest.approx(w_o, rel=1e-9)
            scale = (w_o / w_d) ** 2
            r = rr.entry_ratios(HTH * scale, HTh * scale, ref)
            # entries no selected row touches are exactly zero
            assert not HTH[ref["mHTH"] == 0].any() and not HTh[ref["mHTh"] == 0].any()
            RATIOS.append((f"{label} L={L} N={case.meta['N']}", st.n_eff, geo["grid"], int(geo["fast"]), kappa,
                           float(r.max()), abs(w_d / w_o - 1.0) / rr.U))
            worst = np.unravel_index(int(np.argmax(r)), r.shape)
            assert r.max() <= kappa, f"entry {worst} off by {r.max():.1f} u * sum|t| > kappa = {kappa}"
            if st.n_eff <= MAX_ROWS:
                # the row-level part alone: the device's own rows (with the localization weight the oracle folds into
                # its rows) summed exactly, against the oracle's rows summed exactly
                hx_d, hv_d = model.rows()
                assert hx_d.shape[0] == st.n_eff
                pair = _pair(hx_d * w_o, hv_d * w_o, o["hx"], o["h"])
                ref_d = rr.reduce_ref(hx_d[pair] * w_o, hv_d[pair] * w_o, o["R"])
                r_row = rr.entry_ratios(ref_d["HTH"], ref_d["HTh"], ref)
                r_sum = rr.entry_ratios(HTH * scale, HTh * scale, ref_d)
                assert r_row.max() <= rr.KAPPA_ROW, r_row.max()
                assert r_sum.max() <= kappa - rr.KAPPA_ROW, r_sum.max()
        # a pass re-run on the re-armed scan is bit-identical (the reduction is deterministic)
        model.rearm_scan()
        ok2, HTH2, HTh2, st2 = model.h_share_model(case.x_prop, True)
        assert ok2 == ok_g and st2.n_eff == st.n_eff
        assert np.array_equal(HTH2, HTH) and np.array_equal(HTh2, HTh)
        return st, HTH, HTh
    finally:
        model.close()


# ------------------------------------------------------------------ small scans: empty, partial first tile, n > N_eff
def _small_ns(L):
    c, n = 6 * (L + 1), 17 + 6 * L
    return sorted({0, 1, 127, 128, 129, c - 1, c + 1, n - 1, n + 1})


@pytest.mark.parametrize("L", [1, 2, 3])
def test_small_scans(worlds, L, monkeypatch, capfd):
    base, pw, snap = worlds(L)
    for N in _small_ns(L):
        geo = rr.launch_geometry(N, sm_count())
        assert geo["fast"] and geo["per_block"] == 1
        case = layout(base, pw, N, "interleaved", geo)
        run_shape(case, snap, geo, monkeypatch, capfd, label="small interleaved")


# ------------------------------------------------------------------ the boundaries of the launch geometry
def test_boundary_geometry_formula():
    """What the boundary shapes hit, by the formula the trace is held to."""
    W = 4 * sm_count()
    g = {k: rr.launch_geometry(boundary_n(k), sm_count()) for k in SHAPES_N}
    assert (g["T=W-1"]["per_block"], g["T=W"]["per_block"], g["T=W+1"]["per_block"]) == (1, 1, 2)
    assert g["T=W+1"]["grid"] == (W + 2) // 2 and g["T=W+1"]["n_tiles"] - (g["T=W+1"]["grid"] - 1) * 2 == 1
    assert g["N=256W"]["fast"] and g["N=256W"]["per_block"] == 2
    assert not g["N=256W+1"]["fast"] and g["N=256W+1"]["per_block"] == 3 and boundary_n("N=256W+1") % 128 == 1
    assert (g["T=3W"]["per_block"], g["T=3W+1"]["per_block"]) == (3, 4) and not g["T=3W+1"]["fast"]


SHAPES = [(3, k) for k in ("interleaved", "contiguous", "dead_blocks", "last_only", "lidar_dead")] + \
         [(2, "interleaved"), (2, "last_only"), (1, "interleaved")]


@pytest.mark.parametrize("L,kind", SHAPES, ids=[f"L{L}-{k}" for L, k in SHAPES])
@pytest.mark.parametrize("shape", list(SHAPES_N))
def test_boundaries(worlds, shape, L, kind, monkeypatch, capfd):
    base, pw, snap = worlds(L)
    N = boundary_n(shape)
    geo = rr.launch_geometry(N, sm_count())
    case = layout(base, pw, N, kind, geo)
    st, HTH, HTh = run_shape(case, snap, geo, monkeypatch, capfd, label=f"{shape} {kind}")
    o = oracle_side(case, snap)
    sel = o["sel"] != 0
    lid = case.pts["lidar"].astype(np.int64)
    if kind == "dead_blocks":
        pb, T = geo["per_block"], geo["n_tiles"]
        for b in (0, geo["grid"] // 2, geo["grid"] - 1):
            assert not sel[128 * b * pb: 128 * min((b + 1) * pb, T)].any()
    if kind == "last_only":
        assert sel[N - 1] and (lid[sel] == L - 1).sum() == 1
    if kind == "lidar_dead":
        assert not sel[lid == L - 1].any() and sel.any()
        e = np.r_[6 + 3 * (L - 1): 9 + 3 * (L - 1), 6 + 3 * L + 3 * (L - 1): 9 + 3 * L + 3 * (L - 1)]
        assert not HTH[e, :].any() and not HTH[:, e].any() and not HTh[e].any()
    for l in range(L):
        assert (lid[sel] == l).any() or kind == "lidar_dead"


@pytest.mark.parametrize("shape", list(SHAPES_N))
def test_boundaries_sorted(worlds, shape, monkeypatch, capfd):
    """The default internal order (sort_queries: k-NN cell order, LiDAR-major above 2 * 128 * W points) as bench.py runs."""
    base, pw, snap = worlds(3)
    N = boundary_n(shape)
    geo = rr.launch_geometry(N, sm_count())
    run_shape(layout(base, pw, N, "interleaved", geo), snap, geo, monkeypatch, capfd, sort=True, label=f"{shape} sorted")


@pytest.mark.parametrize("shape", list(SHAPES_N))
def test_boundaries_unfused(worlds, shape, monkeypatch, capfd):
    """The separate gate / reduce / fold kernels (the NCCL path): reduce_kernel over a wave of red_grid blocks."""
    base, pw, snap = worlds(3)
    N = boundary_n(shape)
    geo = rr.launch_geometry(N, sm_count(), fused=False)
    run_shape(layout(base, pw, N, "interleaved", geo), snap, geo, monkeypatch, capfd, fused=False, label=f"{shape} unfused")


@pytest.mark.parametrize("shape", ["N=256W", "N=256W+1"])
def test_device_solve_at_the_fast_generic_switch(worlds, shape, monkeypatch):
    """update_on_device derives the launch on its own: the last FAST and the first generic launch give the host loop's
    passes, searches and state."""
    base, pw, snap = worlds(3)
    N = boundary_n(shape)
    case = layout(base, pw, N, "interleaved", rr.launch_geometry(N, sm_count()))
    monkeypatch.setenv("MALIO_DEVICE_SOLVE", "1")
    dev = H.make_model(case, snap)
    monkeypatch.setenv("MALIO_DEVICE_SOLVE", "0")
    host = H.make_model(case, snap)
    monkeypatch.delenv("MALIO_DEVICE_SOLVE")
    try:
        xd, Pd = case.x_prop.copy(), case.P_prop.copy()
        xh, Ph = case.x_prop.copy(), case.P_prop.copy()
        rd = dev.update_iterated_dyn_share_modified(xd, Pd, case.max_iter)
        rh = host.update_iterated_dyn_share_modified(xh, Ph, case.max_iter)
        assert rd.last_status == 0 and rh.last_status == 0
        assert rd.ms_host_solve == 0.0
        assert rd.passes == rh.passes and rd.searches == rh.searches and rd.n_eff_last == rh.n_eff_last
        assert np.abs(synth.state_to_vec(xd, 3) - synth.state_to_vec(xh, 3)).max() < 1e-9
        assert H.rel_err(Pd, Ph) < 1e-8
    finally:
        dev.close(); host.close()
