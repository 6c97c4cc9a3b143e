"""The extended-precision reference of the reduced system (tests/reduce_ref.py) on the CPU: it is the exact sum of
orc_reduce's terms (both summation methods agree to the last bit but one, and catch cancellations a float64 sum cannot),
orc_reduce lies within its own summation bound of it, and the entry-wise bar the GPU geometry tests use notices one
lost or doubled row at the row counts those tests reach."""
import time

import numpy as np
import pytest

import helpers as H
import reduce_ref as rr
from malio_b200 import plugin, synth

# the largest pass the GPU geometry tests run: 3 * W + 1 tiles for W = 4 * 132 (an H100 SXM); 200k-odd selected rows
GPU_MAX_POINTS = 128 * (3 * 528 + 1)


def test_method_is_declared():
    assert rr.METHOD == ("longdouble" if np.finfo(np.longdouble).nmant >= 63 else "fsum")
    assert rr.reduce_ref(np.ones((2, 3)), np.ones(2), np.ones(2))["method"] == rr.METHOD


def test_exact_where_float64_cancels():
    """Terms 2^60, 1, -2^60 in every order: a float64 sum from the left loses the 1, the reference keeps it."""
    big = 2.0 ** 30
    hx = np.array([[big], [1.0], [-big]])
    h = np.array([big, 1.0, big])
    R = np.ones(3)
    methods = ["fsum"] + (["longdouble"] if rr.LONGDOUBLE_OK else [])
    for perm in ([0, 1, 2], [1, 0, 2], [2, 0, 1], [0, 2, 1]):
        for m in methods:
            ref = rr.reduce_ref(hx[perm], h[perm], R[perm], method=m)
            assert ref["HTh"][0] == 1.0, (perm, m)
            assert ref["mHTh"][0] == 2.0 ** 61
    assert (2.0 ** 60 + 1.0) - 2.0 ** 60 == 0.0    # what a float64 sum in caller order gives
    # R below 1e-4 is clamped to 1e-3 (esekfom.hpp:624-626), R at 1e-4 is not
    ref = rr.reduce_ref(np.array([[1.0], [1.0]]), np.zeros(2), np.array([5e-5, 1e-4]), method="fsum")
    assert ref["HTH"][0, 0] == 1.0 / 1e-3 + 1.0 / 1e-4


@pytest.fixture(scope="module", params=[1, 2, 3], ids=lambda L: f"L{L}")
def dense(request):
    L = request.param
    case = synth.make_case(f"ref{L}", 6000, 60000, L, 3, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    orc = H.make_oracle(case, snap)
    assert orc.h_share_model(case.x_prop, True, 4)
    hx, h, R = orc.dense()
    HTH, HTh = orc.reduce()
    orc.close()
    assert hx.shape[0] > 3000 and hx.shape[1] == 6 * (L + 1)
    return L, hx, h, R, HTH, HTh


def test_reference_reproduces_orc_reduce(dense):
    """orc_reduce sums its n_eff terms left to right: within gamma_{n-1} * sum|t| (+ the reference's own rounding)."""
    L, hx, h, R, HTH, HTh = dense
    ref = rr.reduce_ref(hx, h, R)
    n = hx.shape[0]
    r = rr.entry_ratios(HTH, HTh, ref)
    assert r.max() <= n + 1, r.max()
    assert np.isfinite(r).all()
    # the bar is tight enough to mean something: orc_reduce's observed error is far below its worst case
    assert r.max() < n / 10, r.max()
    print(f"L={L} n_eff={n}: orc_reduce vs reference max ratio {r.max():.1f} (bound {n + 1})")


def test_summation_methods_agree(dense):
    """The two extended summations are both the exact sum rounded once: they differ by at most one float64 rounding
    each, i.e. by u * |S| (plus 2^-60 * sum|t| for the longdouble one's own rounding)."""
    if not rr.LONGDOUBLE_OK:
        pytest.skip("np.longdouble has no 64-bit significand here: only the fsum method exists")
    L, hx, h, R, _, _ = dense
    a = rr.reduce_ref(hx, h, R, method="longdouble")
    b = rr.reduce_ref(hx, h, R, method="fsum")
    for k in ("HTH", "HTh"):
        tol = rr.U * np.abs(b[k]) + 2.0 ** -60 * b["m" + k]
        assert (np.abs(a[k] - b[k]) <= tol).all()
        np.testing.assert_allclose(a["m" + k], b["m" + k], rtol=1e-13)


def test_reference_runtime_at_gpu_scale():
    """A few seconds for ~200k rows and c = 24."""
    rng = np.random.default_rng(1)
    n, c = 200_000, 24
    hx = rng.normal(size=(n, c)); h = rng.normal(size=n); R = rng.uniform(5e-5, 1e-2, n)
    t0 = time.perf_counter()
    rr.reduce_ref(hx, h, R)
    dt = time.perf_counter() - t0
    print(f"{rr.METHOD}: {dt:.2f} s for {n} x {c}")
    assert dt < 30.0


def _kappa_max(L):
    return rr.pass_kappa(rr.launch_geometry(GPU_MAX_POINTS, 132), L)


@pytest.mark.parametrize("change", ["drop", "duplicate"])
def test_bar_catches_one_row(dense, change):
    """Teeth: the oracle's rows repeated until they are as many as the largest GPU pass selects, then one row (first,
    middle, last) dropped or doubled: at least one entry leaves kappa * u * sum|t| (kappa of that largest pass)."""
    L, hx, h, R, _, _ = dense
    reps = -(-GPU_MAX_POINTS // hx.shape[0])
    HX, Hv, Rv = np.tile(hx, (reps, 1)), np.tile(h, reps), np.tile(R, reps)
    base = rr.reduce_ref(HX, Hv, Rv)
    kappa = _kappa_max(L)
    n = HX.shape[0]
    for j in (0, n // 2, n - 1):
        keep = np.delete(np.arange(n), j) if change == "drop" else np.insert(np.arange(n), j, j)
        alt = rr.reduce_ref(HX[keep], Hv[keep], Rv[keep])
        worst = rr.entry_ratios(alt["HTH"], alt["HTh"], base).max()
        assert worst > kappa, (j, worst, kappa)
        print(f"L={L} {change} row {j} of {n}: max ratio {worst:.3g} vs kappa {kappa}")
