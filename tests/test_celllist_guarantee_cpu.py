"""CPU property test of the geometric guarantee the k-NN fast path rests on (DESIGN.md (c), knn_direct_kernel /
knn_keys_kernel / ring2_query_warp in ma-lio_b200/csrc/malio_knn.cu).

The device accepts the result of a (2H+1)^3 cell-block scan iff the 5th squared distance (float32, calc_dist's
expression) is below ((H + fmin - 0.005) * h)^2, claiming that every map point OUTSIDE the block is farther than that.
Cells come from float32 arithmetic, floor((x - o) * inv_h) with map points clamped into [0, n-1]; the claim needs that
mapping to be monotone and the 0.005-cell margin to cover its rounding.  This test replays exactly that float32
arithmetic in numpy on adversarial inputs (coordinates up to thousands of cells from the origin, points a few ulps
either side of cell boundaries two/three cells away from the query) and checks the claim by brute force."""
import numpy as np
import pytest

F = np.float32
MARGIN = F(0.005)      # GRID_MARGIN


def _cells(x, o, inv_h, n=None):
    u = (x.astype(F) - F(o)) * F(inv_h)                 # (x - G.ox) * G.inv_h, float32
    c = np.floor(u).astype(np.int64)
    if n is not None:
        c = np.clip(c, 0, n - 1)                          # map points are clamped (grid_count_kernel)
    return c, u


def _calc_dist(q, p):
    d = (q.astype(F) - p.astype(F))
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]   # float32, no FMA


@pytest.mark.parametrize("h,extent_cells", [(1.0, 3500), (0.3, 3900), (2.5, 400), (1.5, 1200)])
@pytest.mark.parametrize("H", [1, 2])
def test_points_outside_the_block_are_beyond_the_accept_radius(h, extent_cells, H):
    rng = np.random.default_rng(int(h * 100) + H)
    inv_h = F(1.0) / F(h)
    o = F(rng.uniform(-500, 500, 3))
    n = extent_cells
    m = 200000
    # queries anywhere in the grid, biased towards the far end (largest float rounding) and towards cell faces
    qc = np.where(rng.random((m, 3)) < 0.5, rng.integers(0, n, (m, 3)), rng.integers(max(n - 50, 0), n, (m, 3)))
    frac = np.where(rng.random((m, 3)) < 0.5, rng.random((m, 3)), rng.choice([1e-6, 1e-3, 0.5, 1 - 1e-3, 1 - 1e-6], (m, 3)))
    q = (o + (qc + frac) * h).astype(F)
    cq, uq = _cells(q, o, inv_h)
    fq = uq - np.floor(uq)
    fmin = np.minimum(fq, F(1.0) - fq).min(axis=1).astype(F)
    r = ((F(H) + fmin - MARGIN) * F(h)).astype(F)
    r2 = r * r
    # map points: one axis exactly H+1 cells away (both directions) within a few ulps of the face, other axes anywhere nearby
    axis = rng.integers(0, 3, m)
    sign = rng.choice([-1, 1], m)
    p = q.astype(np.float64) + rng.uniform(-(H + 1) * h, (H + 1) * h, (m, 3))
    face_cell = cq[np.arange(m), axis] + np.where(sign > 0, H + 1, -H)          # first cell outside / its lower face
    face = o[axis].astype(np.float64) + face_cell * h
    p[np.arange(m), axis] = face
    p = p.astype(F)
    for k in range(-3, 4):                                                        # walk a few ulps across the face
        pk = p.copy()
        col = pk[np.arange(m), axis]
        for _ in range(abs(k)):
            col = np.nextafter(col, F(np.inf) if k > 0 else F(-np.inf))
        pk[np.arange(m), axis] = col
        cp, _ = _cells(pk, o, inv_h, n)
        outside = (np.abs(cp - cq) > H).any(axis=1)
        d2 = _calc_dist(q, pk)
        bad = outside & (d2 < r2)
        assert not bad.any(), (h, H, k, int(bad.sum()), float(d2[bad].min() if bad.any() else 0))
    # the mapping is monotone in each coordinate (what the argument needs), also through the clamp
    xs = np.sort((o[0] + rng.uniform(-2, n + 2, 100000) * h).astype(F))
    c, _ = _cells(xs, o[0], inv_h, n)
    assert np.all(np.diff(c) >= 0)
