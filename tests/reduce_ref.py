"""HᵀR⁻¹[H|h] of esekfom.hpp:622-635 (orc_reduce) summed in extended precision, with the absolute mass of every entry.

The terms are orc_reduce's own: t_i(a, b) = fl(h_x[i, a] / r_i) * h_x[i, b] and t_i(a) = fl(h_x[i, a] / r_i) * h[i], with
r_i = R[i] clamped (R < 1e-4 -> 1e-3, esekfom.hpp:624-626).  Their sum is formed

  "longdouble"  in np.longdouble when it has a 64-bit significand (x87 extended): every product and every pairwise partial
                sum rounds at 2^-64, so the sum is within ~log2(N) * 2^-64 * sum|t| of the exact one;
  "fsum"        otherwise (aarch64's long double is a slow software quad): each product split exactly into p + e with
                Dekker's two-product (Veltkamp split) and p, e summed exactly by math.fsum.

Either way the result is the true sum of those terms rounded to float64 (within u/2 of it, u = 2^-53), not another
summation order.  A device result then has to be within kappa * u * sum_i |t_i| of it, entry by entry, where kappa counts
the roundings on the longest dependent chain of the device's summation (pass_kappa) plus the row-level differences.
"""
import math

import numpy as np

U = 2.0 ** -53
LONGDOUBLE_OK = np.finfo(np.longdouble).nmant >= 63
METHOD = "longdouble" if LONGDOUBLE_OK else "fsum"

# the pass kernel's constants (malio_device.cuh): tile of RED_THREADS points, RED_KS row-splits per task
RED_THREADS = 128
RED_KS = 14
PASS_FAST_TILES = 2
# row-level allowance (units of u * |t_i|): device and reference rows are the same formulas with a different rounding
# sequence.  Per term the scaling takes 9 roundings between the two sides (device: a*J, 1/rho, * 1/rho, a*J of the other
# factor; reference: a*J, * w, / r, a*J and * w of the other factor).  Each Jacobian entry is within gamma_k of its
# unsigned magnitude on each side (FMA cross products on the device, skew-matrix products in the reference); the deepest,
# B of a LiDAR l != 0, passes R_s^T n, R_c^T and R_e^T (3 each) and a cross product (2): 11 per side, 22 per factor,
# 44 per term.  Summed over many rows these differences mostly cancel; a LiDAR with a single row keeps them whole.
KAPPA_ROW = 9 + 44


def _clamped(R):
    r = np.asarray(R, np.float64).copy()
    r[r < 0.0001] = 0.001
    return r


def _two_product(a, b):
    """p + e == a * b exactly (Dekker, Veltkamp split; no overflow at these magnitudes)."""
    p = a * b
    f = 134217729.0   # 2^27 + 1
    ca, cb = f * a, f * b
    ah = ca - (ca - a); al = a - ah
    bh = cb - (cb - b); bl = b - bh
    e = al * bl - (((p - ah * bh) - al * bh) - ah * bl)
    return p, e


def reduce_ref(h_x, h, R, method: str | None = None):
    """h_x [N, c], h [N], R [N] (po.Oracle.dense()).  Returns dict(HTH [c, c], HTh [c], mHTH, mHTh = sum_i |t_i| per entry,
    method).  method: None (METHOD), "longdouble" or "fsum"."""
    method = METHOD if method is None else method
    hx = np.ascontiguousarray(h_x, np.float64)
    N, c = hx.shape
    hv = np.asarray(h, np.float64).reshape(N)
    q = hx / _clamped(R).reshape(N, 1)              # orc_reduce's HT, one rounding per entry as there
    X = np.ascontiguousarray(np.column_stack([hx, hv]).T)   # [c + 1, N]: row-contiguous, so sums run pairwise
    Q = np.ascontiguousarray(q.T)                   # [c, N]
    S = np.zeros((c, c + 1))
    M = np.zeros((c, c + 1))
    if method == "longdouble":
        assert LONGDOUBLE_OK, "np.longdouble has no 64-bit significand here"
        Xl = X.astype(np.longdouble)
        for a in range(c):
            T = Q[a].astype(np.longdouble)[None, :] * Xl
            S[a] = T.sum(axis=1).astype(np.float64)
            M[a] = np.abs(T).sum(axis=1).astype(np.float64)
    elif method == "fsum":
        for a in range(c):
            p, e = _two_product(Q[a][None, :], X)
            for b in range(c + 1):
                S[a, b] = math.fsum(p[b].tolist() + e[b].tolist())
            M[a] = np.abs(p).sum(axis=1)
    else:
        raise ValueError(method)
    return dict(HTH=S[:, :c].copy(), HTh=S[:, c].copy(), mHTH=M[:, :c].copy(), mHTh=M[:, c].copy(), method=method)


def launch_geometry(n_points: int, sm_count: int, fused: bool = True, blocks_per_sm: int = 4):
    """The pass launch the host picks (malio_pass.cu pass_geometry()): n_tiles tiles of 128
    points, one co-resident wave of W = blocks_per_sm * SMs blocks (also the slot count red_grid), per_block tiles per
    block, grid blocks; FAST (rows kept in shared memory) while per_block <= 2.  The unfused kernels always use the
    generic reduction over a wave of red_grid blocks."""
    W = blocks_per_sm * sm_count
    n_tiles = (n_points + RED_THREADS - 1) // RED_THREADS
    per_block = (n_tiles + W - 1) // W if n_tiles else 1
    grid = (n_tiles + per_block - 1) // per_block if n_tiles else 1
    fast = bool(fused and per_block <= PASS_FAST_TILES)
    return dict(W=W, n_tiles=n_tiles, per_block=per_block, grid=grid, fast=fast)


def pass_kappa(geo: dict, n_lidar: int) -> int:
    """Longest chain of dependent roundings from one term to an entry of the device's reduced system, plus the row-level
    allowance.  Per block and LiDAR each of the RED_KS worker threads of a task folds every RED_KS-th row with an FMA
    (at most ceil(128 * per_block / RED_KS) of them); the RED_KS splits are added in a fixed order (14); the generic path
    adds the splits into the block's slot once per LiDAR run, at most once per tile (per_block); the fold adds
    ceil(grid / 32) slots per lane, then 5 shuffle rounds; the host adds the LiDARs' compact systems into the shared
    columns (n_lidar) and scales by w * w (2); the comparison rescales the device's system to the oracle's localization
    weight, (w_o / w_d)^2 (3); the reference itself is rounded to float64 (1)."""
    pb = geo["per_block"]
    chain = -(-RED_THREADS * pb // RED_KS)
    flush = 0 if geo["fast"] else pb
    fold = -(-geo["grid"] // 32) + 5
    return chain + RED_KS + flush + fold + n_lidar + 6 + KAPPA_ROW


def entry_ratios(HTH, HTh, ref):
    """|dev - ref| / (u * sum|t|) per entry (inf where the mass is 0 and the entry is not exactly 0, 0 where both are)."""
    d = np.concatenate([np.abs(np.asarray(HTH) - ref["HTH"]).ravel(), np.abs(np.asarray(HTh) - ref["HTh"])])
    m = np.concatenate([ref["mHTH"].ravel(), ref["mHTh"]]) * U
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(m > 0, d / np.where(m > 0, m, 1.0), np.where(d == 0, 0.0, np.inf))
    return r
