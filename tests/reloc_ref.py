"""Host restatement of malio_relocalize (include/malio_b200.h, "relocalization in a loaded prior map"), step by step:
  1. candidate rotations through math.cos / math.sin (the C library's) in the header's operation order;
  2. registered points through world_ref.register_world (the bits malio_world_register gives);
  3. base voxels floor((double)w / res), prior voxels floor((double)x / res);
  4. an exhaustive scorer over every candidate, on a dense occupancy grid;
  5. the tie-break: the first maximum in (k, c, b, a) order, the first candidate when nothing scores.
It also restates the occupancy pyramid (the sliding OR) the device bounds nodes with, so that the bound's admissibility can be
checked apart from the device."""
import ctypes as C
import math

import numpy as np

import world_ref
from malio_b200 import capi


def candidate_rotations(rot, yaw_lo, yaw_step, n_yaw):
    """q_k = q_yaw(theta_k) (x) rot, theta_k = yaw_lo + k * yaw_step, as float64 quadruples (w, x, y, z)."""
    w0, x0, y0, z0 = (float(v) for v in rot)
    out = []
    for k in range(n_yaw):
        theta = yaw_lo + float(k) * yaw_step
        c, s = math.cos(theta / 2.0), math.sin(theta / 2.0)
        out.append((c * w0 - s * z0, c * x0 - s * y0, c * y0 + s * x0, c * z0 + s * w0))
    return out


def _with_rot(s, q):
    ps = s.pass_state() if isinstance(s, capi.State) else s
    out = capi.PassState()
    C.memmove(C.byref(out), C.byref(ps), C.sizeof(capi.PassState))
    out.rot[:] = list(q)
    return out


def base_voxels(s, temporal_comp, pts, q, res):
    """The scan (capi.SCAN_PT) under state s with rot = q -> (int64[n_finite, 3] base voxels, n_finite)."""
    w = world_ref.register_world(_with_rot(s, q), temporal_comp, pts["xyz"], pts["lidar"].astype(np.int64), 0.0)[:, :3]
    fin = np.all(np.isfinite(w), axis=1)
    return np.floor(w[fin].astype(np.float64) / res).astype(np.int64), int(fin.sum())


def prior_voxels(prior, res):
    return np.floor(np.asarray(prior, np.float32).reshape(-1, 3).astype(np.float64) / res).astype(np.int64)


def _occupancy(pv, lo, ext):
    """Dense bool grid over [lo, lo + ext) of the occupied voxels pv."""
    g = np.zeros(tuple(int(e) for e in ext), bool)
    r = pv - lo
    m = np.all((r >= 0) & (r < ext), axis=1)
    g[r[m, 0], r[m, 1], r[m, 2]] = True
    return g


def scores(s, temporal_comp, pts, prior, res, half_xy, half_z, n_yaw, yaw_lo, yaw_step):
    """Every candidate's score as int64[n_yaw, Wz, Wxy (b), Wxy (a)], the finite points per yaw and the rotations."""
    qs = candidate_rotations(s.rot[:], yaw_lo, yaw_step, n_yaw)
    wxy, wz = 2 * half_xy + 1, 2 * half_z + 1
    pv = prior_voxels(prior, res)
    out = np.zeros((n_yaw, wz, wxy, wxy), np.int64)
    n_fin = []
    H = np.array([half_xy, half_xy, half_z])
    for k, q in enumerate(qs):
        b, nf = base_voxels(s, temporal_comp, pts, q, res)
        n_fin.append(nf)
        if nf == 0:
            continue
        lo = b.min(axis=0) - H
        g = _occupancy(pv, lo, b.max(axis=0) + H + 1 - lo)
        r = b - lo - H                                    # cell of base + offset = r + offset + H
        ua = np.arange(wxy)[:, None]
        for c in range(wz):
            for bb in range(wxy):
                out[k, c, bb] = g[r[None, :, 0] + ua, r[None, :, 1] + bb, r[None, :, 2] + c].sum(axis=1)
    return out, n_fin, qs


def relocalize(s, temporal_comp, pts, prior, res, half_xy, half_z, n_yaw, yaw_lo, yaw_step):
    """The exhaustive result as malio_relocalize reports it."""
    sc, n_fin, qs = scores(s, temporal_comp, pts, prior, res, half_xy, half_z, n_yaw, yaw_lo, yaw_step)
    i = int(np.argmax(sc))                                # the first maximum in (k, c, b, a) order; 0 when all are 0
    k, c, b, a = np.unravel_index(i, sc.shape)
    off = (int(a) - half_xy, int(b) - half_xy, int(c) - half_z)
    pos = [float(s.pos[j]) + float(off[j]) * res for j in range(3)]
    return dict(yaw_index=int(k), offset=off, score=int(sc.flat[i]), n_points=n_fin[int(k)], rot=np.array(qs[int(k)]),
                pos=np.array(pos), n_candidates=sc.size, scores=sc)


# ------------------------------------------------------------------ the occupancy pyramid and the node bound
def ceil_log2(w):
    d = 0
    while (1 << d) < w:
        d += 1
    return d


def _shift_or(g, axis, s):
    """g | g shifted by -s along axis (cell v takes v + s), zero beyond the box."""
    out = g.copy()
    if s < g.shape[axis]:
        src = [slice(None)] * 3
        dst = [slice(None)] * 3
        src[axis] = slice(s, None)
        dst[axis] = slice(0, g.shape[axis] - s)
        out[tuple(dst)] |= g[tuple(src)]
    return out


def pyramid(g0, half_xy, half_z):
    """Levels 0 .. L of the sliding OR over the box grid g0: level l splits x / y while l <= ceil(log2(Wxy)) and z while
    l <= ceil(log2(Wz)).  Returns (levels, dxy, dz)."""
    dxy, dz = ceil_log2(2 * half_xy + 1), ceil_log2(2 * half_z + 1)
    levels = [g0]
    for l in range(1, max(dxy, dz) + 1):
        g = levels[-1]
        s = 1 << (l - 1)
        if l <= dxy:
            g = _shift_or(_shift_or(g, 0, s), 1, s)
        if l <= dz:
            g = _shift_or(g, 2, s)
        levels.append(g)
    return levels, dxy, dz


def node_bound(level_grid, rel, u):
    """Sum over the points of G_l[rel + u] (rel: base voxels minus their minimum, u: the node's lattice corner)."""
    r = rel + np.asarray(u)
    return int(level_grid[r[:, 0], r[:, 1], r[:, 2]].sum())
