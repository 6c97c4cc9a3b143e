"""Host restatement of malio_place_db_build and malio_relocalize_global (include/malio_b200.h, "relocalization without a position
guess"), step by step:
  1. the binning table: stencil, ring by squared radii, sector by quadrant and boundary sign tests, per-ring level caps;
  2. levels: 0 below z_lo, else 1 + clamp(floor((z_rel - z_lo) / dz), 0, 14), capped per ring;
  3. the database: column grids, lattice positions in (j, i) order, z_s, nibbles and ring keys;
  4. the query: the scan registered with pos = 0 (world_ref.register_world), columns around the slot-0 origin;
  5. stages 1 and 2 by sorting, and the verification guess of a candidate.
Every operation is the header's, in float64 (numpy's IEEE arithmetic, no contraction) where the header says double."""
import ctypes as C
import math

import numpy as np

import world_ref
from malio_b200 import capi


def _args_dict(a):
    if isinstance(a, dict):
        return a
    return {f: getattr(a, f) for f, _ in capi.PlaceArgs._fields_}


def ring_radii2(a):
    a = _args_dict(a)
    out = [0.0]
    for k in range(1, a["n_ring"]):
        rk = a["r_max"] * float(k) / float(a["n_ring"])
        out.append(rk * rk)
    return out


def boundaries(a):
    a = _args_dict(a)
    S = a["n_sector"]
    Q = S // 4
    bx, by = [0.0] * Q, [0.0] * Q
    for j in range(1, Q):
        phi = 2.0 * math.pi * float(j) / float(S)
        bx[j], by[j] = math.cos(phi), math.sin(phi)
        if 8 * j == S:
            bx[j] = by[j] = math.sqrt(0.5)
    return bx, by


def ring_of(a, x, y, rad2=None):
    a = _args_dict(a)
    rad2 = ring_radii2(a) if rad2 is None else rad2
    r2 = x * x + y * y
    return sum(1 for k in range(1, a["n_ring"]) if r2 >= rad2[k])


def sector_of(a, x, y, b=None):
    a = _args_dict(a)
    bx, by = boundaries(a) if b is None else b
    Q = a["n_sector"] // 4
    if x > 0 and y >= 0:
        q, u, v = 0, x, y
    elif x <= 0 and y > 0:
        q, u, v = 1, y, -x
    elif x < 0 and y <= 0:
        q, u, v = 2, -x, -y
    else:
        q, u, v = 3, -y, x
    return q * Q + sum(1 for j in range(1, Q) if bx[j] * v - by[j] * u >= 0.0)


def level(z, z_lo, dz):
    """Vectorised level of heights z (float64): 0 where z < z_lo (or NaN)."""
    z = np.asarray(z, np.float64)
    t = np.floor((z - z_lo) / dz)
    t = np.clip(np.nan_to_num(t, nan=0.0), 0.0, 14.0)
    return np.where(z >= z_lo, 1 + t.astype(np.int64), 0)


def caps(a):
    a = _args_dict(a)
    out = np.full(a["n_ring"], 15, np.int64)
    if a["fov_up"] < math.pi / 2:
        tf = math.tan(a["fov_up"])
        for r in range(a["n_ring"]):
            z = (a["r_max"] * float(r) / float(a["n_ring"])) * tf
            out[r] = max(1, int(level(z, a["z_lo"], a["dz"])))
    return out


def table(a):
    """The stencil: int64 arrays ox, oy, ring, sector, bin and the per-entry cap."""
    a = _args_dict(a)
    R = int(math.ceil(a["r_max"] / a["cell"]))
    rad2, b, cp = ring_radii2(a), boundaries(a), caps(a)
    rows = []
    r2max = a["r_max"] * a["r_max"]
    for oy in range(-R, R + 1):
        for ox in range(-R, R + 1):
            if ox == 0 and oy == 0:
                continue
            x, y = float(ox) * a["cell"], float(oy) * a["cell"]
            if not (x * x + y * y < r2max):
                continue
            r, s = ring_of(a, x, y, rad2), sector_of(a, x, y, b)
            rows.append((ox, oy, r, s, r * a["n_sector"] + s, cp[r]))
    t = np.array(rows, np.int64).reshape(-1, 6)
    return dict(ox=t[:, 0], oy=t[:, 1], ring=t[:, 2], sector=t[:, 3], bin=t[:, 4], cap=t[:, 5], R=R)


def occlude(a, d):
    """In every sector, the rings beyond the first bin of level >= block_level emptied (block_level 0: unchanged)."""
    a = _args_dict(a)
    if not a["block_level"]:
        return d
    X = np.asarray(d, np.int64).reshape(a["n_ring"], a["n_sector"]).copy()
    for c in range(a["n_sector"]):
        hit = np.flatnonzero(X[:, c] >= a["block_level"])
        if len(hit):
            X[hit[0] + 1:, c] = 0
    return X.ravel()


def describe(a, tab, heights):
    """heights: float64 per stencil entry (NaN: empty column) -> bin values int64[n_bins] (capped, then occluded)."""
    a = _args_dict(a)
    lv = np.minimum(level(heights, a["z_lo"], a["dz"]), tab["cap"])
    out = np.zeros(a["n_ring"] * a["n_sector"], np.int64)
    np.maximum.at(out, tab["bin"], lv)
    return occlude(a, out)


def ring_keys(a, d):
    a = _args_dict(a)
    return d.reshape(a["n_ring"], a["n_sector"]).sum(axis=1)


def pack(d):
    d = np.asarray(d, np.int64)
    if d.shape[-1] % 2:
        d = np.concatenate([d, np.zeros(d.shape[:-1] + (1,), np.int64)], axis=-1)
    return (d[..., 0::2] | (d[..., 1::2] << 4)).astype(np.uint8)


def unpack(nib, n_bins):
    nib = np.asarray(nib, np.int64)
    out = np.zeros(nib.shape[:-1] + (2 * nib.shape[-1],), np.int64)
    out[..., 0::2], out[..., 1::2] = nib & 15, nib >> 4
    return out[..., :n_bins]


def database(prior, a):
    """The prior (float32 [n, 3]) -> cols int64[p, 2] ((j, i) order), z_s float64[p], levels int64[p, n_bins], ring keys."""
    a = _args_dict(a)
    tab = table(a)
    p = np.asarray(prior, np.float32).reshape(-1, 3)
    nb = a["n_ring"] * a["n_sector"]
    if p.shape[0] == 0:
        return dict(cols=np.zeros((0, 2), np.int64), z_s=np.zeros(0), levels=np.zeros((0, nb), np.int64),
                    ring_keys=np.zeros((0, a["n_ring"]), np.int64))
    ci = np.floor(p[:, 0].astype(np.float64) / a["cell"]).astype(np.int64)
    cj = np.floor(p[:, 1].astype(np.float64) / a["cell"]).astype(np.int64)
    colmax, colmin = {}, {}
    for i, j, z in zip(ci.tolist(), cj.tolist(), p[:, 2].tolist()):
        colmax[(i, j)] = max(colmax.get((i, j), -np.inf), z)
        colmin[(i, j)] = min(colmin.get((i, j), np.inf), z)
    m = int(round(a["step"] / a["cell"]))
    pos = sorted(((j, i) for (i, j) in colmax if i % m == 0 and j % m == 0))
    cols = np.array([(i, j) for j, i in pos], np.int64).reshape(-1, 2)
    z_s = np.array([float(colmin[(i, j)]) + a["sensor_height"] for i, j in cols.tolist()], np.float64)
    levels = np.zeros((len(cols), nb), np.int64)
    for k, (i, j) in enumerate(cols.tolist()):
        h = np.array([colmax.get((i + ox, j + oy), np.nan) for ox, oy in zip(tab["ox"].tolist(), tab["oy"].tolist())], np.float64)
        levels[k] = describe(a, tab, h - z_s[k])
    rk = np.array([ring_keys(a, d) for d in levels], np.int64).reshape(-1, a["n_ring"])
    return dict(cols=cols, z_s=z_s, levels=levels, ring_keys=rk)


def _zero_pos(s):
    ps = s.pass_state() if isinstance(s, capi.State) else s
    out = capi.PassState()
    C.memmove(C.byref(out), C.byref(ps), C.sizeof(capi.PassState))
    out.pos[:] = [0.0, 0.0, 0.0]
    return out


def query_column(rel, cell):
    """A scan point's column offset from the sensor: round half up, floor(rel / cell + 0.5)."""
    return np.floor(rel / cell + 0.5)


def query_heights(s, temporal_comp, pts, a):
    """The resident scan (capi.SCAN_PT) -> {(cx, cy): largest rel z} of the columns around the slot-0 origin."""
    a = _args_dict(a)
    s0 = _zero_pos(s)
    w = world_ref.register_world(s0, temporal_comp, pts["xyz"], pts["lidar"].astype(np.int64), 0.0)[:, :3]
    o = world_ref.register_world(s0, temporal_comp, np.zeros((1, 3), np.float32), np.zeros(1, np.int64), 0.0)[0, :3]
    w = w[np.all(np.isfinite(w), axis=1)]
    rel = w.astype(np.float64) - o.astype(np.float64)
    cx, cy = query_column(rel[:, 0], a["cell"]), query_column(rel[:, 1], a["cell"])
    out = {}
    for x, y, z in zip(cx.tolist(), cy.tolist(), rel[:, 2].tolist()):
        out[(int(x), int(y))] = max(out.get((int(x), int(y)), -np.inf), z)
    return out


def query(s, temporal_comp, pts, a):
    a = _args_dict(a)
    tab = table(a)
    hq = query_heights(s, temporal_comp, pts, a)
    h = np.array([hq.get((ox, oy), np.nan) for ox, oy in zip(tab["ox"].tolist(), tab["oy"].tolist())], np.float64)
    d = describe(a, tab, h)
    return d, ring_keys(a, d)


def stage1(qk, rk, k1):
    """(d1, p) ascending, the first k1: (positions, d1)."""
    d1 = np.abs(np.asarray(rk, np.int64) - np.asarray(qk, np.int64)[None, :]).sum(axis=1)
    order = np.lexsort((np.arange(len(d1)), d1))[:k1]
    return order, d1[order]


def shift_distances(q, d, n_ring, n_sector):
    """sum_r sum_c |Q[r][c] - D[r][(c + s) mod S]| for every s."""
    Q = np.asarray(q, np.int64).reshape(n_ring, n_sector)
    D = np.asarray(d, np.int64).reshape(n_ring, n_sector)
    return np.array([np.abs(Q - np.roll(D, -s, axis=1)).sum() for s in range(n_sector)], np.int64)


def stage2(q, levels, survivors, a, k2):
    """For the stage-1 survivors: (d2, shift) each, and the k2 smallest (d2, p): (positions, d2, shift)."""
    a = _args_dict(a)
    d2, sh = [], []
    for p in survivors:
        ds = shift_distances(q, levels[p], a["n_ring"], a["n_sector"])
        s = int(np.argmin(ds))                                  # the first minimum: ties to the smallest shift
        d2.append(int(ds[s]))
        sh.append(s)
    d2, sh, surv = np.array(d2, np.int64), np.array(sh, np.int64), np.asarray(survivors, np.int64)
    order = np.lexsort((surv, d2))[:k2]
    return surv[order], d2[order], sh[order]


def _qrot(q, v):
    """Eigen's _transformVector in the device's operation order (uv = 2 (qv x v); v + w uv + qv x uv)."""
    qv = [q[1], q[2], q[3]]
    uv = [qv[1] * v[2] - qv[2] * v[1], qv[2] * v[0] - qv[0] * v[2], qv[0] * v[1] - qv[1] * v[0]]
    uv = [u + u for u in uv]
    c2 = [qv[1] * uv[2] - qv[2] * uv[1], qv[2] * uv[0] - qv[0] * uv[2], qv[0] * uv[1] - qv[1] * uv[0]]
    return [v[i] + q[0] * uv[i] + c2[i] for i in range(3)]


def verification_guess(s, col, z_s, shift, a):
    """The state handed to malio_relocalize for a candidate: rot = q_yaw(theta) (x) s.rot, the slot-0 origin at the position."""
    a = _args_dict(a)
    ps = s.pass_state() if isinstance(s, capi.State) else s
    theta = 2.0 * math.pi * float(shift) / float(a["n_sector"])
    c, sn = math.cos(theta / 2.0), math.sin(theta / 2.0)
    w0, x0, y0, z0 = (float(v) for v in ps.rot[:])
    rot = [c * w0 - sn * z0, c * x0 - sn * y0, c * y0 + sn * x0, c * z0 + sn * w0]
    e = _qrot(rot, [float(v) for v in ps.ext[0].t[:]])
    target = [(float(col[0]) + 0.5) * a["cell"], (float(col[1]) + 0.5) * a["cell"], float(z_s)]
    g = capi.PassState()
    C.memmove(C.byref(g), C.byref(ps), C.sizeof(capi.PassState))
    g.rot[:] = rot
    g.pos[:] = [target[i] - e[i] for i in range(3)]
    return g


def verify_args(n_sector, yaw_step):
    w = 1.5 * (2.0 * math.pi / float(n_sector))
    n_yaw = 2 * int(math.ceil(w / yaw_step)) + 1
    return n_yaw, -float(n_yaw // 2) * yaw_step
