"""Seeded synthetic inputs for the measurement hot path (SURVEY.md §8d): an "urban grid" map, a merged
multi-LiDAR scan expressed in each sensor's frame, pose-uncertainty tables, a perturbed prior state.

Deterministic (numpy PCG64).  Used by tests/, bench.py and __graft_entry__.smoke(); the same buffers go to
the CUDA path and to the CPU oracle.  Extrinsics are the reference's /root/reference/Extrinsic.txt values.
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace

import numpy as np

from . import capi

# Extrinsic.txt (LiDAR from IMU): (qw,qx,qy,qz), t
EXTRINSICS = [
    ((1.0, 0.0, 0.0, 0.0), (0.215, 0.0, 0.018)),                                   # Ouster
    ((0.6965018, -0.0037329, -0.0038405, 0.717535), (-1.2574, 0.413, 0.0324)),     # Livox Avia
    ((0.0074645, 0.0000044, -0.0005919, -0.999972), (-1.306, -0.361, 0.042)),      # Livox Tele
]
LIDAR_SPLIT = (0.70, 0.13, 0.17)   # City01 ratio implied by paper Table VI (8554, +1618, +2072)
GRAV_LEN = 9.809


# ------------------------------------------------------------------ quaternion helpers (w,x,y,z), float64
def q_normalize(q):
    q = np.asarray(q, dtype=np.float64)
    return q / np.linalg.norm(q)


def q_mul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx])


def q_conj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def q_exp(v):
    v = np.asarray(v, dtype=np.float64)
    th = np.linalg.norm(v)
    if th < 1e-12:
        return np.array([1.0, 0.0, 0.0, 0.0])
    return np.concatenate([[np.cos(th / 2)], np.sin(th / 2) * v / th])


def q_to_R(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rand_unit(rng, n=3):
    v = rng.normal(size=n)
    return v / np.linalg.norm(v)


# ------------------------------------------------------------------ world
WALL_H = 20.0
LATTICE = 0.5
BLOCK = 50.0


def _wall_lines(half):
    ks = np.arange(-int(half // BLOCK) - 1, int(half // BLOCK) + 2)
    c = BLOCK / 2 + BLOCK * ks
    return c[np.abs(c) <= half]


def make_world(M: int, seed: int = 42) -> np.ndarray:
    """Ground plane z=0 plus a street grid of 20 m walls every 50 m, sampled on a 0.5 m lattice with in-plane
    jitter U(-0.05,0.05) and normal noise N(0,0.01^2); sub-sampled to exactly M points."""
    rng = np.random.default_rng(seed)
    S = 50.0
    while True:
        half = S / 2
        n_side = int(round(S / LATTICE))
        n_lines = len(_wall_lines(half))
        total = n_side * n_side + 2 * n_lines * n_side * int(WALL_H / LATTICE)
        if total >= M:
            break
        S += 10.0
    half = S / 2
    g = (np.arange(n_side) + 0.5) * LATTICE - half
    gx, gy = np.meshgrid(g, g, indexing="ij")
    ground = np.stack([gx.ravel(), gy.ravel(), np.zeros(gx.size)], axis=1)
    ground[:, :2] += rng.uniform(-0.05, 0.05, size=(ground.shape[0], 2))
    ground[:, 2] += rng.normal(0, 0.01, size=ground.shape[0])
    parts = [ground]
    hz = (np.arange(int(WALL_H / LATTICE)) + 0.5) * LATTICE
    for c in _wall_lines(half):
        a, z = np.meshgrid(g, hz, indexing="ij")
        n = a.size
        wx = np.stack([a.ravel() + rng.uniform(-0.05, 0.05, n), np.full(n, c) + rng.normal(0, 0.01, n),
                       z.ravel() + rng.uniform(-0.05, 0.05, n)], axis=1)   # wall along x at y=c
        wy = np.stack([np.full(n, c) + rng.normal(0, 0.01, n), a.ravel() + rng.uniform(-0.05, 0.05, n),
                       z.ravel() + rng.uniform(-0.05, 0.05, n)], axis=1)   # wall along y at x=c
        parts += [wx, wy]
    pts = np.concatenate(parts, axis=0)
    keep = rng.choice(pts.shape[0], size=M, replace=False)
    keep.sort()
    return np.ascontiguousarray(pts[keep].astype(np.float32))


def world_half_extent(M: int) -> float:
    S = 50.0
    while True:
        n_side = int(round(S / LATTICE))
        total = n_side * n_side + 2 * len(_wall_lines(S / 2)) * n_side * int(WALL_H / LATTICE)
        if total >= M:
            return S / 2
        S += 10.0


def sample_surfaces(N: int, center_xy, radius: float, half: float, rng) -> np.ndarray:
    """N points on the ground / walls within `radius` (horizontal) of center_xy, area-weighted."""
    out = []
    need = N
    cx, cy = center_xy
    lo_x, hi_x = max(cx - radius, -half), min(cx + radius, half)
    lo_y, hi_y = max(cy - radius, -half), min(cy + radius, half)
    lines = _wall_lines(half)
    xl = lines[(lines >= lo_y) & (lines <= hi_y)]     # walls along x (at y = c)
    yl = lines[(lines >= lo_x) & (lines <= hi_x)]     # walls along y (at x = c)
    a_ground = (hi_x - lo_x) * (hi_y - lo_y)
    a_xw = len(xl) * (hi_x - lo_x) * WALL_H
    a_yw = len(yl) * (hi_y - lo_y) * WALL_H
    w = np.array([a_ground, a_xw, a_yw])
    w = w / w.sum()
    while need > 0:
        n = int(need * 1.5) + 64
        kind = rng.choice(3, size=n, p=w)
        p = np.zeros((n, 3))
        u = rng.uniform(size=(n, 3))
        m = kind == 0
        p[m, 0] = lo_x + u[m, 0] * (hi_x - lo_x); p[m, 1] = lo_y + u[m, 1] * (hi_y - lo_y); p[m, 2] = 0.0
        m = kind == 1
        if len(xl):
            p[m, 0] = lo_x + u[m, 0] * (hi_x - lo_x); p[m, 1] = xl[(u[m, 1] * len(xl)).astype(int) % len(xl)]; p[m, 2] = u[m, 2] * WALL_H
        m = kind == 2
        if len(yl):
            p[m, 1] = lo_y + u[m, 0] * (hi_y - lo_y); p[m, 0] = yl[(u[m, 1] * len(yl)).astype(int) % len(yl)]; p[m, 2] = u[m, 2] * WALL_H
        ok = (p[:, 0] - cx) ** 2 + (p[:, 1] - cy) ** 2 <= radius * radius
        p = p[ok][:need]
        out.append(p)
        need -= p.shape[0]
    return np.concatenate(out, axis=0)


# ------------------------------------------------------------------ case container
@dataclass
class Case:
    name: str
    n_lidar: int
    max_iter: int
    map_xyz: np.ndarray            # float32 [M,3]
    map_normal_y: np.ndarray       # float32 [M]
    pts: np.ndarray                # capi.SCAN_PT [N]
    table: np.ndarray              # capi.POSE_ENTRY [sum T_l]
    table_off: np.ndarray          # uint32 [L+1]
    temporal_comp: np.ndarray | None   # capi.RIGID [L-1]
    x_true: capi.State
    x_prop: capi.State
    P_prop: np.ndarray             # [n,n]
    params: capi.Params
    meta: dict = field(default_factory=dict)

    @property
    def n_dof(self):
        return 17 + 6 * self.n_lidar


def make_state(pos, rot, ext_q, ext_t, vel=(0, 0, 0), bg=(0, 0, 0), ba=(0, 0, 0), grav=(0, 0, -GRAV_LEN)) -> capi.State:
    s = capi.State()
    s.pos[:] = list(map(float, pos))
    s.rot[:] = list(map(float, rot))
    for l in range(capi.MAX_LIDAR):
        q = ext_q[l] if l < len(ext_q) else (1.0, 0.0, 0.0, 0.0)
        t = ext_t[l] if l < len(ext_t) else (0.0, 0.0, 0.0)
        s.ext[l].q[:] = list(map(float, q))
        s.ext[l].t[:] = list(map(float, t))
    s.vel[:] = list(map(float, vel))
    s.bg[:] = list(map(float, bg))
    s.ba[:] = list(map(float, ba))
    s.grav[:] = list(map(float, grav))
    return s


def state_to_vec(s: capi.State, L: int) -> np.ndarray:
    """flat numeric dump (for comparisons): pos, rot(4), ext q/t, vel, bg, ba, grav"""
    out = list(s.pos) + list(s.rot)
    for l in range(L):
        out += list(s.ext[l].q) + list(s.ext[l].t)
    out += list(s.vel) + list(s.bg) + list(s.ba) + list(s.grav)
    return np.array(out)


def init_P(n: int) -> np.ndarray:
    """IMU_Processing.hpp:188-199 pattern with the pose block at 1e-4 (SURVEY.md §8d)."""
    P = np.eye(n)
    for i in range(6):
        P[i, i] = 1e-4
    for i in range(6, n):
        if i < n - 8:
            P[i, i] = 1e-6
        elif i < n - 5:
            P[i, i] = 1e-4
        elif i < n - 2:
            P[i, i] = 1e-3
        else:
            P[i, i] = 1e-5
    return P


def table_sizes(L: int, T) -> np.ndarray:
    """Per-LiDAR pose-table lengths: one length for all LiDARs, or one per LiDAR (real scans: pose_unc[l] has one entry per
    IMU sample of LiDAR l, laserMapping.cpp:1028-1045).  upload_scan needs at least 2 per LiDAR."""
    sizes = np.full(L, T, dtype=np.int64) if np.isscalar(T) else np.asarray(T, dtype=np.int64)
    assert sizes.shape == (L,) and sizes.min() >= 2, sizes
    return sizes


def make_tables(L: int, T, rng):
    """pose_unc[l][j]: small SE(3) (<= 2 cm, <= 0.2 deg) and covariance growing with j (seed 45 stream).  T: one table
    length for every LiDAR or a sequence of L lengths; table_off is their cumulative sum."""
    sizes = table_sizes(L, T)
    table_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    table = np.zeros(int(table_off[-1]), dtype=capi.POSE_ENTRY)
    for l in range(L):
        axis = rand_unit(rng)
        tdir = rand_unit(rng)
        Tl = int(sizes[l])
        for j in range(Tl):
            f = (j + 1) / Tl
            q = q_exp(axis * np.deg2rad(0.2) * f)
            Tm = np.eye(4)
            Tm[:3, :3] = q_to_R(q)
            Tm[:3, 3] = tdir * 0.02 * f
            d = np.linspace(1e-8, 1e-6, 6) * (0.2 + f)
            A = rng.normal(size=(6, 6)) * 1e-4 * np.sqrt(f)
            cov = np.diag(d) + A @ A.T * 0.05
            table[table_off[l] + j]["T"] = Tm
            table[table_off[l] + j]["cov"] = cov
    return table, table_off


def draw_table_idx(mode: str, lidar: np.ndarray, T, rng) -> np.ndarray:
    """Pose-table index of each scan point.
      in_range  uniform in [0, T_l) of the point's LiDAR;
      edges     T_l - 2, T_l - 1, T_l, T_l + 1 of the point's LiDAR (the two clamps, laserMapping.cpp:694-696 and 737-739);
      raw       what a merged scan carries when the index is the point's intensity (laserMapping.cpp:972-977) and the
                undistortion left that intensity as the raw reflectivity: uniform in 0..255 with ~1 % at 65535."""
    N = lidar.shape[0]
    if mode == "in_range" and np.isscalar(T):
        return rng.integers(0, T, size=N).astype(np.uint16)   # the original draw: default cases stay byte-identical
    sizes = table_sizes(int(lidar.max(initial=0)) + 1, T) if np.isscalar(T) else np.asarray(T, dtype=np.int64)
    if mode == "in_range":
        return rng.integers(0, sizes[lidar]).astype(np.uint16)
    if mode == "edges":
        return (sizes[lidar] + rng.integers(-2, 2, size=N)).astype(np.uint16)
    if mode == "raw":
        idx = rng.integers(0, 256, size=N)
        idx[rng.random(N) < 0.01] = 65535
        return idx.astype(np.uint16)
    raise ValueError(f"table_idx mode {mode!r}")


def world_to_sensor(pw: np.ndarray, lidar: np.ndarray, pos, rot, extq, extt, tcomp) -> np.ndarray:
    """World points -> the frame of the LiDAR that saw them (float64): the inverse of pointBodyToWorld with the temporal
    compensation of LiDARs 1.. (laserMapping.cpp:134-147)."""
    p_imu = (pw - pos) @ q_to_R(rot)      # R^T (p - pos), row-vector form
    xyz = np.zeros((pw.shape[0], 3))
    for l in range(len(extq)):
        m = lidar == l
        v = p_imu[m]
        if l != 0:
            Rc = q_to_R(tcomp[l - 1]["q"])
            v = (v - tcomp[l - 1]["t"]) @ Rc          # qC^T (p - tC)
        Re = q_to_R(extq[l])
        xyz[m] = (v - extt[l]) @ Re                   # qE^T (. - tE)
    return xyz


def make_case(name: str, N: int, M: int, n_lidar: int, max_iter: int, *, varied_map_cov: bool = False,
              seed_world: int = 42, seed_scan: int = 43, seed_state: int = 44, seed_tables: int = 45,
              det_range: float = 100.0, table_T=10, map_xyz: np.ndarray | None = None,
              pos_err: float = 0.10, rot_err_deg: float = 0.5, table_idx: str = "in_range") -> Case:
    """table_T: pose-table length of every LiDAR, or one length per LiDAR; table_idx: see draw_table_idx."""
    L = n_lidar
    if map_xyz is None:
        map_xyz = make_world(M, seed_world)
    half = world_half_extent(M)
    rng_w = np.random.default_rng(seed_world + 1000)
    if varied_map_cov:
        map_ny = rng_w.uniform(0.0005, 0.02, size=M).astype(np.float32)
        map_ny[rng_w.uniform(size=M) < 0.02] = 0.0   # exercises the W(0,0) > 1e-5 gate and cov_plane == 0
    else:
        map_ny = np.full(M, 0.001, dtype=np.float32)   # laserMapping.cpp:1004

    rng = np.random.default_rng(seed_scan)
    pos_true = np.array([1.0, 2.0, 1.8])
    rot_true = q_mul(q_exp([0, 0, 0.3]), q_exp([0.02, -0.015, 0.0]))
    extq = [q_normalize(EXTRINSICS[l][0]) for l in range(L)]
    extt = [np.array(EXTRINSICS[l][1]) for l in range(L)]
    rng_t = np.random.default_rng(seed_tables)
    tcomp = np.zeros(max(L - 1, 0), dtype=capi.RIGID)
    for l in range(1, L):
        tcomp[l - 1]["q"] = q_exp(rand_unit(rng_t) * np.deg2rad(0.3))
        tcomp[l - 1]["t"] = rand_unit(rng_t) * 0.05
    table, table_off = make_tables(L, table_T, rng_t)

    pw = sample_surfaces(N, pos_true[:2], min(det_range, half), half, rng)
    pw += rng.normal(0, 0.02, size=pw.shape)
    split = np.array(LIDAR_SPLIT[:L], dtype=np.float64)
    split = split / split.sum()
    counts = np.floor(split * N).astype(int)
    counts[0] += N - counts.sum()
    lidar = np.repeat(np.arange(L), counts)
    pts = np.zeros(N, dtype=capi.SCAN_PT)
    pts["xyz"] = world_to_sensor(pw, lidar, pos_true, rot_true, extq, extt, tcomp).astype(np.float32)
    pts["lidar"] = lidar.astype(np.uint16)
    pts["table_idx"] = draw_table_idx(table_idx, lidar, table_T, rng)

    rs = np.random.default_rng(seed_state)
    x_true = make_state(pos_true, rot_true, extq, extt, vel=rs.normal(0, 0.5, 3), bg=rs.normal(0, 1e-3, 3),
                        ba=rs.normal(0, 1e-2, 3))
    pos_p = pos_true + rand_unit(rs) * pos_err
    rot_p = q_mul(rot_true, q_exp(rand_unit(rs) * np.deg2rad(rot_err_deg)))
    extq_p = [q_mul(extq[l], q_exp(rand_unit(rs) * np.deg2rad(0.1))) for l in range(L)]
    extt_p = [extt[l] + rand_unit(rs) * 0.01 for l in range(L)]
    x_prop = make_state(pos_p, rot_p, extq_p, extt_p, vel=x_true.vel[:], bg=x_true.bg[:], ba=x_true.ba[:])
    prm = capi.default_params(L)
    return Case(name, L, max_iter, map_xyz, map_ny, pts, table, table_off, tcomp if L > 1 else None, x_true, x_prop,
                init_P(17 + 6 * L), prm, meta=dict(N=N, M=M, half=half))


# ------------------------------------------------------------------ scenes derived from a case
def _sensor_points(case: Case, pw: np.ndarray, rng) -> np.ndarray:
    """World points as scan points of `case` (seen from its true state), LiDARs assigned round-robin, table index in range."""
    n = pw.shape[0]
    lidar = np.arange(n) % case.n_lidar
    s = case.x_true
    extq = [np.array(s.ext[l].q[:]) for l in range(case.n_lidar)]
    extt = [np.array(s.ext[l].t[:]) for l in range(case.n_lidar)]
    pts = np.zeros(n, dtype=capi.SCAN_PT)
    pts["xyz"] = world_to_sensor(pw, lidar, np.array(s.pos[:]), np.array(s.rot[:]), extq, extt,
                                 case.temporal_comp).astype(np.float32)
    pts["lidar"] = lidar.astype(np.uint16)
    sizes = np.diff(case.table_off.astype(np.int64))
    pts["table_idx"] = rng.integers(0, sizes[lidar]).astype(np.uint16)
    return pts


def with_scan(case: Case, pw: np.ndarray, *, keep: int = 0, seed: int = 0, name: str | None = None, **changes) -> Case:
    """A copy of `case` whose scan is its first `keep` points followed by the world points `pw` (seen from the true state);
    other fields may be replaced through `changes` (e.g. map_xyz, map_normal_y)."""
    pts = np.concatenate([case.pts[:keep], _sensor_points(case, np.asarray(pw, np.float64).reshape(-1, 3),
                                                            np.random.default_rng(seed))])
    meta = dict(case.meta, N=int(pts.shape[0]))
    return replace(case, name=name or case.name, pts=pts, meta=meta, **changes)


def translated(case: Case, offset) -> Case:
    """The same scene moved by `offset` (metres): map points (rounded to float32 again) and both states' positions.  The
    scan is in sensor frames and does not change."""
    off = np.asarray(offset, np.float64)
    xt, xp = case.x_true.copy(), case.x_prop.copy()
    xt.pos[:] = list(np.array(xt.pos[:]) + off)
    xp.pos[:] = list(np.array(xp.pos[:]) + off)
    return replace(case, name=f"{case.name} +{off.tolist()}", x_true=xt, x_prop=xp,
                   map_xyz=np.ascontiguousarray((case.map_xyz.astype(np.float64) + off).astype(np.float32)))


def surface_scan_points(case: Case, n_ground: int, n_xwall: int, n_ywall: int, seed: int = 0) -> np.ndarray:
    """World points on the ground (z = 0) and on the two walls of the street grid closest to the true position (the wall
    along x at y = c and the one along y at x = c), with the scan's 2 cm noise.  The mix sets the spread of plane normals
    and so the ratio of the singular values behind the localization weight (laserMapping.cpp:745-756): ground only
    gives sigma3/sigma1 ~ 0, a box room with equal shares ~ 1."""
    rng = np.random.default_rng(seed)
    px, py = case.x_true.pos[0], case.x_true.pos[1]
    lines = _wall_lines(case.meta["half"])
    cy = lines[np.argmin(np.abs(lines - py))]
    cx = lines[np.argmin(np.abs(lines - px))]
    r = np.sqrt(rng.uniform(0, 1, n_ground)) * 15.0
    a = rng.uniform(-np.pi, np.pi, n_ground)
    ground = np.stack([px + r * np.cos(a), py + r * np.sin(a), np.zeros(n_ground)], axis=1)
    xwall = np.stack([px + rng.uniform(-15, 15, n_xwall), np.full(n_xwall, cy), rng.uniform(0.5, 15, n_xwall)], axis=1)
    ywall = np.stack([np.full(n_ywall, cx), py + rng.uniform(-15, 15, n_ywall), rng.uniform(0.5, 15, n_ywall)], axis=1)
    pw = np.concatenate([ground, xwall, ywall])
    return pw + rng.normal(0, 0.02, size=pw.shape)


# Degenerate plane-fit neighbourhoods (esti_plane, common_lib.h:144-190) planted into a map around known scan points:
#   duplicates     6 copies of one point (A has rank 1; x == y at the site, so two column norms tie exactly)
#   pole           a vertical line at 5 cm spacing (rank 2; again x == y)
#   floor_z0       a patch exactly at z = 0 (a zero column; the plane holds the world origin)
#   origin_plane   a vertical plane through the world origin (A n = -1 has no exact solution)
#   cluster        6 points within 1e-4 m
#   zero_weight    a plane patch whose map weights are all <= 1e-5 (the W(0,0) gate: plane_cov = 0, weight 1)
#   cov_threshold  a plane patch whose map weights all equal cov_threshold (cov_sum = 0: esti_plane computes 0/0)
DEGENERATE_KINDS = ("duplicates", "pole", "floor_z0", "origin_plane", "cluster", "zero_weight", "cov_threshold")


def degenerate_sites(kinds, per_kind: int, half: float):
    """Site centres on a 10 m grid, >= 5 m from every wall and, in the air, >= 5 m above the ground; the two kinds that
    need x == y take diagonal cells.  Returns [(kind, (x, y, z))]."""
    g = np.arange(-half + 5.0, half - 4.0, 10.0)
    diag = [(v, v) for v in g if v != 0.0]
    off = [(x, y) for x in g for y in g if x != y and not (x == 0.0 and y == 0.0)]
    out, nd, no = [], 0, 0
    for k in kinds:
        for i in range(per_kind):
            if k in ("duplicates", "pole"):
                x, y = diag[nd]; nd += 1
            else:
                x, y = off[no]; no += 1
            z = 0.0 if k == "floor_z0" else 5.0 + 5.0 * (i % 3)
            out.append((k, (float(x), float(y), z)))
    return out


def plant_degenerate(map_xyz: np.ndarray, map_ny: np.ndarray, sites, cov_threshold: float = 0.5, seed: int = 0):
    """Clear the map within 4 m of every site and plant the site's structure there.  Returns (map_xyz, map_ny, scan_world
    [n,3], scan_site [n]): three scan points per site, each with its 5 nearest map points inside the structure."""
    rng = np.random.default_rng(seed)
    keep = np.ones(map_xyz.shape[0], bool)
    for _, c in sites:
        keep &= np.sum((map_xyz.astype(np.float64) - c) ** 2, axis=1) > 16.0
    xyz, ny = [map_xyz[keep].astype(np.float64)], [map_ny[keep]]
    scan, owner = [], []
    for s, (kind, c) in enumerate(sites):
        c = np.asarray(c, np.float64)
        uv = np.arange(-1.5, 1.5001, 0.25)
        U, V = np.meshgrid(uv, uv, indexing="ij")
        U, V = U.ravel(), V.ravel()
        w = np.full(U.size, 0.001, np.float32)
        near = np.array([[0.03, -0.02, 0.04], [-0.04, 0.05, 0.02], [0.02, 0.03, -0.05]])
        if kind == "duplicates":
            p = np.repeat(c[None], 6, axis=0)
            w = np.full(6, 0.001, np.float32)
        elif kind == "pole":
            p = c + np.outer(np.arange(-6, 7) * 0.05, [0.0, 0.0, 1.0])
            w = np.full(p.shape[0], 0.001, np.float32)
            near = np.array([[0.04, 0.07, 0.012], [-0.03, 0.02, 0.11], [0.05, -0.04, -0.09]])
        elif kind == "floor_z0":
            p = np.stack([c[0] + U, c[1] + V, np.zeros(U.size)], axis=1)
            near = np.array([[0.1, -0.07, 0.03], [-0.12, 0.05, 0.02], [0.06, 0.11, -0.02]])
        elif kind == "origin_plane":
            d = np.array([c[0], c[1], 0.0]) / np.hypot(c[0], c[1])   # in-plane horizontal direction: the plane holds 0
            nrm = np.array([-d[1], d[0], 0.0])
            p = c + np.outer(U, d) + np.outer(V, [0.0, 0.0, 1.0])
            near = np.array([0.1 * d + 0.03 * nrm, -0.08 * d + [0, 0, 0.1] - 0.02 * nrm, 0.05 * d - [0, 0, 0.07] + 0.04 * nrm])
        elif kind == "cluster":
            p = c + rng.uniform(-1e-4, 1e-4, size=(6, 3))
            w = np.full(6, 0.001, np.float32)
            near = np.array([[0.01, 0.005, -0.008], [-0.006, 0.01, 0.004], [0.003, -0.009, 0.01]])
        elif kind in ("zero_weight", "cov_threshold"):
            p = np.stack([c[0] + U, c[1] + V, np.full(U.size, c[2])], axis=1)
            if kind == "zero_weight":
                w = np.array([0.0, 1e-6, 1e-5], np.float32)[np.arange(U.size) % 3]
            else:
                w = np.full(U.size, cov_threshold, np.float32)
            near = np.array([[0.1, -0.07, 0.03], [-0.12, 0.05, 0.02], [0.06, 0.11, -0.02]])
        else:
            raise ValueError(kind)
        xyz.append(p); ny.append(w)
        scan.append(c + near); owner += [s] * near.shape[0]
    return (np.ascontiguousarray(np.concatenate(xyz).astype(np.float32)), np.ascontiguousarray(np.concatenate(ny).astype(np.float32)),
            np.concatenate(scan), np.array(owner))


# BASELINE.json configs
def case_C1():
    return make_case("C1 single-LiDAR 5k scan vs 50k map, 3 iters", 5000, 50000, 1, 3)


def case_C2():
    return make_case("C2 3-LiDAR 100k scan vs 1M map", 100000, 1000000, 3, 3)


def case_C4():
    return make_case("C4 dense urban 300k scan vs 5M map, 5 iters", 300000, 5000000, 3, 5)


def knn_microbench(M: int = 10_000_000, Q: int = 1_000_000, seed_map: int = 42, seed_q: int = 43):
    """C5: uniform points in [-500,500]^2 x [-5,5]; queries = random map points + N(0, 0.1^2)."""
    rng = np.random.default_rng(seed_map)
    xyz = np.empty((M, 3), dtype=np.float32)
    xyz[:, 0] = rng.uniform(-500, 500, M)
    xyz[:, 1] = rng.uniform(-500, 500, M)
    xyz[:, 2] = rng.uniform(-5, 5, M)
    rq = np.random.default_rng(seed_q)
    q = xyz[rq.integers(0, M, Q)] + rq.normal(0, 0.1, size=(Q, 3)).astype(np.float32)
    return xyz, np.ascontiguousarray(q.astype(np.float32))


# ------------------------------------------------------------------ N2: raw scan + spline for the undistortion (SURVEY.md §8f)
def _se3(q, t):
    T = np.eye(4)
    T[:3, :3] = q_to_R(q)
    T[:3, 3] = t
    return T


#   generic       the default: ~0.7 rad heading plus ~0.6 rad/s about a random axis (every pair turns by ~6e-3 rad)
#   stationary    every control pose equal (log_se3's zero-rotation branch, exp_se3's small-angle branch)
#   straight      20 m/s along the heading with yaw increments per 10 ms pair cycling through 5e-8, 1e-4, 2e-4, 3e-4 and
#                 3.3e-4 rad: most pairs are under log_so3's Taylor threshold (~3.16e-4 rad), some just above it, and the
#                 5e-8 pairs reach exp_se3's small-angle branch with a 0.2 m translation.  All turns share the body z axis.
#   heading_x/y/z base rotations 2.2 rad about x, 2.7 rad about y, pi - 1e-3 about z: the rotation matrices have trace <= 0,
#                 so Eigen's matrix->quaternion takes its else branch with i = 0, 1, 2; plus a 0.3 rad/s turn
#   heading_wrap  yaw about z from ~pi - 0.08 to ~pi + 0.08 across the scan: the heading crosses +-pi mid-scan
#   fast          ~10 rad/s about a random axis
UNDISTORT_MOTIONS = ("generic", "stationary", "straight", "heading_x", "heading_y", "heading_z", "heading_wrap", "fast")
STRAIGHT_YAW_STEPS = (5e-8, 1e-4, 2e-4, 3e-4, 3.3e-4)
# covariance-list / control-point layouts:
#   default     the list from before the scan start to past its end, cov_pointer as IMU_Processing.hpp:455-466 leaves it
#   empty_cov   n_cov = 0, cov_pointer = -1
#   last_cov    cov_pointer = n_cov - 1 (every entry may be popped)
#   max         n_ctrl = MALIO_MAX_CTRL and n_cov = MALIO_MAX_COV (512 each), the scan at the end of both lists
UNDISTORT_LISTS = ("default", "empty_cov", "last_cov", "max")
MAX_CTRL = 512
MAX_COV = 512


def undistort_case(n: int = 60000, lidar: int = 0, seed: int = 51, scan_ms: float = 100.0, imu_hz: float = 200.0,
                   sorted_times: bool = True, *, motion: str = "generic", ties: bool = False, lists: str = "default"):
    """One LiDAR's raw scan for UndistortPcl's point loop: n points with time offsets (`curvature`, ms) over one scan, a
    cubic-spline control-point set at the reference's fixed 10 ms spacing (BsplineSE3.cpp:34) covering the scan with two
    control points of margin on both sides (by default a smooth vehicle motion: ~8 m/s, ~0.6 rad/s), the IMU-covariance
    time list at imu_hz, and cov_pointer as IMU_Processing.hpp:455-466 leaves it.  Returns a dict of plain arrays.

    motion: one of UNDISTORT_MOTIONS; lists: one of UNDISTORT_LISTS.  ties: control-point and covariance stamps are built
    as float64(ms_f32) / 1000 + beg_time, the expression of IMU_Processing.hpp:474, and some points carry exactly those
    ms values, so their times equal a control-point or a covariance stamp bit for bit; every 7th covariance stamp is
    duplicated.  With the defaults the output is the same, byte for byte, as before these options existed."""
    if motion not in UNDISTORT_MOTIONS or lists not in UNDISTORT_LISTS:
        raise ValueError(f"motion {motion!r} / lists {lists!r}")
    rng = np.random.default_rng(seed)
    t0 = 1000.0 + 0.0137          # lidar_beg_time
    end_time = t0 + scan_ms * 1e-3
    n_ctrl = int(scan_ms / 10) + 8
    k_ctrl = np.arange(n_ctrl) if lists != "max" else np.arange(MAX_CTRL) - (MAX_CTRL - n_ctrl)
    if ties:
        ctrl_ms = (-31.0 + 10.0 * k_ctrl).astype(np.float32)
        ctrl_t = ctrl_ms.astype(np.float64) / 1000.0 + t0
    else:
        ctrl_t = t0 - 0.031 + 0.01 * k_ctrl
    axis = rand_unit(rng)
    w = axis * {"fast": 10.0}.get(motion, 0.6)
    v = np.array([8.0, 0.5, -0.1])
    acc = rng.normal(0, 1.0, 3)
    q_base = q_exp([0.1, -0.05, 0.7])
    p_base = np.array([3.0, -2.0, 1.5])
    if motion == "straight":
        steps = np.array(STRAIGHT_YAW_STEPS)[np.arange(ctrl_t.shape[0]) % len(STRAIGHT_YAW_STEPS)]
        yaw = np.concatenate([[0.0], np.cumsum(steps[:-1])])
    heading = {"heading_x": [2.2, 0, 0], "heading_y": [0, 2.7, 0], "heading_z": [0, 0, np.pi - 1e-3]}
    ctrl_T = np.zeros((ctrl_t.shape[0], 4, 4))
    for k, tk in enumerate(ctrl_t):
        dt = tk - t0
        noise = rng.normal(0, 0.01, 3)
        p = p_base + v * dt + 0.5 * acc * dt * dt
        if motion in ("generic", "fast"):
            q = q_mul(q_base, q_exp(w * dt + 0.5 * noise * dt * dt))
        elif motion == "stationary":
            q, p = q_base, p_base
        elif motion == "straight":
            q = q_mul(q_base, q_exp([0.0, 0.0, yaw[k]]))
            p = p_base + q_to_R(q_base) @ np.array([20.0 * dt, 0.0, 0.0])
        elif motion in heading:
            q = q_mul(q_exp(heading[motion]), q_exp(axis * 0.3 * dt))
        else:   # heading_wrap
            q = q_mul(q_exp([0.02, -0.01, 0.0]), q_exp([0.0, 0.0, np.pi + 1.0 * (dt - 0.5 * scan_ms * 1e-3)]))
        ctrl_T[k] = _se3(q, p)
    pts = np.zeros(n, dtype=capi.RAW_PT)
    rad = rng.uniform(1.0, 80.0, n)
    az = rng.uniform(-np.pi, np.pi, n)
    el = rng.uniform(-0.4, 0.4, n)
    pts["xyz"] = np.stack([rad * np.cos(el) * np.cos(az), rad * np.cos(el) * np.sin(az), rad * np.sin(el)], axis=1).astype(np.float32)
    curv = rng.uniform(0.0, scan_ms, n).astype(np.float32)
    # imu_cov: forward-propagation stamps from before the scan start to past its end (IMU_Processing.hpp:327-360)
    n_cov = int((scan_ms * 1e-3 + 0.02) * imu_hz)
    k_cov = np.arange(n_cov) if lists != "max" else np.arange(MAX_COV) - (MAX_COV - n_cov)
    if ties:
        cov_ms = (-4.0 + 1000.0 * k_cov / imu_hz).astype(np.float32)
        cov_t = cov_ms.astype(np.float64) / 1000.0 + t0
        cov_t = np.repeat(cov_t, np.where(np.arange(cov_t.shape[0]) % 7 == 3, 2, 1))
        if lists == "max":   # still MAX_COV entries: the oldest ones make room for the duplicates
            cov_t = cov_t[-MAX_COV:]
        # points at control-point and covariance stamps inside the scan, two at each
        in_scan = lambda ms: ms[(ms >= 0) & (ms <= scan_ms)]
        tie_ms = np.repeat(np.concatenate([in_scan(ctrl_ms), in_scan(cov_ms)]), 2)
        at = np.random.default_rng(seed + 1).choice(n, size=min(n, tie_ms.shape[0]), replace=False)
        curv[at] = tie_ms[: at.shape[0]]
    else:
        cov_t = t0 - 0.004 + k_cov / imu_hz
    pts["curvature"] = np.sort(curv) if sorted_times else curv
    if lists == "empty_cov":
        cov_t = cov_t[:0]
        cp = -1
    else:
        cp = cov_t.shape[0] - 1
        while cov_t[cp] > end_time:   # :455-466
            cp -= 1
        cp += 1
        cp = min(cp, cov_t.shape[0] - 1)
        if lists == "last_cov":
            cp = cov_t.shape[0] - 1
    ext = (q_normalize(EXTRINSICS[lidar][0]), np.array(EXTRINSICS[lidar][1]))
    return dict(pts=pts, beg_time=t0, end_time=end_time, ctrl_t=ctrl_t, ctrl_T=ctrl_T.reshape(-1, 16), imu_cov_t=cov_t,
                cov_pointer=int(cp), extrinsic=ext)


# ------------------------------------------------------------------ a street with traffic, ray-cast (clearing moving objects)
@dataclass
class Street:
    """A straight street along +x: ground z = 0, façades at y = +-half_width up to facade_h, parked boxes beside the right
    façade, and one car-sized box driving along the other lane.  The sensor drives along y = ego_y at sensor_z."""
    half_width: float = 8.0
    facade_h: float = 12.0
    ego_y: float = 1.5
    sensor_z: float = 1.8
    ego_x0: float = 0.0
    ego_step: float = 0.5          # m per scan
    car_y: float = -2.5
    car_x0: float = 20.0
    car_step: float = -1.5         # m per scan (oncoming)
    car_size: tuple = (4.5, 1.8, 1.4)
    car_z0: float = 0.25
    max_range: float = 80.0        # the sensor returns nothing beyond this
    noise: float = 0.01            # m, range noise (1 sigma)
    gone: tuple = ()               # indices into the default parked boxes that have left (a later session of the same street)
    extra: tuple = ()              # boxes (lo, hi) that have appeared, after the remaining parked ones

    def parked(self) -> list:
        boxes = [(np.array([x, 4.6, 0.0]), np.array([x + 4.0, 6.4, 1.4])) for x in np.arange(-12.0, 48.0, 9.0)]
        return [b for i, b in enumerate(boxes) if i not in self.gone] + [(np.asarray(lo, float), np.asarray(hi, float)) for lo, hi in self.extra]

    def car(self, k: int):
        sx, sy, sz = self.car_size
        x = self.car_x0 + self.car_step * k
        return np.array([x - sx / 2, self.car_y - sy / 2, self.car_z0]), np.array([x + sx / 2, self.car_y + sy / 2, self.car_z0 + sz])

    def ego(self, k: int) -> np.ndarray:
        return np.array([self.ego_x0 + self.ego_step * k, self.ego_y, self.sensor_z])


def _ray_box(O, D, lo, hi):
    """Entry parameter of rays O + t D (t > 0) into an axis-aligned box, inf where they miss it."""
    with np.errstate(divide="ignore", invalid="ignore"):
        t1, t2 = (lo - O) / D, (hi - O) / D
    tn = np.nanmax(np.minimum(t1, t2), axis=1)
    tf = np.nanmin(np.maximum(t1, t2), axis=1)
    return np.where((tf >= tn) & (tn > 1e-6), tn, np.inf)


def street_cast(street: Street, k: int, O: np.ndarray, D: np.ndarray, rng):
    """Cast unit rays D from O at scan k.  Returns (hit points float64 (m, 3), what float (m,): 0 ground, 1 façade, 2 parked,
    3 the moving car), rays without a return dropped."""
    n = D.shape[0]
    best = np.full(n, np.inf)
    what = np.full(n, -1)
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = np.where(D[:, 2] < 0, -O[:, 2] / D[:, 2], np.inf)
        best, what = np.where(tg < best, tg, best), np.where(tg < best, 0, what)
        for y in (street.half_width, -street.half_width):
            tw = (y - O[:, 1]) / D[:, 1]
            z = O[:, 2] + tw * D[:, 2]
            tw = np.where((tw > 0) & (z >= 0) & (z <= street.facade_h), tw, np.inf)
            best, what = np.where(tw < best, tw, best), np.where(tw < best, 1, what)
    for lo, hi in street.parked():
        tb = _ray_box(O, D, lo, hi)
        best, what = np.where(tb < best, tb, best), np.where(tb < best, 2, what)
    lo, hi = street.car(k)
    tb = _ray_box(O, D, lo, hi)
    best, what = np.where(tb < best, tb, best), np.where(tb < best, 3, what)
    ok = best <= street.max_range
    t = best[ok] + rng.normal(0.0, street.noise, int(ok.sum()))
    return O[ok] + t[:, None] * D[ok], what[ok]


def _spinning_dirs(n_el: int, n_az: int, az0: float) -> np.ndarray:
    el = np.radians(np.linspace(-22.5, 22.5, n_el))
    az = az0 + np.arange(n_az) * (2 * np.pi / n_az)
    E, A = np.meshgrid(el, az, indexing="ij")
    return np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], axis=-1).reshape(-1, 3)


def _cone_dirs(n: int, yaw: float, rng) -> np.ndarray:
    a = yaw + rng.uniform(-np.radians(35), np.radians(35), n)
    e = rng.uniform(-np.radians(25), np.radians(10), n)
    return np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], axis=1)


STREET_EXT_T = [np.zeros(3), np.array([0.4, 0.3, 0.1]), np.array([-0.4, -0.3, 0.1])]   # slot origins relative to the sensor


def street_scan(street: Street, k: int, L: int = 1, spin=(32, 128), cone: int = 0, seed: int = 0):
    """Scan k of the drive as L slots.  Slot 0 spins (spin = (elevations, azimuths), the azimuths shifted per scan); slots 1 and 2
    look forward and backward with `cone` random rays each.  Returns dict(state, body: L float32 (m_l, 3) clouds in their slot's
    frame (identity rotations, the slot's translation in the state's extrinsics), what: L int arrays (street_cast's labels))."""
    rng = np.random.default_rng((seed, k))
    pos = street.ego(k)
    body, what = [], []
    for l in range(L):
        o = pos + STREET_EXT_T[l]
        D = _spinning_dirs(spin[0], spin[1], rng.uniform(0, 2 * np.pi / spin[1])) if l == 0 else _cone_dirs(cone, 0.0 if l == 1 else np.pi, rng)
        p, wh = street_cast(street, k, np.broadcast_to(o, D.shape), D, rng)
        body.append((p - o).astype(np.float32))
        what.append(wh)
    qid = np.array([1.0, 0.0, 0.0, 0.0])
    state = make_state(pos, qid, [qid] * L, STREET_EXT_T[:L])
    return dict(state=state, body=body, what=what)


def street_scan_city(street: Street, k: int, seed: int = 0):
    """A City-size scan: 128 x 1024 spinning rays and 2 x 24000 cone rays (slots 0, 1, 2), before the rays without a return
    are dropped."""
    return street_scan(street, k, L=3, spin=(128, 1024), cone=24000, seed=seed)
