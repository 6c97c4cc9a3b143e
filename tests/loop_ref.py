"""numpy restatement of malio_scan_store_match (include/malio_b200.h, "Closing loops over the scan store"), bit for bit: the
target and source rows through scan_store_ref / world_ref, the per-level plane model (sums in row order, cyclic Jacobi with
MALIO_MATCH_JACOBI_SWEEPS sweeps), the correspondence over the 27 voxels, the 29 sums of each inlier as a perfect binary tree,
the host's Cholesky solve and right-perturbation update (malio_se3.h's exp_se3, quat_from_R, q_mul, q_rot in Python floats,
whose arithmetic is the host's with -ffp-contract=off), and the report.  Every elementwise numpy operation on float64 is one
IEEE rounding, as each device operation is (-fmad=false)."""
import math

import numpy as np

import scan_store_ref as SR
import world_ref as W
from malio_b200 import capi

SWEEPS = capi.MATCH_JACOBI_SWEEPS
KEY_RANGE = capi.MATCH_KEY_RANGE
NSUM = 29


# ------------------------------------------------------------------ malio_se3.h in Python floats, the header's operation order
def q_to_R(q):
    w, x, y, z = (float(v) for v in q)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)]


def cross3(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def q_rot(q, v):
    qv = [q[1], q[2], q[3]]
    uv = cross3(qv, v)
    uv = [u + u for u in uv]
    c2 = cross3(qv, uv)
    return [(v[i] + q[0] * uv[i]) + c2[i] for i in range(3)]


def q_rot_conj(q, v):
    return q_rot([q[0], -q[1], -q[2], -q[3]], v)


def q_mul(a, b):
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]]


def mul3(A, B):
    return [A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j] for i in range(3) for j in range(3)]


def exp_se3(vec):
    w0, w1, w2 = vec[0], vec[1], vec[2]
    theta = math.sqrt(w0 * w0 + w1 * w1 + w2 * w2)
    K = [0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0]
    if theta < 1e-7:
        A, B, Cc = 1.0, 0.5, 1.0 / 6.0
    else:
        A = math.sin(theta) / theta
        B = (1 - math.cos(theta)) / (theta * theta)
        Cc = (1 - A) / (theta * theta)
    K2 = mul3(K, K)
    V, mat = [0.0] * 9, [0.0] * 16
    for i in range(9):
        I = 1.0 if i % 4 == 0 else 0.0
        V[i] = I + B * K[i] + Cc * K2[i]
        mat[4 * (i // 3) + (i % 3)] = I + A * K[i] + B * K2[i]
    for i in range(3):
        mat[4 * i + 3] = V[3 * i] * vec[3] + V[3 * i + 1] * vec[4] + V[3 * i + 2] * vec[5]
    mat[12:16] = [0.0, 0.0, 0.0, 1.0]
    return mat


def quat_from_R(m):
    t = m[0] + m[4] + m[8]
    if t > 0.0:
        t = math.sqrt(t + 1.0)
        w = 0.5 * t
        t = 0.5 / t
        return [w, (m[7] - m[5]) * t, (m[2] - m[6]) * t, (m[3] - m[1]) * t]
    i = 0
    if m[4] > m[0]:
        i = 1
    if m[8] > m[4 * i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    t = math.sqrt(m[4 * i] - m[4 * j] - m[4 * k] + 1.0)
    qv = [0.0] * 3
    qv[i] = 0.5 * t
    t = 0.5 / t
    w = (m[3 * k + j] - m[3 * j + k]) * t
    qv[j] = (m[3 * j + i] + m[3 * i + j]) * t
    qv[k] = (m[3 * k + i] + m[3 * i + k]) * t
    return [w, qv[0], qv[1], qv[2]]


def right_update(q, p, delta):
    """q <- normalize(q (x) quat_from_R(R(exp_se3(delta)))), p <- p + q_rot(q_old, t(exp_se3(delta)))."""
    T = exp_se3(delta)
    qd = quat_from_R([T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]])
    qn = q_mul(q, qd)
    dp = q_rot(q, [T[3], T[7], T[11]])
    nrm = math.sqrt(((qn[0] * qn[0] + qn[1] * qn[1]) + qn[2] * qn[2]) + qn[3] * qn[3])
    return [v / nrm for v in qn], [p[i] + dp[i] for i in range(3)]


def cholesky_solve(A, b):
    """LL^T of the 6 x 6 A (list of 36) solving A x = b in malio_loop.cu's order; None on a pivot <= 0."""
    L = [0.0] * 36
    for j in range(6):
        s = A[6 * j + j]
        for k in range(j):
            s = s - L[6 * j + k] * L[6 * j + k]
        if not s > 0.0:
            return None
        d = math.sqrt(s)
        L[6 * j + j] = d
        for i in range(j + 1, 6):
            t = A[6 * i + j]
            for k in range(j):
                t = t - L[6 * i + k] * L[6 * j + k]
            L[6 * i + j] = t / d
    y = [0.0] * 6
    for i in range(6):
        t = b[i]
        for k in range(i):
            t = t - L[6 * i + k] * y[k]
        y[i] = t / L[6 * i + i]
    x = [0.0] * 6
    for i in range(5, -1, -1):
        t = y[i]
        for k in range(i + 1, 6):
            t = t - L[6 * k + i] * x[k]
        x[i] = t / L[6 * i + i]
    return x


def full6(ut):
    A, c = [0.0] * 36, 0
    for i in range(6):
        for j in range(i, 6):
            A[6 * i + j] = A[6 * j + i] = float(ut[c])
            c += 1
    return A


# ------------------------------------------------------------------ the plane model
def jacobi3(A):
    """Cyclic Jacobi over voxels at once: A float64 (nv, 3, 3), overwritten; returns V (nv, 3, 3), columns the eigenvectors."""
    nv = A.shape[0]
    V = np.broadcast_to(np.eye(3), (nv, 3, 3)).copy()
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for _ in range(SWEEPS):
            for p, q in ((0, 1), (0, 2), (1, 2)):
                apq = A[:, p, q].copy()
                go = apq != 0.0
                theta = (A[:, q, q] - A[:, p, p]) / (2.0 * apq)
                t = 1.0 / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
                t = np.where(theta < 0.0, -t, t)
                c = 1.0 / np.sqrt(t * t + 1.0)
                s = t * c
                c, s = c[:, None], s[:, None]
                g = go[:, None]
                akp, akq = A[:, :, p].copy(), A[:, :, q].copy()
                A[:, :, p] = np.where(g, c * akp - s * akq, akp)
                A[:, :, q] = np.where(g, s * akp + c * akq, akq)
                vkp, vkq = V[:, :, p].copy(), V[:, :, q].copy()
                V[:, :, p] = np.where(g, c * vkp - s * vkq, vkp)
                V[:, :, q] = np.where(g, s * vkp + c * vkq, vkq)
                apk, aqk = A[:, p, :].copy(), A[:, q, :].copy()
                A[:, p, :] = np.where(g, c * apk - s * aqk, apk)
                A[:, q, :] = np.where(g, s * apk + c * aqk, aqk)
    return V


def pack(k):
    """int64 (n, 3) keys in range -> the device's packed uint64 key (its order does not enter any result)."""
    o = np.int64(KEY_RANGE)
    return ((k[:, 0] + o).astype(np.uint64) << np.uint64(42)) | ((k[:, 1] + o).astype(np.uint64) << np.uint64(21)) | (k[:, 2] + o).astype(np.uint64)


def in_range(k):
    return np.all((k >= -KEY_RANGE) & (k < KEY_RANGE), axis=-1)


class Model:
    """The plane voxels of target rows (float32 (n, >= 3)) at one leaf: keys (sorted uint64), mu, normal, plus every voxel's
    lambda (nv, 3) for the tests.  ValueError for a key out of range (the device's MALIO_ERR_CAPACITY)."""

    def __init__(self, rows, leaf, min_points, planarity):
        x = np.asarray(rows, np.float32)[:, :3].astype(np.float64)
        leaf = float(np.float32(leaf))
        fin = np.all(np.isfinite(x), axis=1)
        x = x[fin]
        with np.errstate(invalid="ignore"):
            k = np.floor(x / leaf)
        if not np.all(in_range(k)):
            raise ValueError("a target key lies outside [-2^20, 2^20)")
        key = pack(k.astype(np.int64))
        order = np.argsort(key, kind="stable")
        uk, start, cnt = np.unique(key[order], return_index=True, return_counts=True)
        xs = x[order]
        nv = uk.shape[0]
        s = np.zeros((nv, 3))
        for r in range(int(cnt.max()) if nv else 0):
            m = cnt > r
            s[m] = s[m] + xs[start[m] + r]
        dn = cnt.astype(np.float64)[:, None]
        mu = s / dn
        c = np.zeros((nv, 6))
        for r in range(int(cnt.max()) if nv else 0):
            m = cnt > r
            d = xs[start[m] + r] - mu[m]
            c[m] = c[m] + np.stack([d[:, 0] * d[:, 0], d[:, 0] * d[:, 1], d[:, 0] * d[:, 2], d[:, 1] * d[:, 1], d[:, 1] * d[:, 2],
                                    d[:, 2] * d[:, 2]], axis=1)
        c = c / dn
        A = np.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], axis=1).reshape(nv, 3, 3).copy()
        V = jacobi3(A)
        lam = np.stack([A[:, 0, 0], A[:, 1, 1], A[:, 2, 2]], axis=1)
        order3 = np.argsort(lam, axis=1, kind="stable")   # (value, index)
        l0 = np.take_along_axis(lam, order3[:, :1], 1)[:, 0]
        l1 = np.take_along_axis(lam, order3[:, 1:2], 1)[:, 0]
        plane = (cnt >= min_points) & (l0 <= planarity * l1)
        normal = np.take_along_axis(V, order3[:, None, :1].repeat(3, 1), 2)[:, :, 0]
        self.all_keys, self.lam, self.vectors, self.plane, self.counts = uk, lam, V, plane, cnt
        self.keys, self.mu, self.normal = uk[plane], mu[plane], normal[plane]
        self.leaf = leaf
        self.n_plane = int(plane.sum())

    def lookup(self, key):
        """Index into the plane voxels of each uint64 key, -1 for none."""
        i = np.searchsorted(self.keys, key)
        i = np.minimum(i, max(self.keys.shape[0] - 1, 0))
        ok = (self.keys.shape[0] > 0) & (self.keys[i] == key) if self.keys.shape[0] else np.zeros(key.shape, bool)
        return np.where(ok, i, -1)


OFFSETS = [(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]


def correspond(model, b, R, p):
    """(plane voxel index or -1, w, squared distance) of each source row b (float64 (n, 3)) under (R, p)."""
    w = np.stack([((R[3 * k] * b[:, 0] + R[3 * k + 1] * b[:, 1]) + R[3 * k + 2] * b[:, 2]) + p[k] for k in range(3)], axis=1)
    kb = np.floor(w / model.leaf)
    best = np.zeros(b.shape[0])
    bv = np.full(b.shape[0], -1, np.int64)
    for dx, dy, dz in OFFSETS:
        k = kb + np.array([dx, dy, dz], np.float64)
        ok = in_range(k)
        key = np.zeros(b.shape[0], np.uint64)
        key[ok] = pack(k[ok].astype(np.int64))
        v = np.where(ok, model.lookup(key), -1)
        has = v >= 0
        d = w - model.mu[np.maximum(v, 0)] if model.keys.shape[0] else np.zeros_like(w)
        e = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        take = has & ((bv < 0) | (e < best))
        best = np.where(take, e, best)
        bv = np.where(take, v, bv)
    return bv, w, best


def tree_sum(a):
    """The perfect binary tree over axis 0, padded with zeros to the smallest power of two >= len (>= 1)."""
    a = np.asarray(a, np.float64)
    n = a.shape[0]
    P = 1
    while P < n:
        P *= 2
    a = np.concatenate([a, np.zeros((P - n,) + a.shape[1:])])
    while a.shape[0] > 1:
        a = a[0::2] + a[1::2]
    return a[0]


def evaluate(model, b, q, p, gate):
    """The 29 sums of the source rows b (float32 (n, >= 3)) under (q, p)."""
    R = q_to_R(q)
    bb = np.asarray(b, np.float32)[:, :3].astype(np.float64)
    fin = np.all(np.isfinite(bb), axis=1)
    bv, w, e = correspond(model, np.where(fin[:, None], bb, 0.0), R, p)
    v = np.maximum(bv, 0)
    leaf2 = model.leaf * model.leaf
    mu, nrm = (model.mu[v], model.normal[v]) if model.keys.shape[0] else (np.zeros_like(w), np.zeros_like(w))
    d = w - mu
    r = (nrm[:, 0] * d[:, 0] + nrm[:, 1] * d[:, 1]) + nrm[:, 2] * d[:, 2]
    inl = fin & (bv >= 0) & (e <= leaf2) & (np.abs(r) <= gate)
    m = [(R[k] * nrm[:, 0] + R[3 + k] * nrm[:, 1]) + R[6 + k] * nrm[:, 2] for k in range(3)]
    J = cross3([bb[:, 0], bb[:, 1], bb[:, 2]], m) + m
    cols = [J[a_] * J[b_] for a_ in range(6) for b_ in range(a_, 6)] + [J[a_] * r for a_ in range(6)] + [r * r, np.ones_like(r)]
    rows = np.where(inl[:, None], np.stack(cols, axis=1), 0.0)
    return tree_sum(rows), int(fin.sum())


def body_state(state):
    s = capi.PassState()
    s.ext[:] = state.ext[:]
    s.rot[:] = [1.0, 0.0, 0.0, 0.0]
    return s


def match(scans, source, anchor, args, guess=None):
    """The report of malio_scan_store_match over `scans` (scan_store_ref dicts).  args: capi.MatchArgs."""
    first, count = int(args.target_first), int(args.target_count)
    target = np.concatenate([SR.register(scans[k]) for k in range(first, first + count)])
    src = SR.register(scans[source], body_state(scans[source]["state"]))
    g = scans[source]["state"] if guess is None else guess
    q, p = [float(v) for v in g.rot], [float(v) for v in g.pos]
    L = int(args.n_levels)
    rep = dict(iterations=[0] * L, converged=True, target_points=int(target.shape[0]), target_voxels=[0] * L)
    model = None
    for l in range(L):
        model = Model(target, args.leaf[l], args.min_points, args.planarity)
        rep["target_voxels"][l] = model.n_plane
        gate = float(np.float32(args.gate[l]))
        done = False
        for it in range(int(args.max_iter)):
            sums, _ = evaluate(model, src, q, p, gate)
            delta = None if sums[28] < 6.0 else cholesky_solve(full6(sums[:21]), [-float(v) for v in sums[21:27]])
            if delta is None:
                break
            q, p = right_update(q, p, delta)
            rep["iterations"][l] = it + 1
            done = all(abs(delta[i]) < (args.eps_rot if i < 3 else args.eps_pos) for i in range(6))
            if done:
                break
        rep["converged"] = done   # the finest level's
    sums, n_fin = evaluate(model, src, q, p, float(np.float32(args.gate[L - 1])))
    s2 = args.sigma * args.sigma
    info = np.array([v / s2 for v in full6(sums[:21])]).reshape(6, 6)
    ninl = float(sums[28])
    sa = scans[anchor]["state"]
    qa, pa = [float(v) for v in sa.rot], [float(v) for v in sa.pos]
    rep.update(rot=np.array(q), pos=np.array(p), info=info, n_inliers=int(ninl), n_points=n_fin,
               rms=math.sqrt(float(sums[27]) / ninl) if ninl > 0 else 0.0, fitness=ninl / n_fin if n_fin else 0.0,
               eig_min=float(np.linalg.eigvalsh(info)[0]),
               rel_rot=np.array(q_mul([qa[0], -qa[1], -qa[2], -qa[3]], q)),
               rel_pos=np.array(q_rot_conj(qa, [p[i] - pa[i] for i in range(3)])))
    return rep
