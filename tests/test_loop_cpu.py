"""CPU tests of loop closure over the scan store (no GPU):
  - tests/loop_ref.py on its own: Jacobi against numpy.linalg.eigh, the correspondence against a brute-force search over the
    plane voxels of the 27, the tree sum against math.fsum, a zero-noise box room whose offset guess is recovered to 1e-9;
  - malio_pose_graph_optimize through the library: random graphs against a dense numpy Gauss-Newton, a corrupted odometry edge
    fixed by an exact loop edge, no loops gives odo byte for byte, node 0 unchanged, a rank-3 loop information, every refusal,
    and n = 20 000 with 256 loops;
  - the C-ABI: struct layouts and signatures against the compiled header, NULL arguments."""
import ctypes as C
import math
import os
import re
import subprocess
import time

import numpy as np
import pytest

import loop_ref as LR
from malio_b200 import capi, plugin

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ the restatement on its own
def test_jacobi_agrees_with_eigh():
    rng = np.random.default_rng(0)
    M = rng.normal(size=(500, 3, 3))
    A = M @ M.transpose(0, 2, 1)
    A[:50, 2, :] = 0.0
    A[:50, :, 2] = 0.0                      # rank-deficient
    A[50:60] = np.diag([1.0, 2.0, 3.0])     # already diagonal: every pair skipped
    B = A.copy()
    V = LR.jacobi3(B)
    lam = np.stack([B[:, 0, 0], B[:, 1, 1], B[:, 2, 2]], axis=1)
    want = np.linalg.eigvalsh(A)
    np.testing.assert_allclose(np.sort(lam, axis=1), want, atol=1e-12 * np.abs(want).max())
    for i in range(A.shape[0]):
        np.testing.assert_allclose(A[i] @ V[i], V[i] * lam[i], atol=1e-10 * max(1.0, np.abs(lam[i]).max()))
        np.testing.assert_allclose(V[i].T @ V[i], np.eye(3), atol=1e-12)


def _planes(rng, n):
    """Points on a few tilted planes of a 12 m cube, float32 (n, 3)."""
    out = []
    for _ in range(6):
        nrm = rng.normal(size=3)
        nrm /= np.linalg.norm(nrm)
        c = rng.uniform(-5, 5, 3)
        u = np.cross(nrm, [1.0, 0.0, 0.0] if abs(nrm[0]) < 0.9 else [0.0, 1.0, 0.0])
        u /= np.linalg.norm(u)
        v = np.cross(nrm, u)
        a, b = rng.uniform(-4, 4, (2, n // 6, 1))
        out.append(c + a * u + b * v + rng.normal(scale=0.01, size=(n // 6, 1)) * nrm)
    return np.concatenate(out).astype(F)


def test_correspondence_is_the_brute_force_nearest_plane_voxel():
    rng = np.random.default_rng(1)
    tgt = _planes(rng, 6000)
    model = LR.Model(tgt, 1.0, 5, 0.2)
    assert model.n_plane > 20
    b = (tgt[rng.integers(0, tgt.shape[0], 800)] + rng.normal(scale=0.4, size=(800, 3))).astype(np.float64)
    q = np.array([0.999, 0.02, -0.03, 0.01])
    q /= np.linalg.norm(q)
    R, p = LR.q_to_R(q), [0.2, -0.1, 0.3]
    bv, w, e = LR.correspond(model, b, R, p)
    kb = np.floor(w / model.leaf)
    vk = np.stack([(model.keys >> np.uint64(s)) & np.uint64((1 << 21) - 1) for s in (42, 21, 0)], 1).astype(np.int64) - (1 << 20)
    for i in range(b.shape[0]):
        near = np.all(np.abs(vk - kb[i]) <= 1, axis=1)
        if not near.any():
            assert bv[i] == -1
            continue
        idx = np.nonzero(near)[0]
        d = w[i] - model.mu[idx]
        dist = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        best = dist.min()
        assert e[i] == best
        # ties go to the first offset in (dz, dy, dx) order
        cand = idx[dist == best]
        off = [tuple((vk[c] - kb[i]).astype(int)) for c in cand]
        first = min(range(len(cand)), key=lambda t: (off[t][2], off[t][1], off[t][0]))
        assert bv[i] == cand[first]


def test_tree_sum_against_fsum():
    rng = np.random.default_rng(2)
    for n in (1, 2, 3, 127, 128, 129, 1000, 4097):
        a = rng.normal(size=(n, 3)) * 10.0 ** rng.integers(-3, 3, (n, 1))
        got = LR.tree_sum(a)
        for c in range(3):
            assert abs(got[c] - math.fsum(a[:, c])) <= 1e-12 * max(1.0, np.abs(a[:, c]).sum())
    x = np.array([[-0.0], [-0.0], [-0.0]])
    assert math.copysign(1.0, LR.tree_sum(x)[0]) == 1.0   # padded to 4 with +0.0


def _room(rng, n_side=40):
    """A box room with axis-aligned walls at exactly representable coordinates: floor z = 0, ceiling z = 3.5, walls x = +-5.5
    and y = +-7.5, each surface at least a voxel away from the others (a voxel holds one plane); points on a jittered grid
    within their plane (float32 (n, 3))."""
    g = np.linspace(-4.4, 4.4, n_side)
    a, b = [v.ravel() for v in np.meshgrid(g, g)]
    A, H = [v.ravel() for v in np.meshgrid(g, np.linspace(0.6, 2.9, n_side // 2))]
    j = lambda n: rng.uniform(-0.01, 0.01, n)
    pts = [np.stack([a + j(a.size), b * 1.45 + j(a.size), np.full_like(a, z)], 1) for z in (0.0, 3.5)]
    pts += [np.stack([np.full_like(A, x), A * 1.45 + j(A.size), H + j(A.size)], 1) for x in (-5.5, 5.5)]
    pts += [np.stack([A + j(A.size), np.full_like(A, y), H + j(A.size)], 1) for y in (-7.5, 7.5)]
    return np.concatenate(pts).astype(F)


def _identity_scan(xyz):
    s = capi.PassState()
    s.rot[:] = [1.0, 0.0, 0.0, 0.0]
    for l in range(capi.MAX_LIDAR):
        s.ext[l].q[:] = [1.0, 0.0, 0.0, 0.0]
    return dict(state=s, temporal_comp=np.zeros(capi.MAX_LIDAR - 1, capi.RIGID), slot_tag=np.zeros(1, F), n_points=[xyz.shape[0]],
                xyz=xyz)


def test_zero_noise_room_recovers_a_known_offset():
    rng = np.random.default_rng(3)
    xyz = _room(rng)
    scans = [_identity_scan(xyz), _identity_scan(xyz)]
    a = plugin.match_args(0, 1, leaf=(2.0, 1.0), gate=(1.0, 0.5), max_iter=30, eps_rot=1e-12, eps_pos=1e-12, min_points=5,
                          planarity=0.05, sigma=0.05)
    g = capi.PassState()
    ang = 0.03
    g.rot[:] = [math.cos(ang / 2), 0.0, 0.0, math.sin(ang / 2)]
    g.pos[:] = [0.25, -0.2, 0.1]
    rep = LR.match(scans, 1, 0, a, guess=g)
    assert rep["n_inliers"] > 0.9 * rep["n_points"]
    assert np.abs(rep["pos"]).max() < 1e-9
    assert np.abs(rep["rot"][1:]).max() < 1e-9 and abs(rep["rot"][0] - 1.0) < 1e-9
    assert rep["rms"] < 1e-9 and rep["eig_min"] > 0


# ------------------------------------------------------------------ the pose graph through the library
def _log_se3(T):
    R, t = T[:3, :3], T[:3, 3]
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    c = max(-1.0, min(1.0, (tr - 1.0) / 2.0))
    th = math.acos(c)
    if th < 1e-7:
        w = 0.5 * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    else:
        w = th / (2 * math.sin(th)) * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    n = np.linalg.norm(w)
    if n < 1e-10:
        return np.concatenate([w, t])
    a = w / n
    Wm = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.concatenate([w, t - 0.5 * n * (Wm @ t) + (1 - n / (2 * math.tan(0.5 * n))) * (Wm @ Wm @ t)])


def _T(q, p):
    T = np.eye(4)
    T[:3, :3] = np.array(LR.q_to_R(q)).reshape(3, 3)
    T[:3, 3] = p
    return T


def _inv(T):
    Ti = np.eye(4)
    Ti[:3, :3] = T[:3, :3].T
    Ti[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return Ti


def _ad(T):
    R, t = T[:3, :3], T[:3, 3]
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    A = np.zeros((6, 6))
    A[:3, :3], A[3:, :3], A[3:, 3:] = R, tx @ R, R
    return A


def dense_gn(qs, ps, loops, sr, sp, max_iter=50, eps_rot=1e-11, eps_pos=1e-10):
    """The contract of malio_pose_graph_optimize with a dense numpy solve."""
    n = len(qs)
    qs, ps = [list(q) for q in qs], [list(p) for p in ps]
    Wo = np.diag([sr ** -2] * 3 + [sp ** -2] * 3)
    edges = [(k, k + 1, _inv(_inv(_T(qs[k], ps[k])) @ _T(qs[k + 1], ps[k + 1])), Wo) for k in range(n - 1)]
    edges += [(a, b, _inv(_T(q, p)), W) for a, b, q, p, W in loops]

    def chi2(qs, ps):
        return sum(float(e @ W @ e) for a, b, Zi, W in edges for e in [_log_se3(Zi @ _inv(_T(qs[a], ps[a])) @ _T(qs[b], ps[b]))])

    chi = chi2(qs, ps)
    for _ in range(max_iter):
        H, g = np.zeros((6 * n, 6 * n)), np.zeros(6 * n)
        for a, b, Zi, W in edges:
            Ta, Tb = _T(qs[a], ps[a]), _T(qs[b], ps[b])
            e = _log_se3(Zi @ _inv(Ta) @ Tb)
            Ja, Jb = -_ad(_inv(Tb) @ Ta), np.eye(6)
            for i, Ji in ((a, Ja), (b, Jb)):
                g[6 * i:6 * i + 6] += Ji.T @ W @ e
                for j, Jj in ((a, Ja), (b, Jb)):
                    H[6 * i:6 * i + 6, 6 * j:6 * j + 6] += Ji.T @ W @ Jj
        d = np.linalg.solve(H[6:, 6:], -g[6:])
        small = all(abs(d[i]) < (eps_rot if i % 6 < 3 else eps_pos) for i in range(d.size))
        for _h in range(21):
            nq, np_ = [qs[0]], [ps[0]]
            for k in range(1, n):
                q, p = LR.right_update(qs[k], ps[k], [float(v) for v in d[6 * k - 6:6 * k]])
                nq.append(q)
                np_.append(p)
            cn = chi2(nq, np_)
            if cn <= chi:
                break
            d = d * 0.5
        else:
            break
        qs, ps, chi = nq, np_, cn
        if small:
            break
    return np.array(qs), np.array(ps)


def _chain(rng, n, step=1.0):
    qs, ps = [np.array([1.0, 0, 0, 0])], [np.zeros(3)]
    for _ in range(n - 1):
        dq = np.array([1.0, *rng.normal(scale=0.05, size=3)])
        dq /= np.linalg.norm(dq)
        q = np.array(LR.q_mul(qs[-1], dq))
        qs.append(q / np.linalg.norm(q))
        ps.append(ps[-1] + np.array(LR.q_rot(qs[-2], [step, *rng.normal(scale=0.1, size=2)])))
    return qs, ps


def _states(qs, ps):
    out = []
    for q, p in zip(qs, ps):
        s = capi.PassState()
        s.rot[:], s.pos[:] = [float(v) for v in q], [float(v) for v in p]
        s.ext[1].t[:] = [0.5, 0.25, 0.125]
        out.append(s)
    return out


def _edge(a, b, q, p, W):
    e = capi.PoseEdge()
    e.a, e.b = a, b
    e.rot[:], e.pos[:], e.info[:] = [float(v) for v in q], [float(v) for v in p], [float(v) for v in np.asarray(W).reshape(36)]
    return e


def _rel(qa, pa, qb, pb):
    return LR.q_mul([qa[0], -qa[1], -qa[2], -qa[3]], qb), LR.q_rot_conj(qa, [pb[i] - pa[i] for i in range(3)])


def _spd(rng, scale=100.0):
    M = rng.normal(size=(6, 6))
    return M @ M.T + scale * np.eye(6)


@pytest.mark.parametrize("seed", range(6))
def test_random_graphs_agree_with_a_dense_gauss_newton(seed):
    rng = np.random.default_rng(100 + seed)
    n, m = int(rng.integers(5, 61)), int(rng.integers(1, 9))
    qs, ps = _chain(rng, n)
    loops = []
    for _ in range(m):
        a, b = sorted(rng.choice(n, 2, replace=False))
        q, p = _rel(qs[a], ps[a], qs[b], ps[b])
        dq = np.array([1.0, *rng.normal(scale=0.01, size=3)])
        q = np.array(LR.q_mul(q, dq / np.linalg.norm(dq)))
        loops.append((int(a), int(b), q / np.linalg.norm(q), np.array(p) + rng.normal(scale=0.1, size=3), _spd(rng)))
    out, chi, rep = plugin.pose_graph_optimize(_states(qs, ps), [_edge(*l) for l in loops], sigma_rot=0.02, sigma_pos=0.2,
                                               max_iter=50, eps_rot=1e-11, eps_pos=1e-10)
    wq, wp = dense_gn(qs, ps, loops, 0.02, 0.2)
    gq, gp = np.array([list(s.rot) for s in out]), np.array([list(s.pos) for s in out])
    assert rep["converged"]
    np.testing.assert_allclose(gp, wp, atol=1e-9)
    np.testing.assert_allclose(gq * np.sign(gq[:, :1]), wq * np.sign(wq[:, :1]), atol=1e-9)
    assert rep["chi2_loop"] <= rep["chi2_loop_before"] and chi.shape == (m,)


def test_a_corrupted_odometry_edge_is_fixed_by_an_exact_loop():
    rng = np.random.default_rng(7)
    qs, ps = _chain(rng, 30)
    q_true, p_true = [q.copy() for q in qs], [p.copy() for p in ps]
    bad_q, bad_p = [q.copy() for q in qs], [p.copy() for p in ps]
    kick = np.array([math.cos(0.05), 0.0, 0.0, math.sin(0.05)])
    for k in range(15, 30):   # edge 14 -> 15 corrupted: everything after it moves rigidly about node 15
        bad_q[k] = np.array(LR.q_mul(kick, q_true[k]))
        bad_p[k] = np.array(LR.q_rot(kick, list(p_true[k] - p_true[15]))) + p_true[15] + np.array([0.7, -0.4, 0.2])
    # the exact edge across the break outweighs the corrupted odometry: the truth is the least-squares optimum (a loop
    # spanning more of the chain would spread the corrupted edge's error over the odometry edges it spans)
    q, p = _rel(q_true[14], p_true[14], q_true[15], p_true[15])
    out, _, rep = plugin.pose_graph_optimize(_states(bad_q, bad_p), [_edge(14, 15, q, p, np.eye(6) * 1e10)], sigma_rot=0.01,
                                             sigma_pos=0.1)
    gp, gq = np.array([list(s.pos) for s in out]), np.array([list(s.rot) for s in out])
    assert rep["converged"] and rep["chi2_loop"] < 1e-6 * rep["chi2_loop_before"]
    assert np.abs(gp - np.array(p_true)).max() < 1e-5, np.abs(gp - np.array(p_true)).max()
    assert np.abs(gq - np.array(q_true)).max() < 1e-6


def test_no_loops_is_odo_byte_for_byte_and_node_zero_stays():
    rng = np.random.default_rng(8)
    qs, ps = _chain(rng, 40)
    st = _states(qs, ps)
    out, chi, rep = plugin.pose_graph_optimize(st, [])
    assert b"".join(bytes(s) for s in out) == b"".join(bytes(s) for s in st)
    assert rep["iterations"] == 0 and chi.shape == (0,)
    loops = [_edge(0, 39, *_rel(qs[0], ps[0], qs[39], ps[39] + 1.0), np.eye(6) * 10)]
    out, _, _ = plugin.pose_graph_optimize(st, loops)
    assert bytes(out[0]) == bytes(st[0])
    assert bytes(out[5].ext[1]) == bytes(st[5].ext[1])


def test_rank_three_loop_information_gives_a_finite_result():
    rng = np.random.default_rng(9)
    qs, ps = _chain(rng, 25)
    W = np.zeros((6, 6))
    W[3:, 3:] = np.diag([1e4, 1e4, 0.0])
    W[0, 0] = 1e4   # rank 3: one rotation, two translations
    loops = [_edge(2, 24, *_rel(qs[2], ps[2], qs[24], np.array(ps[24]) + [0.5, 0.5, 0.5]), W)]
    out, chi, rep = plugin.pose_graph_optimize(_states(qs, ps), loops)
    assert np.all(np.isfinite([v for s in out for v in list(s.rot) + list(s.pos)])) and np.isfinite(chi).all()
    assert rep["chi2_loop"] < rep["chi2_loop_before"]


def test_pose_graph_refusals():
    lib = capi.load()
    rng = np.random.default_rng(10)
    qs, ps = _chain(rng, 5)
    odo = (capi.PassState * 5)(*_states(qs, ps))
    out = (capi.PassState * 5)()
    rep = capi.PoseGraphReport()
    good = capi.PoseGraphArgs(0.01, 0.1, 10, 1e-9, 1e-9)
    e = _edge(0, 4, [1.0, 0, 0, 0], [0.0, 0, 0], np.eye(6))
    call = lambda odo_=odo, n=5, loops=None, m=0, a=good, out_=out, r=rep: lib.malio_pose_graph_optimize(
        odo_, n, loops, m, None if a is None else C.byref(a), out_, None, None if r is None else C.byref(r))
    one = (capi.PoseEdge * 1)(e)
    assert call(loops=one, m=1) == capi.OK
    for bad in (dict(odo_=None), dict(n=0), dict(a=None), dict(out_=None), dict(r=None), dict(loops=None, m=1),
                dict(loops=one, m=capi.POSE_GRAPH_MAX_LOOPS + 1)):
        assert call(**bad) == capi.ERR_INVALID_ARG, bad
    for f, v in (("sigma_rot", 0.0), ("sigma_pos", -1.0), ("eps_rot", 0.0), ("eps_pos", float("nan")), ("max_iter", 0)):
        a = capi.PoseGraphArgs(0.01, 0.1, 10, 1e-9, 1e-9)
        setattr(a, f, v)
        assert call(loops=one, m=1, a=a) == capi.ERR_INVALID_ARG, f
    for mod in (dict(a=5), dict(b=5), dict(a=2, b=2)):
        bad = _edge(0, 4, [1.0, 0, 0, 0], [0.0, 0, 0], np.eye(6))
        for k, v in mod.items():
            setattr(bad, k, v)
        assert call(loops=(capi.PoseEdge * 1)(bad), m=1) == capi.ERR_INVALID_ARG, mod
    W = np.eye(6)
    W[0, 1] = 0.5
    assert call(loops=(capi.PoseEdge * 1)(_edge(0, 4, [1.0, 0, 0, 0], [0.0, 0, 0], W)), m=1) == capi.ERR_INVALID_ARG
    W = np.eye(6)
    W[2, 2] = np.inf
    assert call(loops=(capi.PoseEdge * 1)(_edge(0, 4, [1.0, 0, 0, 0], [0.0, 0, 0], W)), m=1) == capi.ERR_INVALID_ARG


def test_twenty_thousand_nodes_and_256_loops():
    rng = np.random.default_rng(11)
    n, m = 20000, 256
    qs, ps = _chain(rng, n, step=0.5)
    loops = []
    for i in range(m):
        a = int(rng.integers(0, n - 200))
        b = int(rng.integers(a + 100, n))
        q, p = _rel(qs[a], ps[a], qs[b], ps[b])
        loops.append(_edge(a, b, q, np.array(p) + rng.normal(scale=0.05, size=3), _spd(rng, 1e3)))
    t0 = time.perf_counter()
    out, chi, rep = plugin.pose_graph_optimize(_states(qs, ps), loops, max_iter=10, eps_rot=1e-8, eps_pos=1e-7)
    wall = time.perf_counter() - t0
    print(f"pose graph n={n} m={m}: {rep['iterations']} iterations, {rep['ms']:.0f} ms host (wall {wall:.1f} s), "
          f"loop chi2 {rep['chi2_loop_before']:.3g} -> {rep['chi2_loop']:.3g}")
    assert rep["iterations"] >= 1 and rep["chi2_loop"] < rep["chi2_loop_before"]
    assert np.all(np.isfinite([v for s in out[::500] for v in list(s.pos)]))


# ------------------------------------------------------------------ the C-ABI surface
NEW = ["malio_scan_store_match", "malio_pose_graph_optimize"]


def _prototype(hdr, name):
    m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", hdr)
    assert m, name
    return [" ".join(a.split()) for a in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",")]


def _ctype_of(arg):
    if "*" in arg:
        return C.c_void_p
    return {"uint64_t": C.c_uint64, "uint32_t": C.c_uint32, "int": C.c_int}[arg.rsplit(" ", 1)[0]]


def test_signatures_and_constants_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    lib = capi.load()
    for name in NEW:
        assert name in capi.EXPORTS, name
        assert list(getattr(lib, name).argtypes) == [_ctype_of(a) for a in _prototype(hdr, name)], name
    for macro, val in (("MALIO_MATCH_MAX_LEVELS", capi.MATCH_MAX_LEVELS), ("MALIO_MATCH_JACOBI_SWEEPS", capi.MATCH_JACOBI_SWEEPS),
                       ("MALIO_POSE_GRAPH_MAX_LOOPS", capi.POSE_GRAPH_MAX_LOOPS)):
        assert int(re.search(r"#define " + macro + r" (\d+)", hdr).group(1)) == val, macro
    assert "#define MALIO_MATCH_KEY_RANGE (1 << 20)" in hdr and capi.MATCH_KEY_RANGE == 1 << 20
    assert "#define MALIO_MATCH_MAX_BYTES (16ull << 30)" in hdr and capi.MATCH_MAX_BYTES == 16 << 30


STRUCTS = {
    "malio_match_args": (capi.MatchArgs, ["target_first", "target_count", "n_levels", "leaf", "gate", "max_iter", "eps_rot", "eps_pos",
                                          "min_points", "planarity", "sigma"]),
    "malio_match_report": (capi.MatchReport, ["rot", "pos", "rel_rot", "rel_pos", "info", "rms", "fitness", "eig_min", "n_points",
                                              "n_inliers", "iterations", "converged", "target_points", "target_voxels", "device_bytes"]),
    "malio_pose_edge": (capi.PoseEdge, ["a", "b", "rot", "pos", "info"]),
    "malio_pose_graph_args": (capi.PoseGraphArgs, ["sigma_rot", "sigma_pos", "max_iter", "eps_rot", "eps_pos"]),
    "malio_pose_graph_report": (capi.PoseGraphReport, ["iterations", "converged", "chi2_odo", "chi2_loop", "chi2_loop_before", "ms"]),
}


def test_struct_layouts_match_the_compiled_header(tmp_path):
    lines = []
    for name, (_, fields) in STRUCTS.items():
        lines.append(f'printf("%zu", sizeof({name}));')
        for f in fields:
            lines.append(f'printf(" %zu", offsetof({name}, {f}));')
        lines.append('printf("\\n");')
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "malio_b200.h"\nint main(void) {\n' + "\n".join(lines)
                   + "\nreturn 0; }\n")
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-x", "c", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    for line, (name, (S, fields)) in zip(got, STRUCTS.items()):
        want = [C.sizeof(S)] + [getattr(S, f).offset for f in fields]
        assert [int(v) for v in line.split()] == want, name


def test_null_arguments_are_refused():
    lib = capi.load()
    a, rep = capi.MatchArgs(), capi.MatchReport()
    assert lib.malio_scan_store_match(None, 0, 0, None, C.byref(a), C.byref(rep)) == capi.ERR_INVALID_ARG
    assert lib.malio_pose_graph_optimize(None, 0, None, 0, None, None, None, None) == capi.ERR_INVALID_ARG


def test_loop_candidates_take_the_nearest_old_enough_scan():
    recs = []
    for x in (0.0, 1.0, 2.0, 3.0, 10.0, 2.1, 0.5):
        s = capi.PassState()
        s.pos[:] = [x, 0.0, 0.0]
        recs.append(s)
    assert plugin.loop_candidates(recs, radius=1.0, min_gap=3) == [(2, 5), (0, 6)]
    assert plugin.loop_candidates(recs, radius=1.0, min_gap=3, stride=2) == [(0, 6)]


def test_acceptance_does_not_depend_on_the_scan_size_or_sigma():
    rep = dict(converged=True, fitness=0.6, rms=0.03, eig_min=1.2e5, n_inliers=7000, sigma=0.05)
    assert plugin.accept_edge(rep)
    big = dict(rep, eig_min=rep["eig_min"] * 20, n_inliers=rep["n_inliers"] * 20)   # the same geometry, 20x the points
    assert plugin.constraint(big) == pytest.approx(plugin.constraint(rep)) and plugin.accept_edge(big)
    loose = dict(rep, eig_min=rep["eig_min"] / 4, sigma=0.1)                        # the same fit reported with twice the sigma
    assert plugin.constraint(loose) == pytest.approx(plugin.constraint(rep))
    corridor = dict(rep, eig_min=1.8e4 * 20, n_inliers=7916 * 20)                  # a large corridor scan clears any absolute cut
    assert not plugin.accept_edge(corridor)
    assert not plugin.accept_edge(dict(rep, converged=False)) and not plugin.accept_edge(dict(rep, n_inliers=0))
