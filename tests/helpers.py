"""Shared helpers for the test-suite (test infrastructure; may use oracle/)."""
import numpy as np

import pyoracle as po
from malio_b200 import capi, synth, plugin


def snapshot_for(case, churn=False, seed=7):
    """Map snapshot of the case.  With the real reference available: ikd-Tree Build (+ optional scripted churn:
    2% Add_Points with down-sampling, one Delete_Point_Boxes) flattened through malio_flatten.hpp.
    Otherwise the product's static builder.  Returns (MapSnapshot, RefTree | None)."""
    if po.ref_available():
        tree = po.RefTree(box_length=0.5)
        tree.build(case.map_xyz, case.map_normal_y)
        if churn:
            rng = np.random.default_rng(seed)
            M = case.map_xyz.shape[0]
            k = max(M // 50, 10)
            add = case.map_xyz[rng.integers(0, M, k)] + rng.normal(0, 0.3, (k, 3)).astype(np.float32)
            ny = rng.uniform(0.0005, 0.01, k).astype(np.float32)
            tree.add_points(add, ny, downsample=True)
            add2 = case.map_xyz[rng.integers(0, M, k // 4)] + rng.normal(0, 0.2, (k // 4, 3)).astype(np.float32)
            tree.add_points(add2, None, downsample=False)
            c = case.map_xyz[rng.integers(0, M)]
            tree.delete_boxes([[c[0] - 6, c[1] - 6, c[2] - 3, c[0] + 6, c[1] + 6, c[2] + 3]])
            tree.wait_rebuild()
        nodes, cov, ids, depth, live = tree.snapshot()
        return plugin.MapSnapshot(nodes, cov, ids, depth), tree
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    return snap, None


def make_oracle(case, snap):
    orc = po.Oracle(case.params)
    orc.set_map_snapshot(snap.nodes, snap.node_cov)
    orc.set_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    return orc


def make_model(case, snap, sort_queries=True, device=0):
    m = plugin.MeasurementModel(case.n_lidar, device=device, sort_queries=sort_queries, params=case.params)
    m.upload_map(snap)
    m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    return m


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


# ---- N2 references independent of quat_ops.h: generic matrix exp / log (scipy), scipy rotations, plain numpy, float64
def spline_pose_ref(ctrl_t, ctrl_T, ts):
    """BsplineSE3::get_pose (BsplineSE3.cpp:84-118) at many timestamps with scipy's logm / expm.  The bounding control
    points are i1 = the last one at or before ts and i1 - 1, i1 + 1, i1 + 2, all inside the list.  Returns
    (ok[n], P[n,4,4]); P is the identity where ok is False."""
    from scipy.linalg import expm, logm
    ct = np.asarray(ctrl_t, np.float64)
    T = np.asarray(ctrl_T, np.float64).reshape(-1, 4, 4)
    ts = np.atleast_1d(np.asarray(ts, np.float64))
    i1 = np.searchsorted(ct, ts, side="right") - 1
    ok = (i1 >= 1) & (i1 + 2 <= ct.shape[0] - 1)
    P = np.tile(np.eye(4), (ts.shape[0], 1, 1))
    if not ok.any():
        return ok, P
    i1, t = i1[ok], ts[ok]
    logs = {int(k): np.real(logm(np.linalg.inv(T[k]) @ T[k + 1])) for k in np.unique(np.concatenate([i1 - 1, i1, i1 + 1]))}
    u = (t - ct[i1]) / (ct[i1 + 1] - ct[i1])
    b = [(5 + 3 * u - 3 * u * u + u ** 3) / 6, (1 + 3 * u + 3 * u * u - 2 * u ** 3) / 6, u ** 3 / 6]
    M = T[i1 - 1]
    for j in range(3):
        L = np.stack([logs[int(k)] for k in i1 - 1 + j])
        M = M @ expm(b[j][:, None, None] * L)
    P[ok] = M
    return ok, P


def walk_ref(t, imu_cov_t, cov_pointer):
    """The covariance-list walk of IMU_Processing.hpp:476-486 (at most one pop per point, last point first) as the min-plus
    scan pops_s = s + min(1, min_{j<=s}(need_j - j)), need = entries k <= cov_pointer with a time above the point's.
    Returns (idx[n] for points 1.., n_pops, pop_point)."""
    n = t.shape[0]
    top = np.asarray(imu_cov_t, np.float64)[: cov_pointer + 1]
    need = np.count_nonzero(top[None, :] > t[:, None], axis=1) if top.size else np.zeros(n, np.int64)
    s = np.arange(n - 1)
    v = need[::-1][: n - 1] - s
    pops = s + np.minimum(1, np.minimum.accumulate(v)) if n > 1 else np.zeros(0, np.int64)
    idx = np.full(n, capi.IDX_UNTOUCHED, np.int64)
    idx[n - 1 - s] = pops - 1
    first = np.flatnonzero(np.diff(np.concatenate([[0], pops])) > 0)
    n_pops = int(pops[-1]) if n > 1 else 0
    return idx, n_pops, (n - 1 - first)[: len(top)]


def undistort_ref(c, lt):
    """UndistortPcl's point loop (IMU_Processing.hpp:468-508) for a synth.undistort_case dict: spline poses from
    spline_pose_ref, the compensation of :492 with scipy rotations in float64, the walk from walk_ref.  lt = (q wxyz, p),
    the IMU pose at the scan end.  Point 0 is never touched."""
    from scipy.spatial.transform import Rotation
    pts = c["pts"]
    n = pts.shape[0]
    t = pts["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
    ok, P = spline_pose_ref(c["ctrl_t"], c["ctrl_T"], t)
    ok[:1] = False
    wxyz = lambda q: Rotation.from_quat(np.asarray(q, np.float64)[[1, 2, 3, 0]])
    Re, et = wxyz(c["extrinsic"][0]), np.asarray(c["extrinsic"][1], np.float64)
    Rl, lt_t = wxyz(lt[0]), np.asarray(lt[1], np.float64)
    xyz64 = pts["xyz"].astype(np.float64)
    out = pts["xyz"].copy()
    if ok.any():
        Rp = Rotation.from_matrix(P[ok, :3, :3])
        a = Re.apply(xyz64[ok]) + et
        b = Rp.apply(a) + (P[ok, :3, 3] - lt_t)
        out[ok] = Re.inv().apply(Rl.inv().apply(b) - et).astype(np.float32)
    idx, n_pops, pop_point = walk_ref(t, c["imu_cov_t"], c["cov_pointer"])
    idx[~ok] = capi.IDX_UNTOUCHED
    return dict(ok=ok, P=P, xyz=out, idx=idx, n_pops=n_pops, pop_point=pop_point)


def quat_close(q, R, tol):
    """q (w,x,y,z) is the rotation R up to sign, elementwise within tol (also for many q / R at once)."""
    from scipy.spatial.transform import Rotation
    ref = Rotation.from_matrix(R).as_quat()[..., [3, 0, 1, 2]]
    d = np.minimum(np.abs(q - ref).max(axis=-1), np.abs(q + ref).max(axis=-1))
    return bool((d <= tol).all()), float(d.max())


def ulp_diff(a, b):
    """|a - b| in units of the float32 spacing at b (elementwise max over the arrays)."""
    d = np.abs(a.astype(np.float64) - b.astype(np.float64))
    return float((d / np.spacing(np.abs(b).astype(np.float32)).astype(np.float64)).max()) if d.size else 0.0
