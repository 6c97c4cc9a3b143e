"""CPU tier for the undistortion (SURVEY.md §8f N2) and the voxel index (N3) at the motions, time ties and list edges the
default synthetic scan never reaches (synth.UNDISTORT_MOTIONS / UNDISTORT_LISTS, ties=True).

Independent references: scipy's Rotation, expm and logm, and plain numpy in float64 (helpers.spline_pose_ref,
helpers.undistort_ref, helpers.walk_ref).  The product's spline code is reached through malio_bspline_get_pose, which is
host code in the library: it is the device's code compiled for the host, so it loads without a GPU.  No GPU needed."""
import hashlib

import numpy as np
import pytest
from scipy.linalg import expm, logm
from scipy.spatial.transform import Rotation

import helpers as H
import pyoracle as po
from malio_b200 import plugin, synth

REGIMES = [(m, False, "default") for m in synth.UNDISTORT_MOTIONS] + [
    ("generic", True, "default"), ("straight", True, "default"), ("stationary", True, "last_cov"),
    ("generic", True, "empty_cov"), ("heading_wrap", True, "max"), ("fast", False, "max")]


def _rid(r):
    return f"{r[0]}{'-ties' if r[1] else ''}-{r[2]}"


def _digest(c):
    h = hashlib.sha256()
    for k in sorted(c):
        for a in (c[k] if isinstance(c[k], tuple) else (c[k],)):
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def test_undistort_case_defaults_are_unchanged():
    """The regimes are opt-in: the default scans (and the ones the older tests draw) are the same bytes as before."""
    assert _digest(synth.undistort_case()) == "0b1df1ded7290bde74815e670975575f4198d69162a124acb70886693b8ce9e4"
    assert _digest(synth.undistort_case(100)) == "b43d302b3f2acba9a33787911d5c50a23b5283aaa7fb7adf19ddbea63e285e89"
    assert _digest(synth.undistort_case(300, lidar=1, imu_hz=4000.0)) == "b83f4aa8c52a24abaf084d963b1e2adeb89a38edbd2d7ca5be95398d850186b3"
    assert _digest(synth.undistort_case(37000, lidar=1, seed=61)) == "38ca47748ee99946c9d9a95b52e84a578ae16cccea106d8172490de586b72664"


def test_regimes_reach_their_branches():
    """What each regime is for, checked on its data: control-point traces <= 0 with the intended largest diagonal entry,
    pair turns on both sides of log_so3's Taylor threshold, exact time ties, and the list edges."""
    def R_of(c):
        return c["ctrl_T"].reshape(-1, 4, 4)[:, :3, :3]

    def pair_angles(c):
        R = R_of(c)
        return Rotation.from_matrix(np.swapaxes(R[:-1], 1, 2) @ R[1:]).magnitude()

    for m, i in (("heading_x", 0), ("heading_y", 1), ("heading_z", 2), ("heading_wrap", 2)):
        R = R_of(synth.undistort_case(10, motion=m))
        assert (np.trace(R, axis1=1, axis2=2) <= 0).all() and (np.argmax(np.diagonal(R, axis1=1, axis2=2), 1) == i).all(), m
    yaw = np.unwrap(Rotation.from_matrix(R_of(synth.undistort_case(10, motion="heading_wrap"))).as_euler("zyx")[:, 0])
    assert yaw.min() < np.pi < yaw.max()
    a = pair_angles(synth.undistort_case(10, motion="straight"))
    assert (a < 3.16e-4).mean() > 0.5 and (a > 3.2e-4).any() and (a < 1e-7).any()
    assert (pair_angles(synth.undistort_case(10, motion="stationary")) < 1e-10).all()
    assert 0.09 < pair_angles(synth.undistort_case(10, motion="fast")).min()
    c = synth.undistort_case(3000, ties=True)
    t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
    assert np.isin(c["ctrl_t"], t).sum() >= 8 and np.isin(c["imu_cov_t"], t).sum() >= 15
    assert (np.diff(c["imu_cov_t"]) == 0).any()
    c = synth.undistort_case(10, lists="max", ties=True)
    assert c["ctrl_t"].shape[0] == synth.MAX_CTRL and c["imu_cov_t"].shape[0] == synth.MAX_COV
    c = synth.undistort_case(10, lists="empty_cov")
    assert c["imu_cov_t"].shape[0] == 0 and c["cov_pointer"] == -1
    c = synth.undistort_case(10, lists="last_cov")
    assert c["cov_pointer"] == c["imu_cov_t"].shape[0] - 1


# ------------------------------------------------------------------ Eigen's matrix -> quaternion
def _test_rotations():
    rng = np.random.default_rng(11)
    Rs = [np.eye(3), np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, 1.0, -1.0]), np.diag([-1.0, -1.0, 1.0])]
    for v in ([2.2, 0, 0], [0, 2.7, 0], [0, 0, np.pi - 1e-3], [0, 0, -np.pi + 1e-3], [3.0, 0.3, -0.2], [0.1, -2.9, 0.4],
              [0.2, 0.1, 3.1], [1e-9, 0, 0]):
        Rs.append(Rotation.from_rotvec(v).as_matrix())
    Rs += list(Rotation.random(200, random_state=rng).as_matrix())
    return np.array(Rs)


def _eigen_branch(R):
    if np.trace(R) > 0:
        return "t>0"
    d = np.diag(R)
    i = 1 if d[1] > d[0] else 0
    return f"i={2 if d[2] > d[i] else i}"


def test_quat_from_R_oracle_and_product_against_scipy():
    """All four branches of Eigen's conversion, the exact half turns about each axis and random rotations.  The product's
    conversion is reached through the spline of six equal control poses: that spline is the pose itself."""
    Rs = _test_rotations()
    assert {_eigen_branch(R) for R in Rs} == {"t>0", "i=0", "i=1", "i=2"}
    ct = 100.0 + 0.01 * np.arange(6)
    for R in Rs:
        q = po.quat_from_R(R)
        ok, tol = H.quat_close(q, R, 1e-14)
        assert ok, (_eigen_branch(R), tol)
        assert abs(np.linalg.norm(q) - 1.0) < 1e-15
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = (1.0, -2.0, 0.5)
        ok_g, qg, pg = plugin.bspline_get_pose(ct, np.tile(T.reshape(16), (6, 1)), ct[2] + 0.004)
        assert ok_g and H.quat_close(qg, R, 1e-14)[0], _eigen_branch(R)
        assert np.abs(pg - T[:3, 3]).max() < 1e-14


# ------------------------------------------------------------------ log_se3 / exp_se3
def _hat(v):
    w, u = v[:3], v[3:]
    M = np.zeros((4, 4))
    M[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
    M[:3, 3] = u
    return M


ANGLES = (0.0, 1e-12, 1e-8, 2e-4, 3.1e-4, 3.3e-4, 1.0, 3.0, np.pi - 1e-6, np.pi)


@pytest.mark.parametrize("theta", ANGLES)
def test_log_exp_se3_against_expm_logm(theta):
    """exp_se3 against expm and log_se3 against the generator (and logm), at the branch edges of quat_ops.h: exp's
    theta < 1e-7, log_so3's Taylor threshold (~3.16e-4) and its near-pi branch (trace + 1 < 1e-10), log_se3's t < 1e-10.
    Near pi the reference takes the angle to be exactly pi, so there the bar is the distance to pi.  Above 1e-7 the
    closed forms divide 1 - cos(theta) by theta^2 and lose digits as theta shrinks: the bars grow like eps |u| / theta."""
    axis = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    for u in (np.array([0.7, -1.3, 2.1]), np.array([40.0, 3.0, -0.5])):
        v = np.concatenate([axis * theta, u])
        T = po.exp_se3(v)
        Tref = expm(_hat(v))
        um = np.abs(u).max()
        cancel = 4e-16 / theta if theta >= 1e-7 else 0.0
        assert np.abs(T - Tref).max() < (1e-13 + cancel) * um, np.abs(T - Tref).max()
        lg = po.log_se3(Tref)
        near = np.pi - theta
        bar = (1e-11 + cancel) * um if near > 1e-3 else 4 * near * (1 + um) + 1e-9
        if theta < np.pi:
            assert np.abs(lg - v).max() <= bar, (np.abs(lg - v).max(), bar)
            if 0 < theta < 3.0:
                assert np.abs(lg - _vee(np.real(logm(Tref)))).max() <= bar
        else:   # log of a half turn: either axis sign, the translation follows it
            assert min(np.abs(lg[:3] - v[:3]).max(), np.abs(lg[:3] + v[:3]).max()) < 1e-12
        # round trips
        assert np.abs(po.exp_se3(lg) - Tref).max() <= max(bar, 1e-12) * 2
        assert np.abs(po.log_se3(T) - lg).max() <= max(bar, 1e-12) * 2


def _vee(M):
    return np.array([M[2, 1], M[0, 2], M[1, 0], M[0, 3], M[1, 3], M[2, 3]])


# ------------------------------------------------------------------ spline pose and compensation, every regime
@pytest.mark.parametrize("regime", REGIMES, ids=_rid)
def test_spline_pose_and_compensation_against_scipy(regime):
    """The oracle's and the product's spline pose against scipy at every point time and at every control-point time
    (ties); the product's host code must equal the oracle bit for bit (both are restatements of the same expression
    sequence).  The oracle's compensated points against the float64 scipy restatement of :492: <= 1 float ulp, and
    the input itself (<= 1 ulp) when the vehicle stands still."""
    motion, ties, lists = regime
    c = synth.undistort_case(1500, motion=motion, ties=ties, lists=lists)
    t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
    ts = np.unique(np.concatenate([t[1:], c["ctrl_t"][-40:], c["ctrl_t"][:3]]))
    ok_ref, P = H.spline_pose_ref(c["ctrl_t"], c["ctrl_T"], ts)
    assert ok_ref.sum() > 1000
    for k, tk in enumerate(ts):
        ok, q, p = po.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], tk)
        ok2, q2, p2 = plugin.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], tk)
        assert ok == ok_ref[k] == ok2, (k, tk)
        assert np.array_equal(q, q2) and np.array_equal(p, p2), (k, tk)
        if ok:
            assert H.quat_close(q, P[k, :3, :3], 1e-9)[0] and np.abs(p - P[k, :3, 3]).max() < 1e-9, (k, tk)
    ok, q, p = po.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], c["end_time"])
    assert ok
    o = po.undistort(c["pts"], c["beg_time"], c["extrinsic"], (q, p), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
    r = H.undistort_ref(c, (q, p))
    assert np.array_equal(o["ok"] > 0, r["ok"])
    assert H.ulp_diff(o["xyz"], r["xyz"]) <= 1.0
    if motion == "stationary":
        assert H.ulp_diff(o["xyz"], c["pts"]["xyz"]) <= 1.0


def test_straight_motion_yaw_is_the_weighted_sum_of_pair_turns():
    """All turns of the straight regime share the body z axis, so they commute: the spline's heading at u in the segment
    [i1, i1+1] is yaw[i1-1] + b0 d[i1-1] + b1 d[i1] + b2 d[i1+1] with d the pair increments.  The pair turns straddle
    log_so3's Taylor threshold, whose second-order term is ~1e-12 rad here; the bar is 1e-14 rad."""
    c = synth.undistort_case(400, motion="straight", ties=True)
    ct = c["ctrl_t"]
    steps = np.array(synth.STRAIGHT_YAW_STEPS)[np.arange(ct.shape[0]) % len(synth.STRAIGHT_YAW_STEPS)]
    yaw = np.concatenate([[0.0], np.cumsum(steps[:-1])])
    R0 = synth.q_to_R(synth.q_exp([0.1, -0.05, 0.7]))
    t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
    for ts in t:
        i1 = int(np.searchsorted(ct, ts, side="right")) - 1
        u = (ts - ct[i1]) / (ct[i1 + 1] - ct[i1])
        b = ((5 + 3 * u - 3 * u * u + u ** 3) / 6, (1 + 3 * u + 3 * u * u - 2 * u ** 3) / 6, u ** 3 / 6)
        expect = yaw[i1 - 1] + b[0] * steps[i1 - 1] + b[1] * steps[i1] + b[2] * steps[i1 + 1]
        for get in (po.bspline_get_pose, plugin.bspline_get_pose):
            ok, q, _ = get(ct, c["ctrl_T"], ts)
            Rz = R0.T @ synth.q_to_R(q)
            assert ok and abs(np.arctan2(Rz[1, 0], Rz[0, 0]) - expect) < 1e-14, (ts, np.arctan2(Rz[1, 0], Rz[0, 0]) - expect)


@pytest.mark.parametrize("regime", [("generic", True, "default"), ("generic", True, "empty_cov"), ("generic", True, "last_cov"),
                                    ("generic", True, "max"), ("stationary", False, "last_cov")], ids=_rid)
@pytest.mark.parametrize("n,hz", [(600, 200.0), (300, 4000.0), (2, 200.0)])
def test_covariance_list_walk_at_list_edges(regime, n, hz):
    """The oracle's sequential walk (IMU_Processing.hpp:476-486) against the min-plus replay with time ties, duplicate
    stamps, an empty list, cov_pointer at the last entry and full-size lists."""
    motion, ties, lists = regime
    c = synth.undistort_case(n, motion=motion, ties=ties, lists=lists, imu_hz=hz if lists != "max" else 200.0)
    ok, q, p = po.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], c["end_time"])
    o = po.undistort(c["pts"], c["beg_time"], c["extrinsic"], (q, p), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
    t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
    idx, n_pops, pop_point = H.walk_ref(t, c["imu_cov_t"], c["cov_pointer"])
    touched = o["ok"] > 0
    assert np.array_equal(idx[touched], o["idx"][touched].astype(np.int64))
    assert o["n_pops"] == n_pops and np.array_equal(o["pop_point"], pop_point)
    if lists == "empty_cov":
        assert n_pops == 0 and (o["idx"][touched] == -1).all()


# ------------------------------------------------------------------ the voxel index of pcl::VoxelGrid in float
def _pcl_axis_index(f, minb):
    """static_cast<int>(std::floor(p * inverse_leaf) - static_cast<float>(min_b)) with f = the float floor."""
    return (np.float32(f) - np.float32(minb)).astype(np.int64)


def test_voxel_axis_index_reaches_dim_only_above_2_to_24():
    """The float subtraction in PCL's voxel index is exact while the axis spans at most 2^24 voxels, so the index stays in
    [0, dim); above that it can round up to dim itself (the device would count the point one cell past the grid, which
    is why malio_voxel_grid rejects such clouds).  The largest index on an axis is the one of its largest point, so
    checking f = max_b covers every point; min_b and max_b are floats' floors (representable)."""
    lim = 1 << 24
    reached = []
    for minb in (-(1 << 26), -3 * lim - 7, -lim - 1, -12345, -1, 0, 1, 7, 99991, lim - 3, lim + 2, 1 << 27):
        minb = int(np.float32(minb))
        dims = np.arange(1, lim + 1, 997, dtype=np.int64)
        dims = np.concatenate([dims, np.arange(lim - 4096, lim + 1), np.arange(lim + 1, lim + 4096), [2 * lim, 3 * lim + 5]])
        maxb = (minb + dims - 1).astype(np.float32).astype(np.int64)   # the axis' largest floor value is a float
        dim = maxb - minb + 1
        for f in (maxb, (minb + (dim - 1) // 2).astype(np.float32).astype(np.int64), np.full_like(maxb, minb)):
            ijk = _pcl_axis_index(f, minb)
            small = dim <= lim
            assert (ijk[small] == (f - minb)[small]).all() and (ijk[small] < dim[small]).all()
        over = _pcl_axis_index(maxb, minb) >= dim
        assert not over[dim <= lim].any()
        reached.append(over[dim > lim].any())
    assert sum(reached) >= 6
    # the example of the header: min_b = 1, a point at 2^25 (leaf 1): the index rounds up to dim = 2^25
    assert _pcl_axis_index(1 << 25, 1) == (1 << 25) == (1 << 25) - 1 + 1
