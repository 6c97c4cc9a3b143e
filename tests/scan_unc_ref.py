"""numpy restatement of the scan's pose-uncertainty build (test infrastructure): the rest of UndistortPcl
(IMU_Processing.hpp:474-523) and the pose_unc loop of laserMapping.cpp:1028-1048, in the reference's loop form, from
np_oracle's compoundings, helpers.spline_pose_ref's scipy spline and helpers.walk_ref's covariance-list walk.

A scan here is a list of slot dicts (synth.undistort_case fields plus `lt` = (q wxyz, t), the IMU pose at that LiDAR's scan
end) sharing one IMU-covariance list: imu_cov[k] is the 6x6 covariance of imu_cov_t[k]."""
import numpy as np
from scipy.spatial.transform import Rotation

import helpers as H
import np_oracle as npo
from malio_b200 import capi, synth


def quat_of(R):
    """(w, x, y, z) of a rotation matrix (sign as scipy picks it: T_ and every covariance do not depend on it)."""
    return Rotation.from_matrix(R).as_quat()[..., [3, 0, 1, 2]]


def lt_lidar_frames(slots, imu_cov, uncertainty):
    """lt_lidar_frame[num]: PoseInitial with getUncertainty() for LiDAR 0 (:450), imu_cov[cov_pointer] otherwise (:471)."""
    return [npo.Pose(c["lt"][0], c["lt"][1], uncertainty if num == 0 else imu_cov[c["cov_pointer"]]) for num, c in enumerate(slots)]


def entry(pt_q, pt_t, cov, extrinsic, ltl):
    """uncertainty[num][k] (:487-492): the last two compoundings write into their second input."""
    pt = npo.Pose(pt_q, pt_t, cov)
    pc = npo.Pose([1, 0, 0, 0], [0, 0, 0], np.zeros((6, 6)))
    npo.compound_pose_with_cov(pt, pt.cov, extrinsic, extrinsic.cov, pc)
    pc.cov = npo.compound_inv_pose_with_cov(ltl, ltl.cov, pc, pc.cov, pc)
    pc.cov = npo.compound_inv_pose_with_cov(extrinsic, extrinsic.cov, pc, pc.cov, pc)
    return pc


def scan_uncertainty(slots, imu_cov, extrinsic, uncertainty):
    """Returns (lists: per slot a list of npo.Pose = kf.lidar_uncertainty, temporal_comp: L-1 npo.Pose, table: per slot a list
    of npo.Pose = pose_unc).  extrinsic: L npo.Pose.  A pop point the spline cannot reach takes the identity pose."""
    ltl = lt_lidar_frames(slots, imu_cov, uncertainty)
    lists = []
    for num, c in enumerate(slots):
        t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]                  # :482
        _, n_pops, pop_point = H.walk_ref(t, c["imu_cov_t"], c["cov_pointer"])
        ok, P = H.spline_pose_ref(c["ctrl_t"], c["ctrl_T"], t[pop_point])                       # :483
        c0 = c["cov_pointer"]
        lists.append([entry(quat_of(P[k, :3, :3]), P[k, :3, 3], imu_cov[c0 - k], extrinsic[num], ltl[num]) for k in range(n_pops)])
    tcs = []
    for num in range(1, len(slots)):                                                             # :518
        tc = npo.Pose([1, 0, 0, 0], [0, 0, 0], np.zeros((6, 6)))
        tc.cov = npo.compound_inv_pose_with_cov(ltl[0], ltl[0].cov, ltl[num], ltl[num].cov, tc)
        tcs.append(tc)
    return lists, tcs, npo.build_pose_unc(extrinsic, tcs, lists)


# ---- scans for the tests: L slots sharing one spline and one IMU-covariance list, LiDAR l ending 10 ms x l before LiDAR 0
def cov_pointer_at(cov_t, end_time):
    """cov_pointer as IMU_Processing.hpp:455-466 leaves it (clamped to the list)."""
    cp = cov_t.shape[0] - 1
    while cp >= 0 and cov_t[cp] > end_time:
        cp -= 1
    return min(cp + 1, cov_t.shape[0] - 1)


def rand_cov(rng, n):
    A = rng.normal(0, 1, (n, 6, 6))
    return A @ A.transpose(0, 2, 1) * 1e-4 + np.eye(6) * 1e-6


def make_scan(L, n=4000, seed=80, **kw):
    """(slots, imu_cov[n_cov,6,6], extrinsic npo.Pose[L], uncertainty[6,6])."""
    rng = np.random.default_rng(seed)
    slots = []
    for l in range(L):
        c = synth.undistort_case(n if np.isscalar(n) else n[l], lidar=l, seed=seed + l, **kw)
        if l:
            base = slots[0]
            c = dict(c, ctrl_t=base["ctrl_t"], ctrl_T=base["ctrl_T"], imu_cov_t=base["imu_cov_t"], end_time=base["end_time"] - 0.01 * l)
            if kw.get("lists") == "last_cov":
                c["cov_pointer"] = base["cov_pointer"]
            elif base["imu_cov_t"].shape[0]:
                c["cov_pointer"] = cov_pointer_at(base["imu_cov_t"], c["end_time"])
        ok, P = H.spline_pose_ref(c["ctrl_t"], c["ctrl_T"], [c["end_time"]])
        c["lt"] = (quat_of(P[0, :3, :3]), P[0, :3, 3].copy())
        slots.append(c)
    imu_cov = rand_cov(rng, slots[0]["imu_cov_t"].shape[0])
    ext = [npo.Pose(c["extrinsic"][0], c["extrinsic"][1], rand_cov(rng, 1)[0]) for c in slots]
    return slots, imu_cov, ext, rand_cov(rng, 1)[0]


def to_capi(poses):
    """npo.Pose list -> capi.POSE array (T_ as the numpy restatement computed it)."""
    out = np.zeros(len(poses), capi.POSE)
    for k, p in enumerate(poses):
        out[k]["q"], out[k]["t"], out[k]["T"], out[k]["cov"] = p.q, p.t, p.T, p.cov
    return out
