"""The numpy reference of the scan's pose-uncertainty build (tests/scan_unc_ref.py) and the host compounding it is compared with
(no GPU):
  - the reference against a second transcription of IMU_Processing.hpp:474-523 that walks every point with its own
    cov_pointer, as the reference's loop does;
  - where the output-aliases-input field order matters (laserMapping.cpp:1043) and where it cannot (IMU_Processing.hpp:490-491);
  - malio_pose_initial / malio_compound_* / malio_build_pose_unc return the bytes they returned before the compounding moved
    into malio_compound.h, the header the device shares (tests/golden/compound_golden.npz, tests/golden/make_compound_golden.py)."""
import os

import numpy as np
import pytest

import helpers as H
import np_oracle as npo
import scan_unc_ref as R
from malio_b200 import capi, plugin

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "compound_golden.npz")


def _loop_transcription(slots, imu_cov, extrinsic, uncertainty):
    """kf.lidar_uncertainty by the reference's own loop: every point from the last down to the second, one spline pose per
    point, the cov_pointer test and decrement of :484-486."""
    ltl = R.lt_lidar_frames(slots, imu_cov, uncertainty)
    out = []
    for num, c in enumerate(slots):
        t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
        cov_t = c["imu_cov_t"]
        cp = c["cov_pointer"]
        lst = []
        for i in range(t.shape[0] - 1, 0, -1):
            if cp >= 0 and cov_t[cp] > t[i]:
                cp -= 1
                ok, P = H.spline_pose_ref(c["ctrl_t"], c["ctrl_T"], [t[i]])
                lst.append(R.entry(R.quat_of(P[0, :3, :3]), P[0, :3, 3], imu_cov[cp + 1], extrinsic[num], ltl[num]))
        out.append(lst)
    return out


def _close(a, b, tol):
    assert len(a) == len(b)
    for p, q in zip(a, b):
        assert np.abs(p.T - q.T).max() <= tol
        assert np.abs(p.cov - q.cov).max() <= tol * np.abs(q.cov).max()


@pytest.mark.parametrize("L", [1, 2, 3])
def test_reference_matches_loop_transcription(L):
    slots, imu_cov, ext, unc = R.make_scan(L, n=[3000, 2000, 2500][:L], seed=90 + L)
    lists, tcs, table = R.scan_uncertainty(slots, imu_cov, ext, unc)
    loop = _loop_transcription(slots, imu_cov, ext, unc)
    for a, b in zip(lists, loop):
        assert len(a) > 10
        _close(a, b, 1e-12)
    assert len(tcs) == L - 1
    assert [len(t) for t in table] == [len(a) - 1 for a in lists]


def _tc_and_list(seed=5):
    slots, imu_cov, ext, unc = R.make_scan(2, n=[1500, 1500], seed=seed)
    lists, tcs, table = R.scan_uncertainty(slots, imu_cov, ext, unc)
    return slots, imu_cov, ext, unc, lists, tcs, table


def test_aliasing_in_pose_unc_has_teeth():
    """laserMapping.cpp:1043 writes compoundPoseWithCov's output into its second input, so adjointMatrix (associate_uct.hpp:99)
    sees the NEW T_.  Reading the old one instead moves the table entries of LiDAR 1 by far more than the 1e-9 bar."""
    _, _, ext, _, lists, tcs, table = _tc_and_list()
    worst = 0.0
    for i, lu in enumerate(lists[1][:-1]):
        pp = npo.Pose([1, 0, 0, 0], [0, 0, 0], np.zeros((6, 6)))
        npo.compound_pose_with_cov(ext[1], ext[1].cov, lu, lu.cov, pp)
        fresh = npo.Pose([1, 0, 0, 0], [0, 0, 0], np.zeros((6, 6)))
        npo.compound_pose_with_cov(tcs[0], tcs[0].cov, pp, pp.cov, fresh)     # output NOT aliasing the input
        fresh.cov = npo.compound_inv_pose_with_cov(ext[0], ext[0].cov, fresh, fresh.cov, fresh)
        ref = table[1][i]
        assert np.abs(fresh.T - ref.T).max() < 1e-12                           # the pose itself does not depend on it
        worst = max(worst, np.abs(fresh.cov - ref.cov).max() / np.abs(ref.cov).max())
    assert worst > 1e-4, worst


def test_aliasing_in_uncertainty_lists_is_harmless():
    """IMU_Processing.hpp:490-491 also write into their second input, but compoundInvPoseWithCov reads pose_2 only before it
    writes pose_cp, and its adjoint is of the output's T_ either way: the non-aliasing variant gives the same bits."""
    slots, imu_cov, ext, unc, lists, _, _ = _tc_and_list()
    ltl = R.lt_lidar_frames(slots, imu_cov, unc)
    c = slots[1]
    t = c["pts"]["curvature"].astype(np.float64) / 1000.0 + c["beg_time"]
    _, n_pops, pop = H.walk_ref(t, c["imu_cov_t"], c["cov_pointer"])
    ok, P = H.spline_pose_ref(c["ctrl_t"], c["ctrl_T"], t[pop])
    for k in range(n_pops):
        pt = npo.Pose(R.quat_of(P[k, :3, :3]), P[k, :3, 3], imu_cov[c["cov_pointer"] - k])
        a = npo.Pose([1, 0, 0, 0], [0, 0, 0], np.zeros((6, 6)))
        npo.compound_pose_with_cov(pt, pt.cov, ext[1], ext[1].cov, a)
        b = npo.Pose([1, 0, 0, 0], [0, 0, 0], np.zeros((6, 6)))
        b.cov = npo.compound_inv_pose_with_cov(ltl[1], ltl[1].cov, a, a.cov, b)
        d = npo.Pose([1, 0, 0, 0], [0, 0, 0], np.zeros((6, 6)))
        d.cov = npo.compound_inv_pose_with_cov(ext[1], ext[1].cov, b, b.cov, d)
        assert np.array_equal(d.T, lists[1][k].T) and np.array_equal(d.cov, lists[1][k].cov)


def test_host_compounding_bytes_unchanged():
    g = np.load(GOLDEN)
    lib = capi.load()
    p1, p2 = g["p1"].view(capi.POSE), g["p2"].view(capi.POSE)
    # PoseInitial: T_ from q_, t_
    again = np.zeros_like(p1)
    for k in range(p1.shape[0]):
        lib.malio_pose_initial(again[k:k + 1].ctypes.data, capi.ptr(p1[k]["t"].copy()), capi.ptr(p1[k]["q"].copy()),
                               capi.ptr(p1[k]["cov"].copy()))
    assert again.tobytes() == p1.tobytes()
    for name, fn in (("cp", lib.malio_compound_pose_with_cov), ("inv", lib.malio_compound_inv_pose_with_cov)):
        fresh = np.zeros_like(p1)
        alias = p2.copy()
        for k in range(p1.shape[0]):
            a, b, o, s = p1[k:k + 1], p2[k:k + 1], fresh[k:k + 1], alias[k:k + 1]
            fn(a.ctypes.data, a["cov"].ctypes.data, b.ctypes.data, b["cov"].ctypes.data, o.ctypes.data, o["cov"].ctypes.data)
            fn(a.ctypes.data, a["cov"].ctypes.data, s.ctypes.data, s["cov"].ctypes.data, s.ctypes.data, s["cov"].ctypes.data)
        assert fresh.tobytes() == g[name + "_fresh"].tobytes(), name
        assert alias.tobytes() == g[name + "_alias"].tobytes(), name
    counts = {1: [6], 2: [2, 6], 3: [6, 0, 1]}
    for L, cs in counts.items():
        ext = g[f"L{L}_ext"].view(capi.POSE)
        tc = g[f"L{L}_tc"].view(capi.POSE) if L > 1 else None
        flat = g[f"L{L}_lists"].view(capi.POSE)
        ends = np.cumsum(cs)
        lists = [flat[e - c:e] for c, e in zip(cs, ends)]
        table, off = plugin.build_pose_unc(ext, tc, lists)
        assert table.tobytes() == g[f"L{L}_table"].tobytes() and np.array_equal(off, g[f"L{L}_off"])
