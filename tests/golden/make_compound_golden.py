"""Generates tests/golden/compound_golden.npz: the bytes the library's host pose compounding returned when it lived in
malio_host.cpp, before it moved into the header it now shares with the device (malio_compound.h).  Rerun only to pin a new
version on purpose:

    python tests/golden/make_compound_golden.py

Contents: seeded random poses with symmetric positive definite covariances, and the outputs of malio_pose_initial,
malio_compound_pose_with_cov and malio_compound_inv_pose_with_cov (fresh output and output aliasing the second input, as
laserMapping.cpp:1043-1044 and IMU_Processing.hpp:490-491 call them), and of malio_build_pose_unc for L = 1, 2, 3 with lists
of 0, 1, 2 and 6 entries.
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
from malio_b200 import capi, plugin, synth  # noqa: E402

N = 64
COUNTS = {1: [6], 2: [2, 6], 3: [6, 0, 1]}


def rand_poses(rng, n):
    lib = capi.load()
    out = np.zeros(n, capi.POSE)
    for k in range(n):
        q = synth.q_normalize(rng.normal(0, 1, 4))
        t = rng.normal(0, 5, 3)
        A = rng.normal(0, 1, (6, 6))
        cov = A @ A.T * 10.0 ** rng.uniform(-6, -2) + np.eye(6) * 1e-8
        lib.malio_pose_initial(out[k:k + 1].ctypes.data, capi.ptr(np.ascontiguousarray(t)), capi.ptr(np.ascontiguousarray(q)),
                               capi.ptr(np.ascontiguousarray(cov)))
    return out


def compound_all(p1, p2):
    """Per pair: compound / inverse compound into a fresh pose and into the second input (aliased)."""
    lib = capi.load()
    res = {}
    for name, fn in (("cp", lib.malio_compound_pose_with_cov), ("inv", lib.malio_compound_inv_pose_with_cov)):
        fresh = np.zeros(p1.shape[0], capi.POSE)
        alias = p2.copy()
        for k in range(p1.shape[0]):
            a, b, o = p1[k:k + 1], p2[k:k + 1], fresh[k:k + 1]
            fn(a.ctypes.data, a["cov"].ctypes.data, b.ctypes.data, b["cov"].ctypes.data, o.ctypes.data, o["cov"].ctypes.data)
            s = alias[k:k + 1]
            fn(a.ctypes.data, a["cov"].ctypes.data, s.ctypes.data, s["cov"].ctypes.data, s.ctypes.data, s["cov"].ctypes.data)
        res[name + "_fresh"], res[name + "_alias"] = fresh, alias
    return res


def pose_unc_all(rng):
    res = {}
    for L, counts in COUNTS.items():
        ext = rand_poses(rng, L)
        tc = rand_poses(rng, L - 1) if L > 1 else None
        lists = [rand_poses(rng, c) for c in counts]
        table, off = plugin.build_pose_unc(ext, tc, lists)
        res[f"L{L}_ext"], res[f"L{L}_lists"] = ext, np.concatenate(lists)
        if tc is not None:
            res[f"L{L}_tc"] = tc
        res[f"L{L}_table"], res[f"L{L}_off"] = table, off
    return res


def main():
    rng = np.random.default_rng(20261016)
    p1, p2 = rand_poses(rng, N), rand_poses(rng, N)
    out = dict(p1=p1, p2=p2, **compound_all(p1, p2), **pose_unc_all(rng))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "compound_golden.npz")
    np.savez_compressed(path, **{k: v.view(np.uint8) if v.dtype.names else v for k, v in out.items()})
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
