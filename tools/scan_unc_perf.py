"""Time malio_scan_uncertainty on the GPU against the host alternative (download the pop poses, compound on the host).

3 LiDAR slots x 100k raw points; the IMU-covariance list at two rates: ~40 entries per scan (333 Hz) and 512 (4266 Hz).
  device   host clock around the (synchronous) call, median of --reps; the kernel's own time from torch.profiler
  host     the same build through the host C-ABI from the poses malio_undistort returns: once as a Python loop over
           malio_compound_* (ctypes overhead included), and as the C-level floor: malio_build_pose_unc's time per compounding
           (one C call, 3 compoundings per entry) times the number of compoundings the build needs
Prints one JSON line (also written to --out) with the card name and power limit.

    python tools/scan_unc_perf.py --reps 50 --out /tmp/scan_unc_perf.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "ma-lio_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import scan_unc_ref as R  # noqa: E402
import test_gpu_scan_uncertainty as T  # noqa: E402
from malio_b200 import capi, plugin  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def raw_args(imu_cov, ext_c, unc):
    cov = np.ascontiguousarray(imu_cov.reshape(-1, 36))
    u = np.ascontiguousarray(unc.reshape(36))
    a = capi.ScanUncArgs()
    a.imu_cov, a.n_cov, a.extrinsic, a.uncertainty = cov.ctypes.data, cov.shape[0], ext_c.ctypes.data, u.ctypes.data
    return a, (cov, u, ext_c)


def kernel_ms(m, call, n):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        torch.cuda.synchronize()
    ts = [e.device_time_total for e in prof.key_averages() if "scan_unc_kernel" in e.key]
    return (ts[0] / 1000.0 / n) if ts else float("nan")


def run(hz, reps):
    slots, imu_cov, ext, unc = R.make_scan(3, n=100_000, seed=11, imu_hz=hz, lists="max" if hz > 1000 else "default")
    m = plugin.MeasurementModel(3)
    g = T._undistort_all(m, slots)
    ext_c = R.to_capi(ext)
    a, keep = raw_args(imu_cov, ext_c, unc)
    table = np.zeros(3 * capi.MAX_COV, capi.POSE_ENTRY)
    off = np.zeros(4, np.uint32)
    tc = np.zeros(2, capi.POSE)
    call = lambda: m.lib.malio_scan_uncertainty(m._h, C.byref(a), capi.ptr(table), table.shape[0], capi.ptr(off), capi.ptr(tc), None, None)
    for _ in range(5):
        assert call() == capi.OK
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        wall.append((time.perf_counter() - t0) * 1e3)
    pops = [len(x["pop_point"]) for x in g]
    n_tab = int(off[3])
    # host: Python loop over the C-ABI (what a caller without this entry point writes today, in Python)
    t0 = time.perf_counter()
    lists, tch, table_h, off_h = T._host_compound(slots, g, imu_cov, ext_c, unc)
    py_ms = (time.perf_counter() - t0) * 1e3
    assert table_h.tobytes() == table[:n_tab].tobytes()
    # host, C-level floor: time per compounding inside one malio_build_pose_unc call (LiDAR-1 entries, 3 compoundings each)
    big = np.concatenate(lists * 4)[:2000]
    t0 = time.perf_counter()
    for _ in range(5):
        plugin.build_pose_unc(ext_c[:2], tch[:1], [big[:1], big])
    per_comp_us = (time.perf_counter() - t0) / 5 / ((big.shape[0] - 1) * 3) * 1e6
    n_comp = 3 * sum(pops) + 2 + 3 * (n_tab - max(pops[0] - 1, 0))
    res = dict(imu_hz=hz, n_cov=int(imu_cov.shape[0]), pops=pops, table_entries=n_tab, device_call_ms_median=float(np.median(wall)),
               device_call_ms_min=float(np.min(wall)), device_kernel_ms=kernel_ms(m, call, reps), host_python_loop_ms=py_ms,
               host_c_us_per_compounding=per_comp_us, host_c_floor_ms=per_comp_us * n_comp / 1e3, compoundings=n_comp)
    m.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = dict(card=card(), runs=[run(hz, args.reps) for hz in (333.0, 4266.0)])
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
