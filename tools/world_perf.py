"""publish_frame_world and the saved map on the GPU: 3 LiDAR slots x 100k raw points (feats_undistort of a 3-LiDAR scan).

Reports, with the card's name and power limit read in the same run:
  register   malio_world_register(dense) per call: host clock (the call ends in a stream synchronise), and the device time of
             the transform kernels alone and with the one device-to-host copy (torch.profiler, CUDA activities, in a separate
             window of its own)
  accumulate malio_world_accumulate per scan over 100 scans (30 M points in the end, the buffer regrown on the way)
  save       malio_world_save_pcd of that cloud (960 MB file in a temporary directory, removed afterwards)
GPU only: fails without a device.  Usage: python tools/world_perf.py [--reps 50] [--scans 100] [--out file.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
import numpy as np  # noqa: E402

from malio_b200 import capi, plugin, synth  # noqa: E402

N_RAW, L = 100_000, 3


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def setup():
    case = synth.make_case("world-perf", 2000, 20000, L, 3)
    m = plugin.MeasurementModel(L, params=case.params)
    m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    for l in range(L):
        c = synth.undistort_case(N_RAW, lidar=l, seed=500 + l)
        ok, q, p = plugin.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], c["end_time"])
        m.undistort(l, c["pts"], c["beg_time"], c["extrinsic"], (q, p), c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
    return m, case.x_true, np.array([2.0, 1.0, 0.0], np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("world_perf.py needs a CUDA device")
    name, power = card()
    m, x, tags = setup()
    n = L * N_RAW
    out = np.zeros((n, 4), np.float32)
    try:   # pinned destination: the D2H copy at full bandwidth, as a caller that cares would pass it
        out = torch.empty((n, 4), dtype=torch.float32, pin_memory=True).numpy()
    except RuntimeError:
        pass
    ps = x.pass_state()
    nv = capi.load().malio_world_register
    cnt = C.c_uint32(0)

    def reg(cap):
        rc = nv(m._h, C.byref(ps), capi.WORLD_DENSE, capi.ptr(tags), capi.ptr(out) if cap else None, cap, C.byref(cnt))
        assert rc == capi.OK, rc

    for _ in range(10):
        reg(n)
    t = []
    for _ in range(a.reps):
        t0 = time.perf_counter(); reg(n); t.append(time.perf_counter() - t0)
    res = dict(card=name, power_limit=power, points_per_scan=n, register_wall_ms_median=1e3 * float(np.median(t)))

    # device time: a profiled window of its own
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            reg(n)
    k_us, c_us = 0.0, 0.0
    for e in prof.events():
        dt = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
        if "world_kernel" in e.name:
            k_us += dt
        elif "Memcpy DtoH" in e.name:
            c_us += dt
    res["register_kernel_ms"] = k_us / a.reps / 1e3
    res["register_kernel_plus_d2h_ms"] = (k_us + c_us) / a.reps / 1e3
    res["register_bytes_moved_per_call"] = n * (20 + 16)        # d_ud read + staging write (the D2H adds n x 16)

    # accumulate over `scans` scans (the same clouds each time), then save
    t = []
    for _ in range(a.scans):
        t0 = time.perf_counter(); total = m.pcd_accumulate(ps, tags); t.append(time.perf_counter() - t0)
    res.update(accumulate_scans=a.scans, accumulate_points=int(total), accumulate_wall_ms_median=1e3 * float(np.median(t)),
               accumulate_wall_ms_max=1e3 * float(np.max(t)), accumulate_wall_ms_total=1e3 * float(np.sum(t)))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "result.pcd")
        t0 = time.perf_counter(); m.pcd_save(path, clear=True); ts = time.perf_counter() - t0
        size = os.path.getsize(path)
    res.update(save_wall_s=ts, save_file_bytes=size, save_mb_per_s=size / ts / 1e6)
    m.close()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
