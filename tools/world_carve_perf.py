"""Clearing moving objects out of the voxel map (malio_world_voxel_accumulate_carve) at City-rig sizes: street scans of
synth.street_scan_city (128 x 1024 spinning rays and 2 x 24 000 cone rays, before the rays without a return are dropped),
max_range 100 m, end_margin 4 m, at two configurations:
  leaf 0.2 m on a map pre-filled to about 1 M voxels, and leaf 0.1 m on a map pre-filled to about 20 M voxels
(the pre-fill is plain accumulates of uniform points over the street's volume, so that the hash is as large as a mapped
city's).  Two handles hold the same map; per scan the same clouds are planted on both and accumulate_carve (handle A) and
accumulate (handle B) are timed alternately, each call ending in its own stream synchronise, so the host clock around it is
its time.  Then, in a separate profiled run, vc_carve_kernel's time from torch.profiler, and the kept save's time.  Card
name, power limit and max SM clock are read in the same run.  Prints one JSON line; --out also writes it to that file.

  python tools/world_carve_perf.py [--scans 20 --warmup 3 --out profiles/h100_world_carve.json]
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from knn_device_perf import card  # noqa: E402
from malio_b200 import capi, plugin, synth  # noqa: E402

Q_ID = np.array([1.0, 0.0, 0.0, 0.0])
CONFIGS = ((0.2, 1_000_000), (0.1, 20_000_000))


def plant(m, slot, xyz):
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    m.undistort(slot, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), np.array([-10.0, -9.0, -8.0, -7.0]),
                np.tile(np.eye(4), (4, 1, 1)), np.zeros(0), -1)


def stats(ms):
    a = np.array(ms)
    return dict(median_ms=float(np.median(a)), p90_ms=float(np.percentile(a, 90)), n=int(a.size))


def run(leaf, fill, scans, warmup):
    st = synth.Street()
    L = 3
    tags = np.zeros(L, np.float32)
    ms = [plugin.MeasurementModel(L) for _ in range(2)]
    rng = np.random.default_rng(7)
    s0 = synth.make_state([0.0, 0.0, 0.0], Q_ID, [Q_ID] * L, [np.zeros(3)] * L)
    chunk = 1 << 17
    for c in range(0, int(fill * 1.05), chunk):
        pre = rng.uniform([-150, -40, -2], [350, 40, 30], (chunk, 3)).astype(np.float32)
        for m in ms:
            plant(m, 0, pre)
            for l in (1, 2):
                plant(m, l, np.zeros((0, 3), np.float32))
            m.voxel_map_accumulate(s0, tags, leaf)
    carve = plugin.carve_args(100.0, 4.0)
    t_carve, t_plain, n_rays = [], [], []
    for k in range(warmup + scans):
        sc = synth.street_scan_city(st, k)
        for m in ms:
            for l in range(L):
                plant(m, l, sc["body"][l])
        n_rays.append(sum(b.shape[0] for b in sc["body"]))
        order = (0, 1) if k % 2 == 0 else (1, 0)
        for which in order:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if which == 0:
                ms[0].voxel_map_accumulate(sc["state"], tags, leaf, carve=carve)
            else:
                ms[1].voxel_map_accumulate(sc["state"], tags, leaf)
            dt = (time.perf_counter() - t0) * 1e3
            if k >= warmup:
                (t_carve if which == 0 else t_plain).append(dt)
    a, b = ms[0].voxel_map_tensor().cpu().numpy(), ms[1].voxel_map_tensor().cpu().numpy()
    same = a.tobytes() == b.tobytes()
    # the carve kernel alone, profiled in a run of its own (the same scans again on handle A)
    from torch.profiler import ProfilerActivity, profile
    kern = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(warmup + scans, warmup + scans + 5):
            sc = synth.street_scan_city(st, k)
            for l in range(L):
                plant(ms[0], l, sc["body"][l])
            ms[0].voxel_map_accumulate(sc["state"], tags, leaf, carve=carve)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        name = re.search(r"(vc_\w+_kernel)", ev.key)
        if name:
            dev = getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)
            kern.append(dict(kernel=name.group(1), calls=int(ev.count), mean_us=float(dev)))
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "kept.pcd")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ms[0].voxel_map_save(p, clear=False, keep=True)
        t_save = (time.perf_counter() - t0) * 1e3
        n_kept = os.path.getsize(p)
    info = ms[0].voxel_map_info()
    e = ms[0].voxel_map_evidence_tensor().cpu().numpy().view(np.uint32).astype(np.int64)
    res = dict(leaf=leaf, voxels=info["n_voxels"], device_bytes=info["device_bytes"], rays_per_scan=float(np.mean(n_rays)),
               accumulate_carve=stats(t_carve), accumulate=stats(t_plain), centroids_identical=same, profiled_kernels=kern,
               kept_save_ms=t_save, kept_file_bytes=n_kept,
               dropped_by_defaults=int(((e[:, 1] >= 2) & (e[:, 1].astype(np.float64) > 2.0 * e[:, 0])).sum()))
    for m in ms:
        m.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    out = dict(tool="world_carve_perf", card=card(), configs=[run(leaf, fill, a.scans, a.warmup) for leaf, fill in CONFIGS])
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(out, indent=2) + "\n")


if __name__ == "__main__":
    main()
