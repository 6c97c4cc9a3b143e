"""Localization in a prior map on one GPU: prior load time (10 M and 50 M points), window slide time (kill + gather + commit) for a
1000 m cube over a City-like prior (0.5 m map leaf: a ground lattice and a street grid of walls), the call without a move, and
the device bytes.  Medians and p90 of host-clock times around calls that end in a device synchronisation (a load and a slide
wait for the device; a call without a move does no device work).  The card's name and power limit are read in the same run.

Prints the result as JSON; --out also writes it to that file.

  python tools/prior_map_perf.py [--out profiles/h100_prior_map.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
from malio_b200 import plugin  # noqa: E402


def stats(ts):
    a = np.asarray(ts) * 1e3
    return dict(n=len(a), median_ms=float(np.median(a)), p90_ms=float(np.percentile(a, 90)))


def city(x_len=3000.0, y_half=600.0, leaf=0.5, block=50.0, wall_h=20.0):
    """Ground z = 0 on a leaf lattice over [0, x_len) x [-y_half, y_half), walls along y every `block` m in x and along x every
    `block` m in y, each a leaf lattice up to wall_h: what a 0.5 m voxel map of a street grid holds."""
    dev = "cuda"
    gx = torch.arange(0, x_len, leaf, device=dev)
    gy = torch.arange(-y_half, y_half, leaf, device=dev)
    gz = torch.arange(0, wall_h, leaf, device=dev)
    X, Y = torch.meshgrid(gx, gy, indexing="ij")
    parts = [torch.stack([X.reshape(-1), Y.reshape(-1), torch.zeros(X.numel(), device=dev)], 1)]
    for c in torch.arange(block / 2, x_len, block, device=dev):          # walls along y at x = c
        Y2, Z2 = torch.meshgrid(gy, gz, indexing="ij")
        parts.append(torch.stack([torch.full((Y2.numel(),), float(c), device=dev), Y2.reshape(-1), Z2.reshape(-1)], 1))
    for c in torch.arange(-y_half + block / 2, y_half, block, device=dev):   # walls along x at y = c
        X2, Z2 = torch.meshgrid(gx, gz, indexing="ij")
        parts.append(torch.stack([X2.reshape(-1), torch.full((X2.numel(),), float(c), device=dev), Z2.reshape(-1)], 1))
    return torch.cat(parts).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown")
    m = plugin.MeasurementModel(1)
    # ---- load
    g = torch.Generator(device="cuda").manual_seed(1)
    for n in (10_000_000, 50_000_000):
        xyz = torch.rand((n, 3), device="cuda", generator=g) * torch.tensor([10000.0, 10000.0, 100.0], device="cuda")
        ny = torch.full((n,), 0.001, device="cuda")
        m.prior_map_load_tensor(xyz, ny)                       # warm-up: allocations, CUB's first launches
        ts = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.prior_map_load_tensor(xyz, ny)                   # returns after the device has finished
            ts.append(time.perf_counter() - t0)
        info = m.prior_map_info()
        res[f"load_{n // 1_000_000}M"] = dict(stats(ts), n_tiles=info["n_tiles"], device_bytes=info["device_bytes"])
        del xyz, ny
        torch.cuda.empty_cache()
    # ---- slides over a City-like prior
    prior = city()
    n = prior.shape[0]
    m.prior_map_load_tensor(prior, torch.full((n,), 0.001, device="cuda"))
    after_load = m.prior_map_info()
    del prior
    torch.cuda.empty_cache()
    cube, det = 1000.0, 100.0
    slide, still, entered, killed, live = [], [], [], [], []
    x = 500.0
    m.prior_map_window((x, 0.0, 1.8), cube, det)
    for rep in range(2):                                       # there and back again, twice
        for x in list(np.arange(500.0, 2500.0, 5.0)) + list(np.arange(2500.0, 500.0, -5.0)):
            t0 = time.perf_counter()
            r = m.prior_map_window((float(x), 0.0, 1.8), cube, det)
            dt = time.perf_counter() - t0
            if r["moved"]:
                slide.append(dt); entered.append(r["n_entered"]); killed.append(r["n_killed"]); live.append(r["n_live"])
            else:
                still.append(dt)
    info = m.prior_map_info()
    # the first call (a full gather and build of the cube) on a fresh window
    m.map_build(np.zeros((1, 3), np.float32), np.zeros(1, np.float32))
    t0 = time.perf_counter()
    r = m.prior_map_window((1500.0, 0.0, 1.8), cube, det)
    t_first = time.perf_counter() - t0
    res["city_prior"] = dict(n_points=after_load["n_points"], n_tiles=after_load["n_tiles"], device_bytes_after_load=after_load["device_bytes"],
                             device_bytes_after_slides=info["device_bytes"], map_slots_live=list(m.map_info()))
    res["slide"] = dict(stats(slide), entered_median=int(np.median(entered)), killed_median=int(np.median(killed)),
                        live_median=int(np.median(live)))
    res["no_move"] = stats(still)
    res["first_call"] = dict(ms=t_first * 1e3, n_live=r["n_live"])
    m.close()
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
