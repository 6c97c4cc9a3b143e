"""Localization past the prior's edge on one GPU (malio_prior_map_extend): the extend call per C2-size scan (100k points) wholly
off the prior (every candidate admitted and folded) and wholly on it (none admitted), a window slide with a 5 M-point session
against the same slide with an empty session, and the device bytes per session point.  Medians and p90 of host-clock times
around calls that end in a device synchronisation (extend and a slide wait for the device).  The card's name and power limit
are read in the same run.

Prints the result as JSON; --out also writes it to that file.

  python tools/prior_extend_perf.py [--out profiles/h100_prior_extend.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from dataclasses import replace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
from malio_b200 import plugin, synth  # noqa: E402

F = np.float32
N_SCAN = 100_000


def stats(ts):
    a = np.asarray(ts) * 1e3
    return dict(n=len(a), median_ms=float(np.median(a)), p90_ms=float(np.percentile(a, 90)))


def ground(x0, x1, y_half, leaf=0.5):
    """A ground lattice z = 0 at the map leaf: every 0.5 m voxel of the ground layer holds a point."""
    gx, gy = np.meshgrid(np.arange(x0, x1, leaf), np.arange(-y_half, y_half, leaf), indexing="ij")
    return np.column_stack([gx.ravel(), gy.ravel(), np.zeros(gx.size)]).astype(F)


def scan_case(base, x_lo, rng):
    """A scan of N_SCAN points 5 cm to 45 cm above the ground over [x_lo, x_lo + 80) x [-50, 50) (about three points per 0.5 m
    voxel), rendered from a sensor at its centre.  Returns (case, state)."""
    pw = np.column_stack([rng.uniform(x_lo, x_lo + 80, N_SCAN), rng.uniform(-50, 50, N_SCAN), rng.uniform(0.05, 0.45, N_SCAN)])
    x = synth.make_state((x_lo + 40.0, 0.0, 1.8), (1.0, 0.0, 0.0, 0.0), [(1.0, 0.0, 0.0, 0.0)], [(0.0, 0.0, 0.0)])
    return synth.with_scan(replace(base, x_true=x), pw, seed=int(x_lo) & 0xFFFF), x


def extend_once(m, prior, cx, t):
    case, x = cx
    m.prior_map_load(prior, np.full(len(prior), 0.001, F))
    m.prior_map_window(np.zeros(3), 400.0, 50.0)
    m.upload_scan(case.pts, case.table, case.table_off, None)
    m.h_share_model(x, True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = m.prior_map_extend(x, 0.5)
    t.append(time.perf_counter() - t0)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown", scan_points=N_SCAN)
    rng = np.random.default_rng(1)
    base = synth.make_case("c2-size scan", 1000, 1000, 1, 3)
    prior = ground(-180.0, 0.0, 100.0)                  # 144k points west of x = 0
    m = plugin.MeasurementModel(1, params=base.params)
    # ---- extend per scan: off the prior (all admitted) and on it (none)
    off, on = scan_case(base, 20.0, rng), scan_case(base, -120.0, rng)
    t_off, t_on, reps = [], [], {}
    for k in range(args.reps + 3):
        a, b = [], []
        reps["off"] = extend_once(m, prior, off, a)
        reps["on"] = extend_once(m, prior, on, b)
        if k >= 3:
            t_off += a; t_on += b
    res["extend_off_prior"] = dict(stats(t_off), **reps["off"])
    res["extend_on_prior"] = dict(stats(t_on), **reps["on"])
    # ---- a slide with a 5 M-point session (all outside the cube) against the same slide with an empty session
    hs = {}
    for name in ("empty", "session_5M"):
        h = plugin.MeasurementModel(1, params=base.params)
        h.prior_map_load(prior, np.full(len(prior), 0.001, F))
        h.prior_map_window(np.array([-90.0, 0.0, 0.0]), 200.0, 20.0)
        hs[name] = h
    h = hs["session_5M"]
    n_sess, k = 0, 0
    while n_sess < 5_000_000:
        c, x = scan_case(base, 1000.0 + 100.0 * k, rng)   # outside the cube: the session grows, the window does not
        h.upload_scan(c.pts, c.table, c.table_off, None)
        h.h_share_model(x, True)
        r = h.prior_map_extend(x, 0.5)
        if r["n_inserted"] == 0:
            raise RuntimeError(f"a scan outside the prior inserted nothing: {r}")
        n_sess = r["n_session"]
        k += 1
    res["session_points"] = int(n_sess)
    ts = {name: [] for name in hs}
    cube = {name: hh.prior_map_window(np.array([-90.0, 0.0, 0.0]), 200.0, 20.0)["cube"] for name, hh in hs.items()}
    for rep in range(args.reps + 3):
        for name, hh in hs.items():
            c = cube[name]
            pos = np.array([(c[0] + 15.0) if rep % 2 else (c[3] - 15.0), 0.0, 0.0])   # 15 m inside a face: the cube moves
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = hh.prior_map_window(pos, 200.0, 20.0)
            dt = time.perf_counter() - t0
            assert r["moved"]
            cube[name] = r["cube"]
            if rep >= 3:
                ts[name].append(dt)
    res["slide_empty_session"] = stats(ts["empty"])
    res["slide_5M_session"] = stats(ts["session_5M"])
    # after the slides: the window's scratch has grown to what a slide needs, with the session and without
    b_empty = hs["empty"].prior_map_info()["device_bytes"]
    b_sess = hs["session_5M"].prior_map_info()["device_bytes"]
    res["device_bytes_per_session_point"] = dict(store=16, measured=(b_sess - b_empty) / n_sess,
                                                 note="measured after the timed slides: the handle's prior-map bytes with the session "
                                                      "minus without, over the session's points (the store's growth slack, the "
                                                      "slide's compaction scratch and the extend scratch included)")
    for hh in hs.values():
        hh.close()
    m.close()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
