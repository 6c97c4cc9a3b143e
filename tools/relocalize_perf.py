"""Relocalization in a City-scale prior on one GPU: malio_relocalize time (median and p90 of the host clock around the call, which
returns after the device has finished, over --scans scans after one warm-up call per configuration), nodes_bounded / n_candidates,
the peak device_bytes and the success rate against the truth (the yaw within one step, the position within one lattice step per
axis).  The prior is an aperiodic scene (tests/test_gpu_relocalize.py: buildings of random place, size and heading on ground), 2 km
a side at 4 points per m^2 of surface (tens of millions of points: about what a 0.5 m voxel map of it holds); each scan is 8000 points within 60 m of a random true pose, the guess off by up to 0.8 of the
box in position, keeping the true tilt and nothing of the heading.  The card's name and power limit are read in the same run.

  python tools/relocalize_perf.py [--scans 20] [--out profiles/h100_relocalize.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "ma-lio_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
from malio_b200 import plugin, synth  # noqa: E402
from test_gpu_relocalize import make_scene, q_yaw, sample_scene, scan_of  # noqa: E402

CONFIGS = (("pm50m_res1m", 1.0, 50, 2), ("pm100m_res0.5m", 0.5, 200, 2))   # name, res, half_xy, half_z; 360 yaws


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown", n_yaw=360, scan_points=8000)
    rng = np.random.default_rng(1)
    scene = make_scene(rng, 1000.0, 2700)
    prior = sample_scene(scene, rng, 4.0).astype(np.float32)     # about one point per 0.5 m voxel of every surface
    m = plugin.MeasurementModel(1)
    m.prior_map_load(prior)
    res["prior"] = m.prior_map_info()
    del prior
    extq, extt = [synth.q_exp([0.0, 0.05, 0.0])], [np.array([0.1, 0.0, 0.2])]
    for name, r_, hxy, hz in CONFIGS:
        ts, ratio, dev, ok, score = [], [], [], 0, []
        for i in range(args.scans + 1):
            truth = np.array([rng.uniform(-1000, 1000), rng.uniform(-1000, 1000), 1.8])
            tilt = synth.q_exp(np.array([rng.normal(0, 0.03), rng.normal(0, 0.03), 0.0]))
            psi = rng.uniform(0, 2 * np.pi)
            pw = sample_scene(scene, rng, 2.0, truth[:2], 60.0)
            pw = pw[rng.permutation(len(pw))[:8000]] + rng.normal(0, 0.02, (min(len(pw), 8000), 3))
            pts, table, table_off = scan_of(pw, rng, truth, synth.q_mul(q_yaw(psi), tilt), extq, extt, None)
            guess = synth.make_state(truth + rng.uniform(-0.8, 0.8, 3) * r_ * np.array([hxy, hxy, hz]), tilt, extq, extt)
            m.upload_scan(pts, table, table_off, None)
            t0 = time.perf_counter()
            r = m.relocalize(guess, r_, hxy, hz, n_yaw=360)
            dt = time.perf_counter() - t0
            if i == 0:
                continue                                           # warm-up: module load, first allocations
            ts.append(dt)
            ratio.append(r["nodes_bounded"] / r["n_candidates"])
            dev.append(r["device_bytes"])
            score.append(r["score"] / max(r["n_points"], 1))
            dyaw = (r["yaw_index"] * 2 * np.pi / 360 - psi + np.pi) % (2 * np.pi) - np.pi
            ok += abs(dyaw) <= 2 * np.pi / 360 + 1e-9 and bool(np.all(np.abs(r["pos"] - truth) <= r_ + 1e-9))
        a = np.asarray(ts) * 1e3
        res[name] = dict(res_m=r_, half_xy=hxy, half_z=hz, n_candidates=r["n_candidates"], scans=len(ts),
                         median_ms=float(np.median(a)), p90_ms=float(np.percentile(a, 90)), max_ms=float(a.max()),
                         nodes_bounded_over_candidates_median=float(np.median(ratio)), nodes_bounded_over_candidates_max=float(max(ratio)),
                         device_bytes_peak=int(max(dev)), score_over_n_points_median=float(np.median(score)),
                         success_rate=ok / len(ts))
        print(name, json.dumps(res[name]), flush=True)
    m.close()
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
