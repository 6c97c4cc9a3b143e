"""Relocalization without a position guess in a City-scale prior on one GPU: malio_place_db_build (host clock around the call, which
returns after the device has finished) and the database's bytes, then malio_relocalize_global on --scans ray-cast scans at random
free poses with random yaw and the true tilt: the time of the query descriptor plus stages 1-2 and of the verification (the
report's host clocks), how many scans were found (the yaw within one yaw step, the position within one lattice step per axis),
and the stage-2 rank of the truth (the first candidate within one lattice step of it; None when none is).  The prior is tools/relocalize_perf.py's: the
aperiodic scene of tests/test_gpu_relocalize.py, 2 km a side at 4 points per m^2 of surface; the scans are the spinning pattern
of tests/test_gpu_place.py (32 beams over +-22.5 degrees, 900 azimuths, 100 m).  The card's name and power limit are read in
the same run.

  python tools/place_perf.py [--scans 50] [--out profiles/h100_place.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "ma-lio_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
from malio_b200 import plugin, synth  # noqa: E402
from test_gpu_place import _angle_deg, _free, raycast  # noqa: E402
from test_gpu_relocalize import make_scene, q_yaw, sample_scene, scan_of  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown")
    rng = np.random.default_rng(1)
    scene = make_scene(rng, 1000.0, 2700)
    prior = sample_scene(scene, rng, 4.0).astype(np.float32)
    m = plugin.MeasurementModel(1)
    m.prior_map_load(prior)
    res["prior"] = m.prior_map_info()
    del prior
    step, fov = 1.0, math.radians(22.5)
    builds = []
    for _ in range(2):                                             # the first build also loads the module
        t0 = time.perf_counter()
        db = m.place_db_build(1.8, step=step, fov_up=fov)
        builds.append(time.perf_counter() - t0)
    res["database"] = dict(db, build_s_first=builds[0], build_s=builds[1])
    print("database", json.dumps(res["database"]), flush=True)
    extq, extt = [synth.q_exp([0.0, 0.05, 0.0])], [np.array([0.1, 0.0, 0.2])]
    t_rank, t_ver, t_all, r2, ok, ratio = [], [], [], [], 0, []
    for i in range(args.scans + 1):
        while True:
            o = np.array([rng.uniform(-950, 950), rng.uniform(-950, 950), 1.8])
            if _free(scene, o):
                break
        tilt = synth.q_exp(np.array([rng.normal(0, 0.03), rng.normal(0, 0.03), 0.0]))
        psi = rng.uniform(0, 2 * np.pi)
        rot = synth.q_mul(q_yaw(psi), tilt)
        truth = o - synth.q_to_R(rot) @ extt[0]
        pts, table, table_off = scan_of(raycast(scene, o, psi, tilt, rng), rng, truth, rot, extq, extt, None)
        m.upload_scan(pts, table, table_off, None)
        t0 = time.perf_counter()
        r = m.relocalize_global(synth.make_state(np.zeros(3), tilt, extq, extt))
        dt = time.perf_counter() - t0
        if i == 0:
            continue                                               # warm-up
        t_rank.append(r["ms_rank"])
        t_ver.append(r["ms_verify"])
        t_all.append(dt * 1e3)
        ratio.append(r["score"] / max(r["n_points"], 1))
        found = _angle_deg(r["rot"], rot) <= 1.0 + 1e-6 and bool(np.all(np.abs(r["pos"][:2] - truth[:2]) <= 0.5 + 1e-9))
        ok += found
        # the truth's stage-2 rank: the first candidate whose sensor (column centre) lies within one lattice step of the origin
        cand_cols = [tuple(c["col"]) for c in r["cand"]]
        r2.append(next((k for k, c in enumerate(cand_cols) if np.hypot(c[0] + 0.5 - o[0], c[1] + 0.5 - o[1]) <= step), None))
        print(f"scan {i}: found {found} rank {r2[-1]} score {r['score']}/{r['n_points']} rank {r['ms_rank']:.1f} ms "
              f"verify {r['ms_verify']:.1f} ms", flush=True)
    hist = {}
    for v in r2:
        hist[str(v)] = hist.get(str(v), 0) + 1
    a = np.asarray(t_all)
    res["query"] = dict(scans=len(t_all), found=ok, rank_plus_stages_ms_median=float(np.median(t_rank)),
                        rank_plus_stages_ms_p90=float(np.percentile(t_rank, 90)), verify_ms_median=float(np.median(t_ver)),
                        verify_ms_p90=float(np.percentile(t_ver, 90)), total_ms_median=float(np.median(a)),
                        total_ms_p90=float(np.percentile(a, 90)), total_ms_max=float(a.max()),
                        truth_stage2_rank_histogram=hist, score_over_n_points_median=float(np.median(ratio)),
                        defaults=dict(k1=256, k2=8, yaw_step_deg=1.0, res=0.5, half_z=2, cell=1.0, step=step, r_max=60.0, n_ring=20,
                                      n_sector=72, z_lo="-sensor_height + 0.5", block_level=2, fov_up_deg=22.5))
    print(json.dumps(res, indent=1))
    m.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
