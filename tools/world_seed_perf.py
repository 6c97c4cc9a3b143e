"""Keeping a saved map current (malio_world_voxel_seed*, malio_world_voxel_changes_device, malio_world_voxel_save_changes_pcd)
at City-rig sizes.  The prior is synth.make_world's ground and street grid (26 M points, as a City-size saved map) with an
intensity column:
  seed       the prior into a new handle at leaf 0.2 m and 0.1 m, from host memory and from a CUDA tensor, each call timed by
             the host clock (it ends in the library's wait); device_bytes after the seed
  carve      accumulate_carve of City-size street scans (synth.street_scan_city, defaults) on the seeded map (handle A) and on
             a map of the same voxels built by plain accumulates of the same points, never seeded (handle B), alternated per
             scan, each call ending in its own wait
  changes    the removed / added download (voxel_map_changes, ends in a synchronise) and the changes save to a temporary
             directory, after the carved scans
Card name, power limit and max SM clock are read in the same run.  Prints one JSON line; --out also writes it to that file.

  python tools/world_seed_perf.py [--scans 20 --warmup 3 --out profiles/h100_world_seed.json]
"""
import argparse
import json
import os
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
M_PRIOR = 26_000_000
SEED_CHUNK = 1 << 22   # MALIO_SEED_CHUNK


def plant(m, slot, xyz):
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    m.undistort(slot, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), np.array([-10.0, -9.0, -8.0, -7.0]),
                np.tile(np.eye(4), (4, 1, 1)), np.zeros(0), -1)


def stats(ms):
    a = np.array(ms)
    return dict(median_ms=float(np.median(a)), p90_ms=float(np.percentile(a, 90)), n=int(a.size))


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def seed_times(prior, leaf, reps):
    out = {}
    t = torch.from_numpy(prior).cuda()
    for how in ("host", "device"):
        ms = []
        for _ in range(reps):
            m = plugin.MeasurementModel(3)
            dt, n = timed(lambda: m.voxel_map_seed(prior, leaf) if how == "host" else m.voxel_map_seed_tensor(t, leaf))
            ms.append(dt)
            info = m.voxel_map_info()
            m.close()
        out[how] = dict(stats(ms), n_voxels=n, capacity=info["capacity"], device_bytes=info["device_bytes"])
    del t
    return out


def carve_run(prior, leaf, scans, warmup, tmp):
    L = 3
    tags = np.zeros(L, np.float32)
    a, b = plugin.MeasurementModel(L), plugin.MeasurementModel(L)
    a.voxel_map_seed(prior, leaf)
    s0 = synth.make_state([0.0, 0.0, 0.0], Q_ID, [Q_ID] * L, [np.zeros(3)] * L)
    chunk = 1 << 20
    for c in range(0, prior.shape[0], chunk):   # the same voxels, folded by plain accumulates (identity pose: world = body)
        plant(b, 0, prior[c:c + chunk, :3])
        for l in (1, 2):
            plant(b, l, np.zeros((0, 3), np.float32))
        b.voxel_map_accumulate(s0, tags, leaf)
    nva, nvb = a.voxel_map_info()["n_voxels"], b.voxel_map_info()["n_voxels"]
    st = synth.Street()
    ta, tb = [], []
    for k in range(warmup + scans):
        sc = synth.street_scan_city(st, k)
        for m, acc in ((a, ta), (b, tb)) if k % 2 == 0 else ((b, tb), (a, ta)):
            for l in range(L):
                plant(m, l, sc["body"][l])
            dt, _ = timed(lambda: m.voxel_map_accumulate(sc["state"], tags, leaf, carve=True))
            if k >= warmup:
                acc.append(dt)
    ch, sv = [], []
    for _ in range(3):
        dt, (r, ad) = timed(lambda: a.voxel_map_changes())
        ch.append(dt)
        dt, counts = timed(lambda: a.voxel_map_save_changes(os.path.join(tmp, "removed.pcd"), os.path.join(tmp, "added.pcd")))
        sv.append(dt)
    res = dict(leaf=leaf, n_voxels_seeded=nva, n_voxels_unseeded=nvb, carve_seeded=stats(ta), carve_unseeded=stats(tb),
               changes_download=dict(stats(ch), n_removed=int(r.shape[0]), n_added=int(ad.shape[0])),
               changes_save=dict(stats(sv), n_removed=counts[0], n_added=counts[1]),
               device_bytes_seeded=a.voxel_map_info()["device_bytes"])
    a.close()
    b.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.cuda.set_device(0)
    xyz = synth.make_world(M_PRIOR)
    prior = np.concatenate([xyz, np.random.default_rng(1).uniform(0, 255, (xyz.shape[0], 1))], axis=1).astype(np.float32)
    res = dict(card=card(), prior_points=int(prior.shape[0]), seed_chunk=SEED_CHUNK, seed={}, carve=[])
    with tempfile.TemporaryDirectory() as tmp:
        for leaf in (0.2, 0.1):
            res["seed"][str(leaf)] = seed_times(prior, leaf, args.reps)
            res["carve"].append(carve_run(prior, leaf, args.scans, args.warmup, tmp))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
