"""The saved map as a voxel map (malio_world_voxel_*) at City-rig sizes: three LiDAR slots of 131 072 + 24 000 + 24 000 points
(uniform over an 80 m disc, 8 m of height), registered with a state that drives along x, leaf 0.1 m, on one handle that also
keeps the dense cloud (malio_world_accumulate) of the same scans.

  fill       scans at new places (every point a new voxel, about 179k per scan) until the map holds --target voxels; every
             call timed, so the time of a call that adds 179k voxels is seen from an empty map to the target
  revisit    --calls scans over places already mapped (every voxel exists), at about 1 M voxels and again at the target
  dense      malio_world_accumulate per call on the same fill scans
  save       malio_world_voxel_save_pcd of the full map (in a temporary directory, removed afterwards), and the bytes of the
             voxel map against the dense cloud, on the device and as files: the voxel map's device bytes (malio_world_voxel_info,
             scratch included) after the accumulate calls, after a download (which holds the sort area), after the save (which
             releases it) and after one more accumulate

Every call ends with a stream synchronise, so the host clock around it is its time.  Card name, power limit and max SM clock
are read in the same run.  Prints one JSON line; --out also writes it to that file.

  python tools/world_voxel_perf.py [--target 20000000 --calls 50 --out profiles/h100_world_voxel.json]
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

SIZES = (131072, 24000, 24000)
LEAF = 0.1
STEP = 200.0          # m between fill scans: no voxel shared with the previous scan
Q_ID = np.array([1.0, 0.0, 0.0, 0.0])


def plant(m, slot, xyz):
    """malio_undistort with control points that end before the scan: the slot's cloud is xyz as given."""
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    m.undistort(slot, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), np.array([-10.0, -9.0, -8.0, -7.0]),
                np.tile(np.eye(4), (4, 1, 1)), np.zeros(0), -1)


def state(x):
    return synth.make_state((x, 0.0, 0.0), Q_ID, [Q_ID] * 3, [np.zeros(3)] * 3)


def stats(t):
    t = 1e3 * np.asarray(t)
    return dict(n=int(t.size), median_ms=float(np.median(t)), p90_ms=float(np.percentile(t, 90)), min_ms=float(t.min()),
                max_ms=float(t.max()))


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--target", type=int, default=20_000_000)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.cuda.set_device(0)
    rng = np.random.default_rng(3)
    m = plugin.MeasurementModel(3)
    for l, n in enumerate(SIZES):
        r = 80.0 * np.sqrt(rng.uniform(0, 1, n))
        a = rng.uniform(-np.pi, np.pi, n)
        plant(m, l, np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-2.0, 6.0, n)], axis=1).astype(np.float32))
    tags = np.array([0.0, 1.0, 2.0], np.float32)
    n_scan = sum(SIZES)
    m.voxel_map_accumulate(state(-1e4), tags, LEAF)     # warm-up (first allocations), then a fresh map
    with tempfile.TemporaryDirectory() as d:
        m.voxel_map_save(os.path.join(d, "warm.pcd"), clear=True)

    fill, dense, sizes, revisit = [], [], [], {}
    n_dense = 0
    places = []
    x = 0.0

    def revisit_block(label):
        t = []
        for k in range(args.calls):
            dt, n = timed(lambda: m.voxel_map_accumulate(state(places[k % len(places)]), tags, LEAF))
            t.append(dt)
        revisit[label] = dict(stats(t), n_voxels=n)

    while True:
        s = state(x)
        dt, n = timed(lambda: m.voxel_map_accumulate(s, tags, LEAF))
        fill.append(dt)
        sizes.append(n)
        dt, n_dense = timed(lambda: m.pcd_accumulate(s, tags))
        dense.append(dt)
        places.append(x)
        x += STEP
        if "at_1M" not in revisit and n >= 1_000_000:
            revisit_block("at_1M")
        if n >= args.target:
            break
    revisit_block("at_target")
    info = m.voxel_map_info()                        # after accumulate calls only
    n_vox = info["n_voxels"]
    out = m.voxel_map_tensor()                       # a download: the entry-sized sort area stays until the next save
    torch.cuda.current_stream().synchronize()
    held = m.voxel_map_info()["device_bytes"]
    del out
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "voxels.pcd")
        t_save, _ = timed(lambda: m.voxel_map_save(p, clear=False))
        file_bytes = os.path.getsize(p)
    after_save = m.voxel_map_info()["device_bytes"]
    m.voxel_map_accumulate(state(places[0]), tags, LEAF)   # the next scan regrows its scan-sized scratch
    next_scan = m.voxel_map_info()["device_bytes"]
    k = min(10, len(fill) // 2)
    res = dict(tool="world_voxel_perf", card=card(), points_per_scan=n_scan, leaf=LEAF, scans=len(fill),
               voxels=n_vox, new_voxels_per_fill_scan=int(np.median(np.diff([0] + sizes))),
               fill_first=dict(stats(fill[:k]), map_voxels=[0, sizes[k - 1]]),
               fill_last=dict(stats(fill[-k:]), map_voxels=[sizes[-k - 1], sizes[-1]]),
               revisit=revisit, dense_accumulate=stats(dense),
               save=dict(seconds=t_save, file_bytes=file_bytes),
               bytes=dict(voxel_map_device=info["device_bytes"], voxel_map_device_after_download=held,
                          voxel_map_device_after_save=after_save, voxel_map_device_next_scan=next_scan,
                          voxel_map_entries=n_vox * 32, dense_device=n_dense * 16,
                          dense_file_records=n_dense * 32, voxel_file=file_bytes, dense_points=n_dense))
    m.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
