"""Time the 2-D occupancy grid (malio_grid_build_device) at the sizes a user exports, and write profiles/h100_grid.json:
  - the kept voxel map of the carve perf scenes (tools/world_carve_perf.py's fill: 1.4 M voxels at 0.2 m, 21.5 M at 0.1 m, then
    carved street scans), gridded in place over its whole extent at 0.1 m;
  - synth.make_world's 26 M-point prior over its whole extent at 0.1 m and 0.05 m (a raster above MALIO_GRID_MAX_BYTES is
    exported in equal tiles, which stitch without seams; the time is the whole export);
  - each call's peak scratch bytes and the PGM / YAML write of the largest raster.
Time per call is the host clock around the call, which ends in its own wait; medians and p90 over --reps after --warmup.
The card's name and power limit are read in the same run.
  python tools/grid_perf.py [--reps 10 --warmup 2 --out profiles/h100_grid.json]
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
from world_carve_perf import Q_ID, plant, stats  # noqa: E402

MAP_CONFIGS = ((0.2, 1_000_000), (0.1, 20_000_000))
PRIOR_POINTS = 26_000_000


def timed(fn, reps, warmup):
    out, ms = None, []
    for k in range(warmup + reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        dt = (time.perf_counter() - t0) * 1e3
        if k >= warmup:
            ms.append(dt)
    return out, stats(ms)


def tiled(m, source, keep, res, tiles):
    """The grid of the whole extent in tiles x tiles equal regions (the last ones take the remainder): peak scratch, cells."""
    lo_i, lo_j, hi_i, hi_j = m.grid_extent(source, keep=keep, res=res)
    nx, ny = hi_i - lo_i + 1, hi_j - lo_j + 1
    peak, occ = 0, 0
    for ti in range(tiles):
        for tj in range(tiles):
            i0, j0 = lo_i + ti * (nx // tiles), lo_j + tj * (ny // tiles)
            tnx = nx // tiles if ti < tiles - 1 else nx - (tiles - 1) * (nx // tiles)
            tny = ny // tiles if tj < tiles - 1 else ny - (tiles - 1) * (ny // tiles)
            cls, _, rep = m.grid(source, keep=keep, args=plugin.grid_args(res, i0, j0, tnx, tny))
            peak, occ = max(peak, rep["device_bytes"]), occ + rep["n_occupied"]
    return dict(nx=nx, ny=ny, tiles=tiles, peak_scratch_bytes=peak, occupied=occ, last=cls)


def fits(m, source, keep, res):
    """The fewest tiles per axis whose largest tile stays under MALIO_GRID_MAX_BYTES."""
    lo_i, lo_j, hi_i, hi_j = m.grid_extent(source, keep=keep, res=res)
    nx, ny, w = hi_i - lo_i + 1, hi_j - lo_j + 1, plugin.GRID_GROUND_HALFWIDTH
    t = 1
    while True:
        tx, ty = nx - (t - 1) * (nx // t), ny - (t - 1) * (ny // t)
        if 4 * ((tx + 2 * w) * (ty + 2 * w) + tx * (ty + 2 * w) + tx * ty) + 64 + tx * ty * 5 <= capi.GRID_MAX_BYTES:
            return t
        t += 1


def voxel_map_run(leaf, fill, reps, warmup):
    st = synth.Street()
    L = 3
    tags = np.zeros(L, np.float32)
    m = plugin.MeasurementModel(L)
    rng = np.random.default_rng(7)
    s0 = synth.make_state([0.0, 0.0, 0.0], Q_ID, [Q_ID] * L, [np.zeros(3)] * L)
    chunk = 1 << 17
    for c in range(0, int(fill * 1.05), chunk):
        pre = rng.uniform([-150, -40, -2], [350, 40, 30], (chunk, 3)).astype(np.float32)
        plant(m, 0, pre)
        for l in (1, 2):
            plant(m, l, np.zeros((0, 3), np.float32))
        m.voxel_map_accumulate(s0, tags, leaf)
    for k in range(5):
        sc = synth.street_scan_city(st, k)
        for l in range(L):
            plant(m, l, sc["body"][l])
        m.voxel_map_accumulate(sc["state"], tags, leaf, carve=True)
    info0 = m.voxel_map_info()
    res = 0.1
    t = fits(m, "voxel_map", True, res)
    r, tm = timed(lambda: tiled(m, "voxel_map", True, res, t), reps, warmup)
    r.pop("last")
    out = dict(source="voxel_map kept", leaf=leaf, voxels=info0["n_voxels"], res=res, grid=r, call=tm,
               handle_bytes_unchanged=m.voxel_map_info() == info0)
    m.close()
    return out


def prior_run(reps, warmup):
    m = plugin.MeasurementModel(1)
    xyz = synth.make_world(PRIOR_POINTS)
    m.prior_map_load(xyz)
    out = []
    for res in (0.1, 0.05):
        t = fits(m, "prior", None, res)
        r, tm = timed(lambda: tiled(m, "prior", None, res, t), reps, warmup)
        last = r.pop("last")
        out.append(dict(source="prior", points=int(xyz.shape[0]), res=res, grid=r, call=tm))
    with tempfile.TemporaryDirectory() as d:
        c = last.cpu().numpy()
        a = plugin.grid_args(0.05, 0, 0, c.shape[1], c.shape[0])
        t0 = time.perf_counter()
        plugin.save_grid(os.path.join(d, "map"), c, a)
        pgm_ms = (time.perf_counter() - t0) * 1e3
    m.close()
    return out, dict(cells=int(c.size), write_ms=pgm_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    runs = [voxel_map_run(leaf, fill, a.reps, a.warmup) for leaf, fill in MAP_CONFIGS]
    pr, pgm = prior_run(a.reps, a.warmup)
    out = dict(tool="grid_perf", card=card(), defaults=dict(res=plugin.GRID_RES, w=plugin.GRID_GROUND_HALFWIDTH, h_lo=plugin.GRID_H_LO,
               h_hi=plugin.GRID_H_HI, m=plugin.GRID_MIN_OBSTACLE_POINTS), runs=runs + pr, pgm_write=pgm)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
