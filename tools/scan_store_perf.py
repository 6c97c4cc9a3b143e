"""Time the scan store and the voxel map's rebuild (malio_scan_store_add, malio_world_voxel_rebuild) on City-size scans, and write
profiles/h100_scan_store.json:
  - malio_scan_store_add per scan and the store's bytes per scan;
  - a plain rebuild of 200 and 1000 stored scans at 0.2 m and 0.1 m, against the median per-scan time of
    malio_world_voxel_accumulate on the same scans in the same run;
  - a carved rebuild (the default carve arguments) of 200 scans at 0.2 m and 0.1 m and of 1000 scans at 0.2 m, against the
    median per-scan time of malio_world_voxel_accumulate_carve.
The scans: DISTINCT synth.street_scan_city scans of the street drive; stored scan k is distinct scan k % DISTINCT, stored with
the state of drive position k (the street continues along x), so a store of 1000 scans maps 500 m of street.  Each rebuild
runs on a fresh handle whose store was filled with malio_scan_store_put, and is timed once with the host clock around the call
(it ends in its own wait), after a warm-up rebuild on another handle.  The card's name and power limit are read in the same run.
  python tools/scan_store_perf.py [--distinct 20 --out profiles/h100_scan_store.json]
"""
import argparse
import ctypes as C
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
from world_carve_perf import plant, stats  # noqa: E402

L = 3
TAGS = np.arange(L, dtype=np.float32)


def state_at(street, rec, j, k):
    """Scan j's stored state moved to drive position k."""
    s = capi.PassState()
    C.memmove(C.byref(s), C.byref(rec.state), C.sizeof(capi.PassState))
    s.pos[0] += street.ego_step * (k - j)
    return s


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--distinct", type=int, default=20)
    ap.add_argument("--baseline-scans", type=int, default=100)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_scan_store.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scan_store_perf: no CUDA device (nothing is measured without one)")
    street = synth.Street()
    scans = [synth.street_scan_city(street, k) for k in range(a.distinct)]
    res = dict(card=card(), distinct_scans=a.distinct, L=L)

    # add: plant each distinct scan, time the add (it returns after enqueueing; the time includes the copy's completion)
    m = plugin.MeasurementModel(L)
    add_ms = []
    for k, sc in enumerate(scans):
        for l in range(L):
            plant(m, l, np.asarray(sc["body"][l], np.float32))
        _, ms = timed(lambda: m.scan_store_add(sc["state"], TAGS, time=0.1 * k))
        add_ms.append(ms)
    recs, pts = zip(*[m.scan_store_get(k) for k in range(a.distinct)])
    info = m.scan_store_info()
    m.close()
    n_pts = [p.shape[0] for p in pts]
    res["add"] = dict(stats(add_ms[2:]), points_per_scan_mean=float(np.mean(n_pts)),
                      store_bytes_per_scan=float(np.mean(n_pts)) * 12 + C.sizeof(capi.StoredScan),
                      record_bytes=C.sizeof(capi.StoredScan), block_bytes_after=int(info["device_bytes"]))

    def store(n):
        h = plugin.MeasurementModel(L)
        for k in range(n):
            j = k % a.distinct
            rec = capi.StoredScan.from_buffer_copy(bytes(recs[j]))
            rec.state = state_at(street, recs[j], j, k)
            rec.time = 0.1 * k
            h.scan_store_put(rec, pts[j])
        return h

    def baseline(leaf, carve, n):
        h = plugin.MeasurementModel(L)
        ms = []
        for k in range(n):
            j = k % a.distinct
            for l in range(L):
                plant(h, l, np.asarray(scans[j]["body"][l], np.float32))
            s = state_at(street, recs[j], j, k)
            _, t = timed(lambda: h.voxel_map_accumulate(s, TAGS, leaf, carve=carve))
            ms.append(t)
        nv = h.voxel_map_info()["n_voxels"]
        h.close()
        return dict(stats(ms[2:]), scans=n, n_voxels_after=nv)

    w = store(a.distinct)   # warm-up: modules, CUB's algorithms
    w.voxel_map_rebuild(0.2)
    with tempfile.TemporaryDirectory() as d:
        w.voxel_map_save(os.path.join(d, "warm.pcd"), clear=True)
    w.voxel_map_rebuild(0.2, carve=True)
    w.close()

    res["plain"], res["carved"], res["accumulate"], res["accumulate_carve"] = [], [], {}, {}
    for leaf in (0.2, 0.1):
        res["accumulate"][str(leaf)] = baseline(leaf, None, a.baseline_scans)
        res["accumulate_carve"][str(leaf)] = baseline(leaf, True, a.baseline_scans)
    for carve, configs in ((None, ((200, 0.2), (1000, 0.2), (200, 0.1), (1000, 0.1))), (True, ((200, 0.2), (200, 0.1), (1000, 0.2)))):
        for n, leaf in configs:
            h = store(n)
            nv, ms = timed(lambda: h.voxel_map_rebuild(leaf, carve=carve))
            base = res["accumulate_carve" if carve else "accumulate"][str(leaf)]["median_ms"]
            row = dict(scans=n, leaf=leaf, rows=int(h.scan_store_info()["n_points"]), ms=ms, ms_per_scan=ms / n,
                       accumulate_median_ms_per_scan=base, speedup_per_scan=base / (ms / n), n_voxels=nv,
                       map_device_bytes=h.voxel_map_info()["device_bytes"], store_device_bytes=h.scan_store_info()["device_bytes"])
            (res["carved"] if carve else res["plain"]).append(row)
            print(json.dumps(row), flush=True)
            h.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(dict(card=res["card"], add=res["add"])))


if __name__ == "__main__":
    main()
