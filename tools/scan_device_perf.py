"""One C2 scan (3 LiDARs, 100k points against a 1M-point snapshot, bench.py's seeds) through the measurement path, twice per
round on one handle: from and to pinned host arrays (malio_upload_scan, malio_download_aux, malio_map_incremental,
malio_world_register) and from and to torch CUDA tensors (upload_scan_tensor, aux_tensor, map_incremental_tensor,
publish_frame_world_tensor).  A scan = the upload, the IESKF update (malio_ieskf_update, the same host call on both paths), all
five aux outputs, map_incremental with its world points and the down-sampled registration.

The two paths alternate scan by scan.  Per path: the median over --scans scans after --warmup scans of the host clock from the
upload to the end of a synchronise of the current stream (the host calls are synchronous; the output calls on tensors return
after enqueueing), split into upload, update and outputs.  The L2 is not flushed: the scan is the steady state of a mapping
loop.  The outputs of the two paths are compared bit for bit.  Card name, power limit and max SM clock are read in the same
run.  Prints one JSON object; --out also writes it to that file.

  python tools/scan_device_perf.py [--scans 200 --warmup 20 --out profiles/h100_c2_scan_device.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from knn_device_perf import card  # noqa: E402
from malio_b200 import capi, plugin, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.cuda.set_device(0)
    case = synth.case_C2()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    m = plugin.MeasurementModel(case.n_lidar, device=0, params=case.params)
    m.upload_map(snap)
    lib, h = m.lib, m._h
    n = case.pts.shape[0]
    rec_np = np.ascontiguousarray(case.pts).view(np.int32).reshape(n, 4)
    pin = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory()
    hp = {"pts": torch.from_numpy(rec_np.copy()).pin_memory(), "normal_y": pin(n, torch.float32), "nn_idx": pin((n, capi.K), torch.int32),
          "nn_sqdist": pin((n, capi.K), torch.float32), "selected": pin(n, torch.uint8), "world": pin((n, 3), torch.float32),
          "cls": pin(n, torch.uint8), "w": pin((n, 3), torch.float32), "reg": pin((n, 4), torch.float32)}
    rec = torch.from_numpy(rec_np).cuda()
    tab, off, tc = case.table, case.table_off, case.temporal_comp
    last = {}

    def ok(rc):
        if rc != capi.OK:
            raise capi.MalioError(rc, lib.malio_last_error(h).decode())

    def update():
        x, P = case.x_prop.copy(), case.P_prop.copy()
        m.update_iterated_dyn_share_modified(x, P, case.max_iter)
        return x

    def host_scan():
        t0 = time.perf_counter()
        ok(lib.malio_upload_scan(h, hp["pts"].data_ptr(), n, capi.ptr(tab), capi.ptr(off), capi.ptr(tc)))
        m.n_points = n
        t1 = time.perf_counter()
        x = update()
        ps = x.pass_state()
        t2 = time.perf_counter()
        ok(lib.malio_download_aux(h, *(hp[k].data_ptr() for k in ("normal_y", "nn_idx", "nn_sqdist", "selected", "world"))))
        ok(lib.malio_map_incremental(h, C.byref(ps), C.c_double(0.5), 1, hp["cls"].data_ptr(), hp["w"].data_ptr()))
        k = C.c_uint32(0)
        ok(lib.malio_world_register(h, C.byref(ps), capi.WORLD_DOWNSAMPLED, None, hp["reg"].data_ptr(), n, C.byref(k)))
        t3 = time.perf_counter()
        return t1 - t0, t2 - t1, t3 - t2

    def device_scan():
        t0 = time.perf_counter()
        m.upload_scan_tensor(rec, tab, off, tc)
        t1 = time.perf_counter()
        x = update()
        t2 = time.perf_counter()
        last["aux"] = m.aux_tensor()
        last["cls"], last["w"] = m.map_incremental_tensor(x, 0.5, True)
        last["reg"] = m.publish_frame_world_tensor(x, False)
        torch.cuda.current_stream().synchronize()
        t3 = time.perf_counter()
        return t1 - t0, t2 - t1, t3 - t2

    paths = {"host_pinned": host_scan, "device_tensor": device_scan}
    times = {k: [] for k in paths}
    for _ in range(args.warmup):
        for fn in paths.values():
            fn()
    torch.cuda.synchronize()
    for _ in range(args.scans):
        for name, fn in paths.items():
            times[name].append(fn())

    dev = {k: v.cpu() for k, v in last["aux"].items()}
    dev.update(cls=last["cls"].cpu(), w=last["w"].cpu(), reg=last["reg"].cpu())
    same = all(dev[k].numpy().tobytes() == hp[k].numpy().tobytes() for k in dev)
    res = {"what": "one C2 scan (3 LiDARs, 100k points vs a 1M-point snapshot, bench.py's seeds): upload, IESKF update, all aux "
                   "outputs, map_incremental with world points, down-sampled registration",
           "card": card(), "points": n, "map_points": int(case.map_xyz.shape[0]), "scans_per_path": args.scans, "warmup": args.warmup,
           "timing": "host clock, upload to the end of a current-stream synchronise; paths alternate scan by scan; L2 not flushed",
           "paths": {}, "outputs_bit_identical": bool(same)}
    for name, ts in times.items():
        ts = np.array(ts)
        tot = ts.sum(axis=1)
        res["paths"][name] = {"median_ms": float(np.median(tot)) * 1e3, "p10_ms": float(np.percentile(tot, 10)) * 1e3,
                              "p90_ms": float(np.percentile(tot, 90)) * 1e3,
                              "upload_median_ms": float(np.median(ts[:, 0])) * 1e3, "update_median_ms": float(np.median(ts[:, 1])) * 1e3,
                              "outputs_median_ms": float(np.median(ts[:, 2])) * 1e3}
    res["device_minus_host_median_ms"] = res["paths"]["device_tensor"]["median_ms"] - res["paths"]["host_pinned"]["median_ms"]
    m.close()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
