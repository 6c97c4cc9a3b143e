"""Stand-alone k-NN (BASELINE config C5: 1M queries vs a 10M-point map, bench.py's seeds) through three paths on one handle:
malio_knn from pageable host arrays, malio_knn from pinned host arrays, and malio_knn_device on torch CUDA tensors (knn_tensor).

Per path: median wall time of one call over --calls calls after --warmup calls, the host clock running from the call to the end
of a synchronise of the current stream (the host paths are synchronous; the device path returns after enqueueing), and
queries/s = Q / that median.  The L2 is flushed (256 MiB write) and the device synchronised before every timed call, as in
bench.py --config C5.  The paths alternate over --rounds rounds.  The kernel rate is malio_knn's own device time (CUDA events
around the search kernels, after the query sort: what bench.py --config C5 reports) of the host calls in the same run.
--profile adds torch.profiler's device time per kernel over 10 more device-path calls, after the timed ones.  Outputs of the
three paths are compared bit for bit.  Card name, power limit and max SM clock are read in the same run.  Prints one JSON
object; --out also writes it to that file.

  python tools/knn_device_perf.py [--calls 50 --warmup 5 --rounds 3 --profile --out /tmp/knn_device_perf.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from malio_b200 import capi, plugin, synth  # noqa: E402


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().split(",")]
        out.update(smi_name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # the rate is still reported; the missing field says why
        out["smi_error"] = repr(e)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.cuda.set_device(0)
    xyz, q = synth.knn_microbench()
    Q = q.shape[0]
    snap = plugin.build_static_snapshot(xyz)
    m = plugin.MeasurementModel(1, device=0)
    m.upload_map(snap)
    lib, h = m.lib, m._h
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    pg = {"q": q, "idx": np.zeros((Q, capi.K), np.uint32), "d2": np.zeros((Q, capi.K), np.float32)}
    pn = {"q": torch.from_numpy(q).pin_memory(), "idx": torch.zeros((Q, capi.K), dtype=torch.int32).pin_memory(),
          "d2": torch.zeros((Q, capi.K), dtype=torch.float32).pin_memory()}
    qt = torch.from_numpy(q).cuda()
    kernel_ms = []
    out = {}

    def host_call(qp, ip, dp):
        ms = C.c_float(0)
        rc = lib.malio_knn(h, qp, Q, ip, dp, C.byref(ms))
        if rc != capi.OK:
            raise capi.MalioError(rc, lib.malio_last_error(h).decode())
        kernel_ms.append(ms.value)

    def pageable():
        host_call(pg["q"].ctypes.data, pg["idx"].ctypes.data, pg["d2"].ctypes.data)

    def pinned():
        host_call(pn["q"].data_ptr(), pn["idx"].data_ptr(), pn["d2"].data_ptr())

    def device():
        out["dev"] = m.knn_tensor(qt)
        torch.cuda.current_stream().synchronize()

    paths = {"host_pageable": pageable, "host_pinned": pinned, "device_tensor": device}
    times = {k: [] for k in paths}
    for fn in paths.values():
        for _ in range(args.warmup):
            fn()
    kernel_ms.clear()
    for _ in range(args.rounds):
        for name, fn in paths.items():
            for _ in range(args.calls):
                flush.fill_(1)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                times[name].append(time.perf_counter() - t0)
    m.counters()   # folds in the last device call's statistics (and would report its fault)

    di, dd = out["dev"][0].cpu().numpy().view(np.uint32), out["dev"][1].cpu().numpy()
    same = {"host_pinned": bool(np.array_equal(pn["idx"].numpy().view(np.uint32), pg["idx"])
                                and np.array_equal(pn["d2"].numpy().view(np.uint32), pg["d2"].view(np.uint32))),
            "device_tensor": bool(np.array_equal(di, pg["idx"]) and np.array_equal(dd.view(np.uint32), pg["d2"].view(np.uint32)))}
    res = {"what": "stand-alone k-NN, C5 shape: 1M queries vs 10M-point map (synth.knn_microbench, bench.py's seeds), k=5",
           "card": card(), "queries": Q, "map_points": int(xyz.shape[0]), "calls_per_round": args.calls, "rounds": args.rounds,
           "warmup": args.warmup, "l2": "flushed (256 MiB write) and device synchronised before every timed call",
           "paths": {}, "bit_identical_to_host_pageable": same}
    for name, ts in times.items():
        ts = np.array(ts)
        per_round = [float(np.median(ts[r * args.calls:(r + 1) * args.calls])) for r in range(args.rounds)]
        med = float(np.median(ts))
        res["paths"][name] = {"median_ms": med * 1e3, "queries_per_s": Q / med, "p10_ms": float(np.percentile(ts, 10)) * 1e3,
                              "p90_ms": float(np.percentile(ts, 90)) * 1e3, "round_median_ms": [t * 1e3 for t in per_round]}
    kms = float(np.median(kernel_ms))
    res["kernel"] = {"median_ms": kms, "queries_per_s": Q / (kms * 1e-3),
                     "what": "malio_knn's device time (CUDA events around the search kernels, the query sort excluded) of the host calls above"}
    res["device_path_over_kernel_rate"] = res["paths"]["device_tensor"]["queries_per_s"] / res["kernel"]["queries_per_s"]
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        n_prof = 10
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                flush.fill_(1)
                torch.cuda.synchronize()
                device()
        rows = [(e.key, e.device_time_total / n_prof, e.count // n_prof) for e in prof.key_averages()]
        rows = [r for r in rows if "fill" not in r[0] and r[1] > 0]
        res["profile_device_path"] = {"what": f"torch.profiler device time per call (us), mean of {n_prof} knn_tensor calls, L2 flushed",
                                      "kernels": {k: {"us": us, "launches": c} for k, us, c in sorted(rows, key=lambda r: -r[1])}}
    m.close()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
