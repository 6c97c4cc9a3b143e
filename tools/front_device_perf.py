"""The front half of one scan at the City rig's sizes (raw clouds of 131 072 + 24 000 + 24 000 points, synth.undistort_case,
one shared spline and IMU list) — three undistortions, the scan's pose-uncertainty table, three voxel grids (leaf 0.5) and the
upload of the merged scan — through three paths, each on its own handle:

  host_pageable   malio_undistort / malio_scan_uncertainty / malio_voxel_grid / malio_upload_scan_device on pageable arrays
  host_pinned     the same calls on pinned arrays
  device_tensor   malio_undistort_device / malio_scan_uncertainty_resident / malio_voxel_grid_device / malio_upload_scan_resident
                  on torch CUDA tensors, the table never leaving the device

No path asks for per-point outputs (the undistortion returns its pop points only, the voxel grid its count): what is timed is
what a mapping loop needs.  Two IMU-list sizes: 39 entries and 512 entries with 512 control points (the library's maxima).

The paths alternate scan by scan.  Per path: median, p10 and p90 over --scans scans after --warmup scans of the host clock from
the first call to the end of a synchronise of the current stream, and the median of every stage (host clock to the call's
return: the host calls are synchronous, malio_voxel_grid_device returns with its last kernel enqueued).  The L2 is not flushed.
After the timed scans the paths' results are compared bit for bit: the dense registered cloud (every undistorted point), the
down-sampled clouds, table_off, the temporal compensations and the merged size.  Card name, power limit and max SM clock are
read in the same run.  Prints one JSON line per path and list size, then a summary line; --out also writes them to that file.

  python tools/front_device_perf.py [--scans 100 --warmup 10 --out profiles/h100_front_device.json]
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

SIZES = (131072, 24000, 24000)
LEAF = 0.5
STAGES = ("undistort", "scan_uncertainty", "voxel_grid", "upload")


def make_scan(kw, seed=7):
    """L slots sharing slot 0's spline and IMU list, LiDAR l ending 10 ms x l before LiDAR 0; lt = the spline pose at the
    slot's scan end through the library's host code."""
    rng = np.random.default_rng(seed)
    slots = []
    for l, n in enumerate(SIZES):
        c = synth.undistort_case(n, lidar=l, seed=seed + l, **kw)
        if l:
            base = slots[0]
            c = dict(c, ctrl_t=base["ctrl_t"], ctrl_T=base["ctrl_T"], imu_cov_t=base["imu_cov_t"], end_time=base["end_time"] - 0.01 * l)
            cp = int(np.searchsorted(c["imu_cov_t"], c["end_time"], side="right"))      # IMU_Processing.hpp:455-466
            c["cov_pointer"] = min(cp, c["imu_cov_t"].shape[0] - 1)
        ok, q, p = plugin.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], c["end_time"])
        assert ok
        c["lt"] = (q, p)
        slots.append(c)

    def cov(k):
        A = rng.normal(0, 1, (k, 6, 6))
        return A @ A.transpose(0, 2, 1) * 1e-4 + np.eye(6) * 1e-6

    ext = np.zeros(len(slots), capi.POSE)
    lib = capi.load()
    for l, c in enumerate(slots):
        lib.malio_pose_initial(ext[l:l + 1].ctypes.data, capi.ptr(np.ascontiguousarray(c["extrinsic"][1], np.float64)),
                               capi.ptr(np.ascontiguousarray(c["extrinsic"][0], np.float64)), capi.ptr(cov(1).reshape(36)))
    return slots, cov(slots[0]["imu_cov_t"].shape[0]), ext, cov(1)[0]


class Path:
    def __init__(self, name, slots, imu_cov, ext, unc):
        self.name = name
        self.L = len(slots)
        self.m = plugin.MeasurementModel(self.L, device=0)
        self.lib, self.h = self.m.lib, self.m._h
        self.keep = []
        self.ud = []
        for c in slots:
            a, cv, keep = plugin._undistort_args(c["beg_time"], c["extrinsic"], c["lt"], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
            self.keep.append(keep + (cv,))
            self.ud.append(a)
        self.sa, keep = plugin._scan_unc_args(imu_cov, ext, unc)
        self.keep.append(keep)
        self.k = C.c_uint32(0)
        self.times = []

    def ok(self, rc):
        if rc != capi.OK:
            raise capi.MalioError(rc, self.lib.malio_last_error(self.h).decode())

    def scan(self):
        t = [time.perf_counter()]
        self.undistort(); t.append(time.perf_counter())
        self.scan_uncertainty(); t.append(time.perf_counter())
        self.voxel_grid(); t.append(time.perf_counter())
        self.upload(); t.append(time.perf_counter())
        torch.cuda.current_stream().synchronize()
        t.append(time.perf_counter())
        return [t[i + 1] - t[i] for i in range(4)] + [t[5] - t[0]]


class HostPath(Path):
    def __init__(self, name, slots, imu_cov, ext, unc, pinned):
        super().__init__(name, slots, imu_cov, ext, unc)
        buf = (lambda a: torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).pin_memory()) if pinned else \
              (lambda a: torch.from_numpy(a.view(np.uint8).reshape(-1).copy()))
        self.raw = [buf(np.ascontiguousarray(c["pts"])) for c in slots]
        self.n = [c["pts"].shape[0] for c in slots]
        self.pop = [buf(np.zeros(capi.MAX_COV, np.int32)) for _ in slots]
        self.cap = self.L * capi.MAX_COV
        self.table = buf(np.zeros(self.cap, capi.POSE_ENTRY))
        self.off = buf(np.zeros(self.L + 1, np.uint32))
        self.tc = buf(np.zeros(self.L - 1, capi.POSE))
        self.rigid = np.zeros(self.L - 1, capi.RIGID)

    def undistort(self):
        for l in range(self.L):
            self.ok(self.lib.malio_undistort(self.h, l, self.raw[l].data_ptr(), self.n[l], C.byref(self.ud[l]), None, None, None,
                                             self.pop[l].data_ptr(), C.byref(self.k), None))

    def scan_uncertainty(self):
        self.ok(self.lib.malio_scan_uncertainty(self.h, C.byref(self.sa), self.table.data_ptr(), self.cap, self.off.data_ptr(),
                                                self.tc.data_ptr(), None, None))
        tc = self.tc.numpy().view(capi.POSE)
        self.rigid["q"], self.rigid["t"] = tc["q"], tc["t"]

    def voxel_grid(self):
        for l in range(self.L):
            self.ok(self.lib.malio_voxel_grid(self.h, l, None, 0, C.c_float(LEAF), None, 0, C.byref(self.k)))

    def upload(self):
        self.ok(self.lib.malio_upload_scan_device(self.h, self.table.data_ptr(), self.off.data_ptr(), capi.ptr(self.rigid), C.byref(self.k)))

    def results(self):
        return dict(off=self.off.numpy().view(np.uint32).copy(), tc=self.tc.numpy().view(capi.POSE).copy(), n=int(self.k.value),
                    down=[self.m.voxel_grid(l, None, LEAF) for l in range(self.L)])


class TensorPath(Path):
    def __init__(self, name, slots, imu_cov, ext, unc):
        super().__init__(name, slots, imu_cov, ext, unc)
        self.raw = [torch.from_numpy(np.ascontiguousarray(c["pts"]).view(np.float32).reshape(-1, 4)).cuda() for c in slots]
        self.off = np.zeros(self.L + 1, np.uint32)
        self.tc = np.zeros(self.L - 1, capi.POSE)
        self.st = torch.cuda.current_stream().cuda_stream

    def undistort(self):
        for l in range(self.L):
            self.ok(self.lib.malio_undistort_device(self.h, l, self.raw[l].data_ptr(), self.raw[l].shape[0], C.addressof(self.ud[l]), None,
                                                    None, None, None, None, C.addressof(self.k), self.st))

    def scan_uncertainty(self):
        self.ok(self.lib.malio_scan_uncertainty_resident(self.h, C.addressof(self.sa), capi.ptr(self.off), capi.ptr(self.tc)))

    def voxel_grid(self):
        for l in range(self.L):
            self.ok(self.lib.malio_voxel_grid_device(self.h, l, None, 0, C.c_float(LEAF), None, 0, C.addressof(self.k), self.st))

    def upload(self):
        self.ok(self.lib.malio_upload_scan_resident(self.h, C.addressof(self.k)))

    def results(self):
        self.m._slot_rows = {l: r.shape[0] for l, r in enumerate(self.raw)}
        return dict(off=self.off.copy(), tc=self.tc.copy(), n=int(self.k.value),
                    down=[self.m.voxel_grid_tensor(l, None, LEAF).cpu().numpy() for l in range(self.L)])


def run(label, kw, args):
    slots, imu_cov, ext, unc = make_scan(kw)
    paths = [HostPath("host_pageable", slots, imu_cov, ext, unc, False), HostPath("host_pinned", slots, imu_cov, ext, unc, True),
             TensorPath("device_tensor", slots, imu_cov, ext, unc)]
    for _ in range(args.warmup):
        for p in paths:
            p.scan()
    torch.cuda.synchronize()
    for _ in range(args.scans):
        for p in paths:
            p.times.append(p.scan())
    # the same results on every path, bit for bit
    x = synth.make_state([0, 0, 0], [1, 0, 0, 0], [c["extrinsic"][0] for c in slots], [c["extrinsic"][1] for c in slots])
    tags = np.arange(len(slots), dtype=np.float32)
    res = []
    for p in paths:
        r = p.results()
        r["dense"] = p.m.publish_frame_world(x, True, tags)
        res.append(r)
    same = all(r["n"] == res[0]["n"] and r["off"].tobytes() == res[0]["off"].tobytes() and r["tc"].tobytes() == res[0]["tc"].tobytes() and
               r["dense"].tobytes() == res[0]["dense"].tobytes() and
               all(a.tobytes() == b.tobytes() for a, b in zip(r["down"], res[0]["down"])) for r in res[1:])
    lines = []
    for p in paths:
        ts = np.array(p.times) * 1e3
        line = {"path": p.name, "imu_list": label, "n_cov": int(imu_cov.shape[0]), "n_ctrl": int(slots[0]["ctrl_t"].shape[0]),
                "table_entries": int(res[0]["off"][-1]), "raw_points": list(SIZES), "scan_points": res[0]["n"],
                "median_ms": float(np.median(ts[:, 4])), "p10_ms": float(np.percentile(ts[:, 4], 10)), "p90_ms": float(np.percentile(ts[:, 4], 90)),
                "stage_median_ms": {s: float(np.median(ts[:, i])) for i, s in enumerate(STAGES)}, "scans": args.scans, "warmup": args.warmup}
        lines.append(line)
        p.m.close()
    return lines, bool(same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures on the GPU only")
    torch.cuda.set_device(0)
    out, same = [], {}
    for label, kw in (("39", dict(imu_hz=325.0)), ("512", dict(lists="max", imu_hz=4000.0))):
        lines, same[label] = run(label, kw, args)
        out += lines
    med = {(l["path"], l["imu_list"]): l["median_ms"] for l in out}
    out.append({"summary": "front half of one City-size scan", "card": card(), "leaf": LEAF,
                "timing": "host clock, first call to the end of a current-stream synchronise; paths alternate scan by scan; L2 not flushed",
                "results_bit_identical": same,
                "device_minus_pinned_median_ms": {k: med[("device_tensor", k)] - med[("host_pinned", k)] for k in same},
                "device_minus_pageable_median_ms": {k: med[("device_tensor", k)] - med[("host_pageable", k)] for k in same}})
    text = "\n".join(json.dumps(l) for l in out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    if not all(same.values()):
        raise SystemExit("the paths' results differ")


if __name__ == "__main__":
    main()
