"""Timing of the stages before the hot path (SURVEY.md §8f N2, N3, N4) on the GPU: malio_undistort / malio_voxel_grid /
malio_upload_scan_device through the C-ABI with HOST buffers (copies inside the timed region) next to the CPU oracle
(oracle/oracle_undistort.cpp, one thread: UndistortPcl's point loop and pcl::VoxelGrid are serial in the reference), and
the .bin reader (host code) on a synthetic City-format file.  Prints one JSON line per stage.  Not a bench value: context for DESIGN.md."""
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyoracle as po                                   # noqa: E402
from malio_b200 import capi, plugin, synth, dataset     # noqa: E402


def best_of(f, reps=7, warm=2):
    for _ in range(warm):
        f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), 1e3 * float(np.min(ts))


def main():
    m = plugin.MeasurementModel(3)
    # raw scan sizes of the City rig at 10 Hz: Ouster OS1-128 (128 x 1024), Livox Avia and Tele (24k each)
    for name, n, lidar in (("ouster 131072 pts", 131072, 0), ("livox 24000 pts", 24000, 1)):
        c = synth.undistort_case(n, lidar=lidar, imu_hz=200.0)
        ok, q, p = po.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], c["end_time"])
        lt = (q, p)
        args = (c["pts"], c["beg_time"], c["extrinsic"], lt, c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
        g_med, g_min = best_of(lambda: m.undistort(lidar, *args))
        o_med, o_min = best_of(lambda: po.undistort(*args, want_pose=False), reps=3, warm=1)
        ctr0 = m.counters()
        m.undistort(lidar, *args)
        ctr1 = m.counters()
        print(json.dumps({"stage": "N2 undistort", "input": name, "gpu_ms_median": g_med, "gpu_ms_min": g_min,
                          "cpu_oracle_ms_median": o_med, "cpu_threads": 1, "speedup": o_med / g_med,
                          "h2d_bytes": int(ctr1.h2d_bytes - ctr0.h2d_bytes), "d2h_bytes": int(ctr1.d2h_bytes - ctr0.d2h_bytes),
                          "kernel_launches": int(ctr1.kernel_launches - ctr0.kernel_launches),
                          "what": "C-ABI call with host buffers: H2D points + control points, seglog + undistort kernels, D2H xyz/idx/ok/pop list"}))
        # N3 on the un-down-sampled cloud of the same size
        rng = np.random.default_rng(5)
        p5 = np.zeros((n, 5), np.float32)
        p5[:, :3] = c["pts"]["xyz"]
        p5[:, 3] = rng.integers(0, 20, n)
        p5[:, 4] = c["pts"]["curvature"]
        p8 = np.zeros((n, 8), np.float32)
        p8[:, :4] = p5[:, :4]; p8[:, 7] = p5[:, 4]
        g_med, g_min = best_of(lambda: m.voxel_grid(lidar, p5, 0.5))
        o_med, o_min = best_of(lambda: po.voxel_grid(p8, 0.5), reps=3, warm=1)
        out = m.voxel_grid(lidar, p5, 0.5)
        print(json.dumps({"stage": "N3 voxel grid (leaf 0.5 m)", "input": name, "output_points": int(out.shape[0]),
                          "gpu_ms_median": g_med, "gpu_ms_min": g_min, "cpu_oracle_ms_median": o_med, "cpu_threads": 1,
                          "speedup": o_med / g_med,
                          "what": "plugin.voxel_grid = two C-ABI calls (count, then fetch): H2D cloud, bounds/count/scan/scatter/rank/centroid kernels, D2H centroids"}))
    # the device-resident chain for the 3-LiDAR rig: undistort x3 -> voxel grid x3 (no host bounce) -> merged scan
    case = synth.make_case("chain", 1000, 120000, 3, 3)
    cs = [synth.undistort_case(n, lidar=l, seed=60 + l) for l, n in enumerate((131072, 24000, 24000))]
    lts = []
    for c in cs:
        ok, q, p = po.bspline_get_pose(c["ctrl_t"], c["ctrl_T"], c["end_time"])
        lts.append((q, p))

    def chain():
        for l, c in enumerate(cs):
            m.undistort(l, c["pts"], c["beg_time"], c["extrinsic"], lts[l], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"])
            mm = capi.C.c_uint32(0)
            m._check(m.lib.malio_voxel_grid(m._h, l, None, 0, capi.C.c_float(0.5), None, 0, capi.C.byref(mm)))
        return m.upload_scan_device(case.table, case.table_off, case.temporal_comp)

    g_med, g_min = best_of(chain)
    n_out = chain()

    def cpu_chain():
        for l, c in enumerate(cs):
            o = po.undistort(c["pts"], c["beg_time"], c["extrinsic"], lts[l], c["ctrl_t"], c["ctrl_T"], c["imu_cov_t"], c["cov_pointer"], want_pose=False)
            o8 = np.zeros((c["pts"].shape[0], 8), np.float32)
            o8[:, :3] = o["xyz"]; o8[:, 7] = c["pts"]["curvature"]
            po.voxel_grid(o8, 0.5)

    o_med, _ = best_of(cpu_chain, reps=3, warm=1)
    print(json.dumps({"stage": "N2+N3 chain, 3 LiDARs (131072 + 24000 + 24000 raw points) -> merged device-resident scan",
                      "merged_points": int(n_out), "gpu_ms_median": g_med, "gpu_ms_min": g_min, "cpu_oracle_ms_median": o_med,
                      "cpu_threads": 1, "speedup": o_med / g_med}))
    m.close()
    # N4: the reader + handler on a synthetic City-format Ouster file (22 B records)
    import np_dataset as nd
    with tempfile.TemporaryDirectory() as td:
        rng = np.random.default_rng(1)
        n = 131072
        rec = np.zeros(n, dtype=nd.OUSTER_REC)
        for f in ("x", "y", "z"):
            rec[f] = rng.uniform(-50, 50, n).astype(np.float32)
        rec["intensity"] = rng.uniform(0, 255, n).astype(np.float32)
        rec["ring"] = rng.integers(0, 128, n)
        rec["t"] = np.sort(rng.integers(0, 100_000_000, n)).astype(np.uint32)
        path = os.path.join(td, "ouster.bin")
        rec.tofile(path)
        t_med, _ = best_of(lambda: dataset.read_ouster_bin(path), reps=5, warm=1)
        pts = dataset.read_ouster_bin(path)
        h_med, _ = best_of(lambda: dataset.preprocess_ouster(pts, 1, 0.5), reps=5, warm=1)
        print(json.dumps({"stage": "N4 read_ouster_bin + oust64_handler", "records": n, "bytes": int(os.path.getsize(path)),
                          "read_ms_median": t_med, "handler_ms_median": h_med,
                          "read_GBps": os.path.getsize(path) / (t_med * 1e-3) / 1e9}))


if __name__ == "__main__":
    main()
