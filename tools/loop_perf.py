"""Time loop closure over the scan store and write profiles/h100_loop.json:
  - malio_scan_store_match of a City-size scan (synth.street_scan_city, 3 slots) against submaps of 5, 21 and 41 stored scans:
    the whole call at the default three levels (leaves 2.0, 1.0, 0.5 m), and per leaf the model build and the time per
    Gauss-Newton iteration.  Per leaf, a one-level call runs max_iter = 1 and max_iter = K with ends it cannot meet
    (eps = 1e-300): one iteration costs (T_K - T_1) / (K - 1), the model build T_1 - 2 iterations (a call with one step runs
    two evaluations: the step's and the report's);
  - malio_pose_graph_optimize (host) at n = 1 000 and 20 000 nodes with m = 16 and 256 loop edges.
Stored scan k is the City-size scan at drive position k (each scan cast on its own); the source is the scan after the submap,
its guess the true state moved by 0.3 m and 1 degree.  Each row reports the match's result and plugin.accept_edge's verdict.  Each time is the host clock around
one call (each ends in its own wait), repeated; median and p90.  The card's name and power limit are read in the same run.
  python tools/loop_perf.py [--reps 10 --out profiles/h100_loop.json]
"""
import argparse
import ctypes as C
import json
import math
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
from world_carve_perf import stats  # noqa: E402

L = 3


def record(sc):
    rec = capi.StoredScan()
    s = sc["state"].pass_state() if isinstance(sc["state"], capi.State) else sc["state"]
    C.memmove(C.byref(rec.state), C.byref(s), C.sizeof(capi.PassState))
    for i in range(L - 1):
        rec.temporal_comp[i].q[0] = 1.0
    for l in range(L):
        rec.slot_tag[l] = l
        rec.n_points[l] = sc["body"][l].shape[0]
    return rec


def timed(fn, reps):
    out, ms = None, []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    return out, ms


def graph(n, m, rng):
    qs, ps = [np.array([1.0, 0, 0, 0])], [np.zeros(3)]
    for _ in range(n - 1):
        dq = np.array([1.0, *rng.normal(scale=0.02, size=3)])
        q = synth.q_mul(qs[-1], dq / np.linalg.norm(dq))
        qs.append(q / np.linalg.norm(q))
        ps.append(ps[-1] + synth.q_to_R(qs[-2]) @ np.array([0.5, *rng.normal(scale=0.05, size=2)]))
    states = []
    for q, p in zip(qs, ps):
        s = capi.PassState()
        s.rot[:], s.pos[:] = list(q), list(p)
        states.append(s)
    edges = []
    for _ in range(m):
        a = int(rng.integers(0, n - n // 10))
        b = int(rng.integers(a + n // 20, n))
        e = capi.PoseEdge()
        e.a, e.b = a, b
        qa = qs[a]
        qa_c = np.array([qa[0], -qa[1], -qa[2], -qa[3]])
        e.rot[:] = list(synth.q_mul(qa_c, qs[b]))
        e.pos[:] = list(synth.q_to_R(qa).T @ (ps[b] - ps[a]) + rng.normal(scale=0.05, size=3))
        M = rng.normal(size=(6, 6))
        e.info[:] = list((M @ M.T + 1e3 * np.eye(6)).reshape(36))
        edges.append(e)
    return states, edges


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_loop.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loop_perf: no CUDA device (nothing is measured without one)")
    street = synth.Street()
    scans = [synth.street_scan_city(street, k) for k in range(42)]
    res = dict(card=card(), reps=a.reps, points_per_scan=[int(sum(b.shape[0] for b in s["body"])) for s in scans],
               match=[], pose_graph=[])
    for window in (5, 21, 41):
        m = plugin.MeasurementModel(L)
        for k in range(window + 1):
            m.scan_store_put(record(scans[k]), np.concatenate(scans[k]["body"]).astype(np.float32))
        src = window
        truth = m.scan_store_records()[src].state
        g = capi.PassState()
        C.memmove(C.byref(g), C.byref(truth), C.sizeof(capi.PassState))
        yaw = math.radians(1.0)
        g.rot[:] = list(synth.q_mul(np.array([math.cos(yaw / 2), 0, 0, math.sin(yaw / 2)]), np.array(truth.rot[:])))
        g.pos[0] += 0.3
        anchor = window // 2
        call = lambda **kw: m.scan_store_match(src, anchor, g, target_first=0, target_count=window, **kw)
        call()   # warm-up
        rep, ms = timed(call, a.reps)
        row = dict(submap_scans=window, target_points=rep["target_points"], device_bytes=rep["device_bytes"],
                   iterations=rep["iterations"], converged=rep["converged"], fitness=rep["fitness"], rms=rep["rms"],
                   n_inliers=rep["n_inliers"], eig_min=rep["eig_min"], constraint=plugin.constraint(rep),
                   accepted=plugin.accept_edge(rep),
                   pos_error_m=float(np.abs(rep["pos"] - np.array(truth.pos[:])).max()), call=stats(ms), levels=[])
        for leaf, gate in zip(plugin.MATCH_LEAF, plugin.MATCH_GATE):
            _, t1 = timed(lambda: call(leaf=(leaf,), gate=(gate,), max_iter=1, eps_rot=1e-300, eps_pos=1e-300), a.reps)
            _, tk = timed(lambda: call(leaf=(leaf,), gate=(gate,), max_iter=a.iters, eps_rot=1e-300, eps_pos=1e-300), a.reps)
            it = (np.median(tk) - np.median(t1)) / (a.iters - 1)
            row["levels"].append(dict(leaf=leaf, one_step_call=stats(t1), iter_ms=float(it), model_build_ms=float(np.median(t1) - 2 * it),
                                      plane_voxels=call(leaf=(leaf,), gate=(gate,), max_iter=1)["target_voxels"][0]))
        res["match"].append(row)
        print(json.dumps(row))
        m.close()
    rng = np.random.default_rng(0)
    for n in (1000, 20000):
        for mm in (16, 256):
            states, edges = graph(n, mm, rng)
            ms = []
            for _ in range(3):
                _, _, r = plugin.pose_graph_optimize(states, edges, max_iter=10, eps_rot=1e-9, eps_pos=1e-8)
                ms.append(r["ms"])
            row = dict(nodes=n, loops=mm, iterations=r["iterations"], host=stats(ms), host_threads=os.cpu_count())
            res["pose_graph"].append(row)
            print(json.dumps(row))
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
