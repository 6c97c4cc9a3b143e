"""Workload for ncu / timing: C2, a few full iterated updates on a resident scan."""
import sys, os, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
from malio_b200 import synth, plugin
which = sys.argv[1] if len(sys.argv) > 1 else "C2"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 3
case = {"C1": synth.case_C1, "C2": synth.case_C2, "C4": synth.case_C4}[which]()
snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
m = plugin.MeasurementModel(case.n_lidar, sort_queries=True, params=case.params)
m.upload_map(snap)
m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
for i in range(n):
    m.rearm_scan()
    x, P = case.x_prop.copy(), case.P_prop.copy()
    t0 = time.perf_counter()
    rep = m.update_iterated_dyn_share_modified(x, P, case.max_iter)
    print(f"update {i}: wall {1e3 * (time.perf_counter() - t0):.3f} ms, device {rep.ms_device_total:.3f} ms, passes {rep.passes}")
m.close()
