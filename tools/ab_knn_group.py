"""Ad-hoc sweep of the lanes-per-query of the cell-list scan (MALIO_KNN_GROUP is read once per process, so one process per
setting): device time of the search kernels of a measurement pass on C2 sub-sampled to n queries, and on C4."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) > 1 and sys.argv[1] == "child":
    sys.path.insert(0, os.path.join(ROOT, "ma-lio_b200"))
    import numpy as np
    from malio_b200 import synth, plugin
    out = []
    case = synth.case_C2()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    m = plugin.MeasurementModel(case.n_lidar, sort_queries=True, params=case.params)
    m.upload_map(snap)
    rng = np.random.default_rng(3)
    for n in (12500, 25000, 50000, 100000):
        pts = case.pts if n == case.pts.shape[0] else case.pts[np.sort(rng.choice(case.pts.shape[0], n, replace=False))]
        m.upload_scan(pts, case.table, case.table_off, case.temporal_comp)
        ts = []
        for i in range(10):
            ok, HTH, HTh, st = m.h_share_model(case.x_prop, True)
            ts.append(st.ms_knn * 1e3)
        out.append(f"C2/{n}: {np.median(ts[3:]):.1f}")
    m.close()
    if len(sys.argv) > 2 and sys.argv[2] == "c4":
        case = synth.case_C4()
        snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
        m = plugin.MeasurementModel(case.n_lidar, sort_queries=True, params=case.params)
        m.upload_map(snap); m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
        ts = []
        for i in range(8):
            ok, HTH, HTh, st = m.h_share_model(case.x_prop, True)
            ts.append(st.ms_knn * 1e3)
        out.append(f"C4/300000: {np.median(ts[3:]):.1f}")
        m.close()
    print("keys", os.environ.get("MALIO_KNN_KEYS", "1"), "group", os.environ.get("MALIO_KNN_GROUP", "auto"), "knn us:", "  ".join(out), flush=True)
else:
    # "old" = knn_direct_kernel; 2 / 4 = the key scan with that many lanes per query (4 lanes also preload the rows' first candidates).
    # An earlier sweep also varied the preload and tried 1 and 8 lanes: those instantiations were
    # removed from the library afterwards (MALIO_KNN_GROUP accepts 1, 2, 4).
    for g in ("old", "2", "4", "auto"):
        env = dict(os.environ)
        env.pop("MALIO_KNN_GROUP", None)
        if g == "old":
            env["MALIO_KNN_KEYS"] = "0"
        elif g != "auto":
            env["MALIO_KNN_GROUP"] = g
        subprocess.run([sys.executable, os.path.abspath(__file__), "child", "c4"], env=env, check=False)
