"""More GPU parity cases: golden vectors of the real reference ikd-Tree, deep (unbalanced) snapshots that take the
local-memory-stack variant, degenerate filter branches, the C5 microbench shape, empty / tiny inputs, and the
2-GPU sharded path (skipped with fewer than 2 devices)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
import pyoracle as po
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_knn_matches_reference_golden():
    g = np.load(os.path.join(ROOT, "tests", "golden", "ikd_knn_golden.npz"))
    nodes = g["nodes"].view(capi.MAP_NODE).reshape(-1)
    snap = plugin.MapSnapshot(nodes, g["node_cov"], g["node_ids"], int(g["max_depth"]))
    for sort in (True, False):
        m = plugin.MeasurementModel(1, sort_queries=sort)
        m.upload_map(snap)
        idx, d2, _ = m.Nearest_Search(g["queries"])
        ok = idx != 0xFFFFFFFF
        assert np.array_equal(ok.sum(1), g["ref_found"])
        mapped = np.where(ok, g["node_ids"][np.where(ok, idx, 0)], -1)
        assert np.array_equal(mapped, g["ref_ids"])
        assert np.array_equal(d2[ok], g["ref_d2"][ok])
        m.close()


def _chain_snapshot(xyz):
    """A valid but maximally unbalanced snapshot: every node's left subtree is a single leaf (or empty), the rest
    hangs on the right => depth ~ n/2.  Boxes are exact AABBs of the subtrees."""
    n = xyz.shape[0]
    nodes = np.zeros(n, dtype=capi.MAP_NODE)
    order = np.argsort(xyz[:, 0], kind="stable")
    p = xyz[order]
    # layout: slot i (even) = spine node, slot i+1 = its left leaf (smaller x), right child = slot i+2
    # spine node k takes point 2k+1, its left leaf point 2k  (x sorted: leaf < node <= everything to the right)
    slots = []
    i = 0
    while i < n:
        if i + 1 < n:
            slots.append((i + 1, i))       # (spine point, leaf point)
            i += 2
        else:
            slots.append((i, None))
            i += 1
    # suffix AABBs of the remaining points
    suf_min = np.minimum.accumulate(p[::-1], axis=0)[::-1]
    suf_max = np.maximum.accumulate(p[::-1], axis=0)[::-1]
    s = 0
    depth = 0
    ids = np.zeros(n, np.int64)
    for k, (sp_, lf) in enumerate(slots):
        depth += 1
        node = nodes[s]
        node["xyz"] = p[sp_]
        ids[s] = order[sp_]
        link = 0
        nxt = s + 1
        if lf is not None:
            link |= capi.LINK_HAS_LEFT
            nodes[s + 1]["xyz"] = p[lf]
            ids[s + 1] = order[lf]
            nodes[s + 1]["link"] = 0
            node["lbox"] = [p[lf][0], p[lf][0], p[lf][1], p[lf][1], p[lf][2], p[lf][2]]
            nxt = s + 2
        first_rest = sp_ + 1
        if first_rest < n:
            link |= capi.LINK_HAS_RIGHT | nxt
            mn, mx = suf_min[first_rest], suf_max[first_rest]
            node["rbox"] = [mn[0], mx[0], mn[1], mx[1], mn[2], mx[2]]
        node["link"] = link
        s = nxt
    return plugin.MapSnapshot(nodes, np.full(n, 0.001, np.float32), ids, depth + 1)


def test_deep_snapshot_uses_local_stack_variant():
    rng = np.random.default_rng(9)
    xyz = (rng.random((120, 3)) * [30, 5, 2]).astype(np.float32)
    snap = _chain_snapshot(xyz)
    assert 32 <= snap.max_depth <= 96
    q = (rng.random((500, 3)) * [30, 5, 2]).astype(np.float32)
    m = plugin.MeasurementModel(1)
    m.upload_map(snap)
    idx, d2, _ = m.Nearest_Search(q)
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, q)
    assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64))
    assert np.array_equal(d2, o_d2)
    # and it is the true 5-NN
    d = q[:, None, :] - xyz[None, :, :]
    bd = (d[:, :, 0] * d[:, :, 0] + d[:, :, 1] * d[:, :, 1]) + d[:, :, 2] * d[:, :, 2]
    assert np.array_equal(np.sort(snap.node_ids[idx.astype(np.int64)], 1), np.sort(np.argsort(bd, 1, kind="stable")[:, :5], 1))
    # deeper than the bound is rejected loudly
    too_deep = _chain_snapshot((rng.random((400, 3)) * [30, 5, 2]).astype(np.float32))
    with pytest.raises(capi.MalioError) as e:
        m.upload_map(too_deep)
    assert e.value.status == capi.ERR_TREE_TOO_DEEP
    m.close()


def test_degenerate_branches_match_oracle():
    base = synth.make_case("b", 3000, 40000, 3, 3, varied_map_cov=True)
    snap = plugin.build_static_snapshot(base.map_xyz, base.map_normal_y)
    # (1) fewer effective points than state DOF -> dense branch through malio_download_rows (esekfom.hpp:574-582)
    sub = synth.make_case("tiny", 25, 40000, 3, 3, map_xyz=base.map_xyz)
    model = H.make_model(sub, snap)
    orc = H.make_oracle(sub, snap)
    xg, Pg = sub.x_prop.copy(), sub.P_prop.copy()
    xo, Po = sub.x_prop.copy(), sub.P_prop.copy()
    rep = model.update_iterated_dyn_share_modified(xg, Pg, 3)
    rc, _, _, rep_o = orc.update_iterated(xo, Po, 3)
    assert rep.passes == rep_o.passes and 1 <= rep.n_eff_last < 35
    assert np.abs(synth.state_to_vec(xg, 3) - synth.state_to_vec(xo, 3)).max() < 1e-4
    assert H.rel_err(Pg, Po) < 1e-6
    hx, hv = model.rows()
    assert hx.shape[0] == rep.n_eff_last
    model.close()
    # (2) no effective points -> every pass invalid, state and covariance untouched
    far = plugin.build_static_snapshot(base.map_xyz[:50] + np.float32(1e4))
    model = H.make_model(base, far)
    ok, _, _, st = model.h_share_model(base.x_prop, True)
    assert not ok and st.n_eff == 0 and st.valid == 0
    xg, Pg = base.x_prop.copy(), base.P_prop.copy()
    rep = model.update_iterated_dyn_share_modified(xg, Pg, 3)
    assert rep.last_status == capi.ERR_NO_EFFECTIVE_POINTS and rep.passes == 4
    assert np.array_equal(synth.state_to_vec(xg, 3), synth.state_to_vec(base.x_prop, 3))
    assert np.array_equal(Pg, base.P_prop)
    model.close()
    # (3) a map with fewer than 5 points: found < 5 everywhere
    three = plugin.build_static_snapshot(base.map_xyz[:3])
    model = H.make_model(base, three)
    ok, _, _, st = model.h_share_model(base.x_prop, True)
    assert not ok
    a = model.aux()
    assert np.all(a["nn_idx"][:, 3:] == 0xFFFFFFFF) and np.all(a["nn_idx"][:, :3] < 3)
    model.close()


def test_single_lidar_and_two_lidar_layouts():
    for L in (1, 2):
        case = synth.make_case(f"L{L}", 4000, 40000, L, 3, varied_map_cov=True)
        snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
        model = H.make_model(case, snap)
        orc = H.make_oracle(case, snap)
        ok, HTH, HTh, st = model.h_share_model(case.x_prop, True)
        assert orc.h_share_model(case.x_prop, True, 2) and ok
        HTH_o, HTh_o = orc.reduce()
        assert HTH.shape == (6 * (L + 1), 6 * (L + 1))
        assert H.rel_err(HTH, HTH_o) < 1e-9 and H.rel_err(HTh, HTh_o) < 1e-9
        xg, Pg = case.x_prop.copy(), case.P_prop.copy()
        xo, Po = case.x_prop.copy(), case.P_prop.copy()
        model.update_iterated_dyn_share_modified(xg, Pg, 3)
        orc.update_iterated(xo, Po, 3, nthreads=2)
        assert np.abs(synth.state_to_vec(xg, L) - synth.state_to_vec(xo, L)).max() < 1e-4
        model.close()


def test_full_size_properties_c2():
    """BASELINE configs[1] size (100k vs 1M): size-independent properties instead of a full oracle run —
    sorted distances, in-range indices, idempotence of the search, re-arm reproducibility (bit-identical system),
    sorted vs unsorted execution order (k-NN lists identical, system equal to rounding), and an oracle spot-check
    of the neighbour lists on a 2k-query sample."""
    case = synth.case_C2()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    model = H.make_model(case, snap, sort_queries=True)
    ok, HTH, HTh, st = model.h_share_model(case.x_prop, True)
    a = model.aux()
    assert ok and st.n_eff > 50000
    assert np.all(np.diff(a["nn_sqdist"], axis=1) >= 0) and a["nn_idx"].max() < snap.n_nodes
    assert np.allclose(HTH, HTH.T, rtol=1e-12, atol=1e-6 * np.abs(HTH).max())
    ok2, HTH2, HTh2, _ = model.h_share_model(case.x_prop, True)
    assert np.array_equal(HTH, HTH2) and np.array_equal(HTh, HTh2)
    model.rearm_scan()
    ok3, HTH3, HTh3, _ = model.h_share_model(case.x_prop, True)
    assert np.array_equal(HTH, HTH3) and np.array_equal(HTh, HTh3)
    rng = np.random.default_rng(0)
    pick = rng.choice(case.pts.shape[0], 2000, replace=False)
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, a["world"][pick], nthreads=4)
    assert np.array_equal(a["nn_idx"][pick].astype(np.int64), o_idx.astype(np.int64))
    assert np.array_equal(a["nn_sqdist"][pick], o_d2)
    model.close()
    m2 = H.make_model(case, snap, sort_queries=False)
    ok4, HTH4, HTh4, st4 = m2.h_share_model(case.x_prop, True)
    b = m2.aux()
    assert np.array_equal(a["nn_idx"], b["nn_idx"]) and np.array_equal(a["selected"], b["selected"])
    assert st4.n_eff == st.n_eff and H.rel_err(HTH4, HTH) < 1e-11
    m2.close()


def test_empty_scan_and_reupload():
    case = synth.case_C1()
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    model = H.make_model(case, snap)
    model.upload_scan(case.pts[:0], case.table, case.table_off, case.temporal_comp)
    ok, _, _, st = model.h_share_model(case.x_prop, True)
    assert not ok and st.n_eff == 0
    model.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    ok, HTH, _, st = model.h_share_model(case.x_prop, True)
    assert ok and st.n_eff > 4000
    with pytest.raises(capi.MalioError):
        model.upload_scan(case.pts, case.table[:1], np.array([0, 1], np.uint32), None)   # table too short
    model.close()


def test_two_gpu_sharded_update_matches_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29611",
                          os.path.join(ROOT, "tests", "mgpu_worker.py")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "MGPU_OK" in out.stdout and "MGPU_DEGENERATE_OK" in out.stdout


def test_unfused_kernel_path_matches_fused_pass(monkeypatch):
    """The separate gate / reduce / fold kernels (the path the NCCL fallback uses) and the fused cooperative pass must
    agree: identical gates and neighbour lists, reduced system to FP64 rounding, same iterated update."""
    case = synth.make_case("3L-20k-200k", 20000, 200000, 3, 3, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    fused = H.make_model(case, snap)
    monkeypatch.setenv("MALIO_FUSED_PASS", "0")
    plain = H.make_model(case, snap)
    monkeypatch.delenv("MALIO_FUSED_PASS")
    for conv in (True, False):
        okf, Hf, hf, sf = fused.h_share_model(case.x_prop, conv)
        okp, Hp, hp, sp = plain.h_share_model(case.x_prop, conv)
        assert okf and okp and sf.n_eff == sp.n_eff
        assert H.rel_err(Hf, Hp) < 1e-11 and H.rel_err(hf, hp) < 1e-11
        af, ap = fused.aux(), plain.aux()
        for k in ("nn_idx", "selected", "world", "normal_y"):
            assert np.array_equal(af[k], ap[k]), k
    xf, Pf = case.x_prop.copy(), case.P_prop.copy()
    xp, Pp = case.x_prop.copy(), case.P_prop.copy()
    fused.rearm_scan(); plain.rearm_scan()
    rf = fused.update_iterated_dyn_share_modified(xf, Pf, 3)
    rp = plain.update_iterated_dyn_share_modified(xp, Pp, 3)
    assert rf.passes == rp.passes and rf.searches == rp.searches
    assert np.abs(synth.state_to_vec(xf, 3) - synth.state_to_vec(xp, 3)).max() < 1e-9
    # large scan: more than two tiles per block -> the generic (global-memory rows, LiDAR-major order) variant of the pass
    big = synth.make_case("3L-180k", 180000, 200000, 3, 3, varied_map_cov=True, map_xyz=case.map_xyz)
    mb = H.make_model(big, snap)
    monkeypatch.setenv("MALIO_FUSED_PASS", "0")
    pb = H.make_model(big, snap)
    monkeypatch.delenv("MALIO_FUSED_PASS")
    okf, Hf, hf, sf = mb.h_share_model(big.x_prop, True)
    okp, Hp, hp, sp = pb.h_share_model(big.x_prop, True)
    assert okf and okp and sf.n_eff == sp.n_eff and H.rel_err(Hf, Hp) < 1e-11 and H.rel_err(hf, hp) < 1e-11
    for m in (fused, plain, mb, pb):
        m.close()


def test_map_incremental_decision_matches_oracle():
    """SURVEY §8f N1: map_incremental's per-point decision (laserMapping.cpp:398-446) evaluated on the device from the
    data the update left there; classes and feats_down_world must equal the oracle's for the same state, bit for bit
    (1 and 3 LiDARs, filter initialised or not, two voxel sizes)."""
    for L, n, m in ((1, 5000, 50000), (3, 20000, 200000)):
        case = synth.make_case(f"mi{L}", n, m, L, 3, varied_map_cov=True)
        snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
        model = H.make_model(case, snap)
        orc = H.make_oracle(case, snap)
        xg, Pg = case.x_prop.copy(), case.P_prop.copy()
        xo, Po = case.x_prop.copy(), case.P_prop.copy()
        model.update_iterated_dyn_share_modified(xg, Pg, case.max_iter)
        orc.update_iterated(xo, Po, case.max_iter, nthreads=4)
        ag, ao = model.aux(), orc.aux()
        gi = ag["nn_idx"].astype(np.int64); gi[gi == 0xFFFFFFFF] = -1
        assert np.array_equal(gi, ao["nn_idx"].astype(np.int64))
        for fs in (0.5, 0.2):
            for inited in (True, False):
                cls_g, w_g = model.map_incremental(xg, fs, inited)
                cls_o, w_o = orc.map_incremental(xg, fs, inited)
                assert np.array_equal(cls_g, cls_o), (L, fs, inited, int((cls_g != cls_o).sum()))
                assert np.array_equal(w_g, w_o)
        assert len(set(cls_g.tolist())) >= 1
        model.close()


EXAMPLE = os.path.join(ROOT, "oracle", "_ref", "replay_city")


@pytest.mark.skipif(not os.path.exists(EXAMPLE), reason="oracle/_ref/replay_city not built (needs the reference's ikd_Tree.cpp)")
def test_cpp_example_full_program_on_the_gpu():
    """examples/replay_city.cpp end to end on the device: undistortion + voxel grid of three synthetic LiDARs, merged scan,
    iterated update against the device-resident map, map_incremental and the map deltas; the device's live point count must
    equal the reference tree's valid count afterwards (the program's exit code says so)."""
    r = subprocess.run([EXAMPLE], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])
    lines = r.stdout.splitlines()
    assert lines[0].startswith("malio_b200") and sum(l.startswith("LiDAR ") for l in lines) == 3
    upd = [l for l in lines if l.startswith("update:")][0].split()
    passes, n_eff = int(upd[1]), int(upd[upd.index("N_eff") + 1].rstrip(","))
    assert 1 <= passes <= 4 and n_eff > 0
    assert any(l.startswith("map: tree holds") for l in lines)
