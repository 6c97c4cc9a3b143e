"""GPU parity of the k-NN fast path (cell-list index over the snapshot, knn_direct_kernel / knn_keys_kernel) and its
hand-over to the exact ikd-Tree-order traversal (knn_list_kernel).  Whatever the cell edge — automatic, tiny, huge, or the index
switched off — the neighbour lists and float distances must be the reference's, index for index: compared with
the restated Search (oracle) and, through the golden file, with the real ikd_Tree.cpp."""
import os

import numpy as np
import pytest

import helpers as H
import pyoracle as po
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CELLS = [0.0, -1.0, 0.3, 1.0, 2.5]   # automatic, index off (tree only), small, the default start, large


def _search(snap, q, cell, sort=True):
    m = plugin.MeasurementModel(1, sort_queries=sort, knn_cell_size=cell)
    m.upload_map(snap)
    c0 = m.counters()
    idx, d2, _ = m.Nearest_Search(q)
    c1 = m.counters()
    m.close()
    return idx, d2, int(c1.knn_fallback_queries - c0.knn_fallback_queries), int(c1.knn_ring2_queries - c0.knn_ring2_queries)


def test_golden_reference_lists_for_every_cell_size():
    g = np.load(os.path.join(ROOT, "tests", "golden", "ikd_knn_golden.npz"))
    nodes = g["nodes"].view(capi.MAP_NODE).reshape(-1)
    snap = plugin.MapSnapshot(nodes, g["node_cov"], g["node_ids"], int(g["max_depth"]))
    for cell in CELLS:
        idx, d2, fb, r2 = _search(snap, g["queries"], cell)
        ok = idx != 0xFFFFFFFF
        assert np.array_equal(ok.sum(1), g["ref_found"]), cell
        mapped = np.where(ok, g["node_ids"][np.where(ok, idx, 0)], -1)
        assert np.array_equal(mapped, g["ref_ids"]), cell
        assert np.array_equal(d2[ok], g["ref_d2"][ok]), cell
        if cell < 0:
            assert fb == 0 and r2 == 0


def test_ties_send_queries_to_the_exact_traversal():
    """Perfect lattice + duplicates: exact float ties at the k-th boundary.  The fast path must notice every one of
    them and hand the query over; the result is the reference's first-visited-wins list."""
    rng = np.random.default_rng(11)
    g = np.arange(-16, 16, dtype=np.float32) * 0.5
    X, Y, Z = np.meshgrid(g, g, g[:6], indexing="ij")
    lattice = np.stack([X.ravel(), Y.ravel(), Z.ravel()], axis=1).astype(np.float32)
    dup = lattice[rng.integers(0, lattice.shape[0], 1000)]
    xyz = np.concatenate([lattice, dup], axis=0)
    xyz = xyz[rng.permutation(xyz.shape[0])]
    snap = plugin.build_static_snapshot(xyz)
    q = np.concatenate([
        lattice[rng.integers(0, lattice.shape[0], 2000)] + np.float32(0.25),
        lattice[rng.integers(0, lattice.shape[0], 2000)],
        rng.uniform(-8, 8, (2000, 3)).astype(np.float32),
    ]).astype(np.float32)
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, q, nthreads=4)
    for cell in CELLS:
        idx, d2, fb, _ = _search(snap, q, cell)
        assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)), cell
        assert np.array_equal(d2, o_d2), cell
        if cell >= 0:
            assert fb >= 4000, (cell, fb)   # every lattice-centre / lattice-point query ties


def test_sparse_map_far_queries_and_outside_of_grid():
    """Neighbourhoods sparser than the cell block (5x5x5 block, then the traversal), queries far outside the map's
    bounding box, and a map with deleted points (they must never be returned)."""
    rng = np.random.default_rng(12)
    xyz = np.concatenate([rng.uniform(-40, 40, (3000, 3)),                 # ~0.006 pts/m^3: 5-NN at ~6 m
                          rng.uniform(-5, 5, (4000, 3)) + [100, 0, 0]]).astype(np.float32)   # a dense blob
    snap = plugin.build_static_snapshot(xyz)
    nodes = snap.nodes.copy()
    dead = rng.choice(nodes.shape[0], 700, replace=False)
    nodes["link"][dead] |= capi.LINK_POINT_DELETED
    snap = plugin.MapSnapshot(nodes, snap.node_cov, snap.node_ids, snap.max_depth)
    q = np.concatenate([rng.uniform(-45, 45, (3000, 3)), rng.uniform(-6, 6, (3000, 3)) + [100, 0, 0],
                        rng.uniform(-500, 500, (500, 3)), xyz[dead[:200]]]).astype(np.float32)
    o_idx, o_d2, _, _ = po.knn_snapshot(nodes, snap.node_cov, q, nthreads=4)
    assert not np.isin(o_idx, dead).any()
    seen_fb = seen_r2 = 0
    for cell in CELLS:
        idx, d2, fb, r2 = _search(snap, q, cell)
        assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)), cell
        assert np.array_equal(d2, o_d2), cell
        seen_fb += fb; seen_r2 += r2
    assert seen_fb > 0 and seen_r2 > 0


@pytest.mark.parametrize("cell", [-1.0, 0.4, 3.0])
def test_measurement_pass_identical_with_and_without_index(cell):
    """A full pass on the churned 3-LiDAR case: neighbour lists, gates and the reduced system with the given cell edge
    equal the automatic configuration bit for bit (the k-NN result is the only thing the index may influence)."""
    case = synth.make_case("3L-20k-200k", 20000, 200000, 3, 3, varied_map_cov=True)
    snap, _ = H.snapshot_for(case, churn=True)
    ref = H.make_model(case, snap)
    ok_r, HTH_r, HTh_r, st_r = ref.h_share_model(case.x_prop, True)
    a_r = ref.aux()
    m = plugin.MeasurementModel(case.n_lidar, params=case.params, knn_cell_size=cell)
    m.upload_map(snap)
    m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    ok, HTH, HTh, st = m.h_share_model(case.x_prop, True)
    a = m.aux()
    assert ok == ok_r and st.n_eff == st_r.n_eff
    for k in ("nn_idx", "nn_sqdist", "selected", "world", "normal_y"):
        assert np.array_equal(a[k], a_r[k]), k
    assert np.array_equal(HTH, HTH_r) and np.array_equal(HTh, HTh_r)
    ref.close(); m.close()


def _tight_boxes(nodes):
    """numpy restatement of the box rule: box(node) = bounding box of the live points of its subtree."""
    n = nodes.shape[0]
    out = nodes.copy()
    lo = np.full((n, 3), np.inf, np.float32)
    hi = np.full((n, 3), -np.inf, np.float32)
    link = nodes["link"]
    for i in range(n - 1, -1, -1):   # children have larger indices than their parent (DFS pre-order)
        if not (link[i] & capi.LINK_POINT_DELETED):
            lo[i] = np.minimum(lo[i], nodes["xyz"][i]); hi[i] = np.maximum(hi[i], nodes["xyz"][i])
        for child, key in (((i + 1) if (link[i] & capi.LINK_HAS_LEFT) else -1, "lbox"),
                           (int(link[i] & capi.LINK_INDEX_MASK) if (link[i] & capi.LINK_HAS_RIGHT) else -1, "rbox")):
            if child >= 0:
                out[key][i] = np.stack([lo[child], hi[child]], axis=1).reshape(6)
                lo[i] = np.minimum(lo[i], lo[child]); hi[i] = np.maximum(hi[i], hi[child])
    return out


def test_compact_upload_rebuilds_the_reference_boxes():
    """malio_upload_map_compact: 16 B per node go up, the device rebuilds both children's boxes of every node.  On the
    churned real ikd-Tree (lazy deletes, down-sampling adds) they must equal the node_range_* boxes the flattener copied
    out of the reference tree, float for float; and searches / passes through the compact upload are identical."""
    case = synth.make_case("3L-20k-200k", 20000, 200000, 3, 3, varied_map_cov=True)
    snap, _ = H.snapshot_for(case, churn=True)
    m = plugin.MeasurementModel(case.n_lidar, params=case.params)
    m.upload_map_compact(snap)
    dev = m.download_map_nodes(snap.n_nodes)
    ref = snap.nodes
    assert np.array_equal(dev["xyz"], ref["xyz"]) and np.array_equal(dev["link"], ref["link"])
    has_l = (ref["link"] & capi.LINK_HAS_LEFT) != 0
    has_r = (ref["link"] & capi.LINK_HAS_RIGHT) != 0
    assert np.array_equal(dev["lbox"][has_l], ref["lbox"][has_l])
    assert np.array_equal(dev["rbox"][has_r], ref["rbox"][has_r])
    m.upload_scan(case.pts, case.table, case.table_off, case.temporal_comp)
    ok, HTH, HTh, st = m.h_share_model(case.x_prop, True)
    a = m.aux()
    full = H.make_model(case, snap)
    ok_f, HTH_f, HTh_f, st_f = full.h_share_model(case.x_prop, True)
    a_f = full.aux()
    for k in ("nn_idx", "nn_sqdist", "selected", "world", "normal_y"):
        assert np.array_equal(a[k], a_f[k]), k
    assert np.array_equal(HTH, HTH_f) and np.array_equal(HTh, HTh_f)
    # the exact traversal on device-built boxes: index off => every query walks the tree
    t = plugin.MeasurementModel(1, knn_cell_size=-1.0)
    t.upload_map_compact(snap)
    q = a["world"][:4000]
    idx, d2, _ = t.Nearest_Search(q)
    assert np.array_equal(idx, a["nn_idx"][:4000]) and np.array_equal(d2, a["nn_sqdist"][:4000])
    # deleted points in a static snapshot (boxes must exclude them)
    rng = np.random.default_rng(3)
    s2 = plugin.build_static_snapshot(case.map_xyz[:5000])
    nodes = s2.nodes.copy()
    nodes["link"][rng.choice(5000, 300, replace=False)] |= capi.LINK_POINT_DELETED
    tight = _tight_boxes(nodes)
    s2 = plugin.MapSnapshot(nodes, s2.node_cov, s2.node_ids, s2.max_depth)
    t.upload_map_compact(s2)
    dev2 = t.download_map_nodes(5000)
    hl = (nodes["link"] & capi.LINK_HAS_LEFT) != 0
    hr = (nodes["link"] & capi.LINK_HAS_RIGHT) != 0
    assert np.array_equal(dev2["lbox"][hl], tight["lbox"][hl]) and np.array_equal(dev2["rbox"][hr], tight["rbox"][hr])
    o_idx, o_d2, _, _ = po.knn_snapshot(tight, s2.node_cov, q[:1000], nthreads=4)
    idx, d2, _ = t.Nearest_Search(q[:1000])
    assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)) and np.array_equal(d2, o_d2)
    m.close(); full.close(); t.close()


@pytest.mark.parametrize("offset", [1.0e5, 1.0e6])
def test_map_far_from_the_origin_float32_quantisation(offset):
    """Maps at large absolute coordinates (UTM-like 1e5..1e6 m): float32 spacing there is 0.008..0.06 m, so coordinates —
    and with them squared distances — collapse onto a coarse lattice and exact ties become common.  Correctness must
    hold by construction (ties go to the exact ikd-order traversal); the fallback fraction is what it costs, recorded
    in the test output (pytest -s) and in DESIGN.md."""
    rng = np.random.default_rng(31)
    base = rng.uniform(-30, 30, (60000, 3)).astype(np.float64)
    base[:, 2] = rng.uniform(0, 6, 60000)
    xyz = (base + np.array([offset, -0.7 * offset, 50.0])).astype(np.float32)
    snap = plugin.build_static_snapshot(xyz)
    q = (xyz[rng.integers(0, xyz.shape[0], 20000)].astype(np.float64) + rng.normal(0, 0.3, (20000, 3))).astype(np.float32)
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, q, nthreads=8)
    for cell in (0.0, -1.0, 1.0):
        idx, d2, fb, r2 = _search(snap, q, cell)
        assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)), (offset, cell)
        assert np.array_equal(d2, o_d2), (offset, cell)
        if cell >= 0:
            print(f"[far-from-origin] offset {offset:.0e} cell {cell}: {fb} of {q.shape[0]} queries ({100.0 * fb / q.shape[0]:.2f} %) took "
                  f"the exact traversal, {r2} the 5x5x5 block")


def test_many_queries_in_one_sort_cell_do_not_go_quadratic():
    """ADVICE round 1: the scan sort ranks the points of one 2 m bin against each other; 60k queries inside a single bin must
    not cost 60k^2 operations (bins above 2048 points keep the scatter's arrival order).  Results stay exact."""
    import time
    rng = np.random.default_rng(41)
    xyz = rng.uniform(-6, 6, (40000, 3)).astype(np.float32)
    snap = plugin.build_static_snapshot(xyz)
    q = rng.uniform(0.05, 1.9, (60000, 3)).astype(np.float32)      # one 2 m sort cell
    m = plugin.MeasurementModel(1)
    m.upload_map(snap)
    m.Nearest_Search(q[:100])
    t0 = time.perf_counter()
    idx, d2, _ = m.Nearest_Search(q)
    dt = time.perf_counter() - t0
    m.close()
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, q, nthreads=8)
    assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)) and np.array_equal(d2, o_d2)
    assert dt < 0.5, dt


@pytest.mark.parametrize("nq", [3000, 60000, 250000])
def test_every_scan_variant_matches_the_oracle(nq):
    """The 3x3x3 scan runs as 4 lanes per query with 32-bit keys (few queries), 2 lanes per query, or one thread per query
    (knn_direct_kernel) depending on the number of queries: all three must give the oracle's lists bit for bit."""
    rng = np.random.default_rng(100 + nq)
    xyz = np.concatenate([rng.uniform(-40, 40, (150000, 2)), rng.normal(0, 0.15, (150000, 1))], axis=1).astype(np.float32)
    snap = plugin.build_static_snapshot(xyz)
    q = np.concatenate([rng.uniform(-41, 41, (nq, 2)), rng.normal(0, 0.3, (nq, 1))], axis=1).astype(np.float32)
    idx, d2, fb, r2 = _search(snap, q, 0.0)
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, q, nthreads=8)
    assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64))
    assert np.array_equal(d2, o_d2)
    assert fb < nq // 20      # queries beyond the map edge walk the tree


def test_key_scan_boundary_cases_and_overlong_rows():
    """(a) 5th and 6th neighbour whose squared distances agree in the 13 mantissa bits the keys keep: the key scan cannot
    separate them and must redo the query exactly; (b) rows of more than 64 candidates do not fit the key's offset field:
    those queries are handed to the exact traversal.  Both must end with the oracle's lists."""
    rng = np.random.default_rng(77)
    nq = 1500
    centres = (np.stack(np.meshgrid(np.arange(40), np.arange(40), indexing="ij"), -1).reshape(-1, 2)[:nq] * 3.0).astype(np.float64)
    d2s = np.array([0.02, 0.05, 0.08, 0.11, 0.2500, 0.250004, 0.250008, 0.4, 0.5])
    pts = []
    for c in centres:
        for d in d2s * rng.uniform(0.98, 1.02):
            v = rng.normal(size=3); v /= np.linalg.norm(v)
            pts.append(np.array([c[0], c[1], 0.0]) + v * np.sqrt(d))
    xyz = np.array(pts, np.float32)
    q = np.concatenate([centres, np.zeros((nq, 1))], axis=1).astype(np.float32)
    snap = plugin.build_static_snapshot(xyz)
    for cell in (0.0, 1.0, 1.5):
        idx, d2, fb, r2 = _search(snap, q, cell)
        o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, q, nthreads=8)
        assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)), cell
        assert np.array_equal(d2, o_d2), cell
    # (b) 30k points inside 3 x 3 x 1 m with 1.5 m cells: thousands of candidates per row
    dense = rng.uniform([0, 0, 0], [3, 3, 1], (30000, 3)).astype(np.float32)
    snap = plugin.build_static_snapshot(dense)
    q = rng.uniform([0, 0, 0], [3, 3, 1], (2000, 3)).astype(np.float32)
    idx, d2, fb, r2 = _search(snap, q, 1.5)
    o_idx, o_d2, _, _ = po.knn_snapshot(snap.nodes, snap.node_cov, q, nthreads=8)
    assert np.array_equal(idx.astype(np.int64), o_idx.astype(np.int64)) and np.array_equal(d2, o_d2)
    assert fb == 2000
