"""Host-side mirror of the reference's measurement plug-in, over the C-ABI.

Names follow the reference (paths relative to /root/reference/MA_LIO):
  MeasurementModel.h_share_model(state, converge)        src/laserMapping.cpp:552-760  (+ esekfom.hpp:622-635)
  MeasurementModel.update_iterated_dyn_share_modified()  include/IKFoM_toolkit/esekfom/esekfom.hpp:495-721
  MeasurementModel.Nearest_Search(points)                include/ikd-Tree/ikd_Tree.cpp:426-461
Everything heavy happens inside libmalio_b200.so on the GPU; this file is marshalling only.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass

import numpy as np

from . import capi


@dataclass
class MapSnapshot:
    """Flattened ikd-Tree (include/malio_flatten.hpp or malio_build_static_snapshot)."""
    nodes: np.ndarray        # capi.MAP_NODE[M]
    node_cov: np.ndarray     # float32[M]  map-side weight normal_y (common_lib.h:164)
    node_ids: np.ndarray     # int32/uint32[M] caller's id of the point stored in each node
    max_depth: int

    @property
    def n_nodes(self) -> int:
        return int(self.nodes.shape[0])


def build_static_snapshot(xyz: np.ndarray, normal_y: np.ndarray | float = 0.001) -> MapSnapshot:
    """Balanced k-d tree over xyz directly in snapshot form (median split on the longest axis, like
    KD_TREE::BuildTree, ikd_Tree.cpp:696-735).  Host C++ inside the product library."""
    lib = capi.load()
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    n = xyz.shape[0]
    nodes = np.zeros(n, dtype=capi.MAP_NODE)
    order = np.zeros(n, dtype=np.uint32)
    depth = C.c_uint32(0)
    rc = lib.malio_build_static_snapshot(capi.ptr(xyz), n, capi.ptr(nodes), capi.ptr(order), C.byref(depth))
    if rc != capi.OK:
        raise capi.MalioError(rc, "malio_build_static_snapshot")
    if np.isscalar(normal_y):
        cov = np.full(n, normal_y, dtype=np.float32)
    else:
        cov = np.ascontiguousarray(np.asarray(normal_y, dtype=np.float32)[order])
    return MapSnapshot(nodes, cov, order.astype(np.int64), int(depth.value))


def compact_points(nodes: np.ndarray) -> np.ndarray:
    """capi.MAP_NODE[M] -> capi.MAP_POINT[M]: the first 16 bytes (point + link) of every record."""
    out = np.empty(nodes.shape[0], dtype=capi.MAP_POINT)
    out["xyz"] = nodes["xyz"]
    out["link"] = nodes["link"]
    return out


def build_pose_unc(extrinsic: np.ndarray, temporal_comp: np.ndarray | None, lidar_uncertainty: list[np.ndarray]):
    """pose_unc of one scan (laserMapping.cpp:1028-1048) through the library's host code.  extrinsic: capi.POSE[L],
    temporal_comp: capi.POSE[L-1] or None, lidar_uncertainty: L arrays of capi.POSE.  Returns (table capi.POSE_ENTRY[],
    table_off uint32[L+1]) ready for MeasurementModel.upload_scan."""
    lib = capi.load()
    L = len(lidar_uncertainty)
    lists = [np.ascontiguousarray(a, dtype=capi.POSE) for a in lidar_uncertainty]
    counts = np.array([a.shape[0] for a in lists], np.uint32)
    ptrs = (C.c_void_p * L)(*[a.ctypes.data for a in lists])
    n = int(sum(max(int(c) - 1, 0) for c in counts))
    table = np.zeros(max(n, 1), dtype=capi.POSE_ENTRY)
    off = np.zeros(L + 1, np.uint32)
    ext = np.ascontiguousarray(extrinsic, dtype=capi.POSE)
    tc = None if temporal_comp is None else np.ascontiguousarray(temporal_comp, dtype=capi.POSE)
    rc = lib.malio_build_pose_unc(L, capi.ptr(ext), capi.ptr(tc), C.cast(ptrs, C.c_void_p), capi.ptr(counts), capi.ptr(table),
                                  capi.ptr(off))
    if rc < 0:
        raise capi.MalioError(-rc, "malio_build_pose_unc")
    return table[:rc], off


def bspline_get_pose(ctrl_t: np.ndarray, ctrl_T: np.ndarray, timestamp: float):
    """BsplineSE3::get_pose (BsplineSE3.cpp:84-118) through the library's host code.  Returns (ok, q wxyz, p)."""
    ct = np.ascontiguousarray(ctrl_t, np.float64)
    cT = np.ascontiguousarray(ctrl_T, np.float64).reshape(-1, 16)
    q, p = np.zeros(4), np.zeros(3)
    ok = capi.load().malio_bspline_get_pose(capi.ptr(ct), capi.ptr(cT), ct.shape[0], float(timestamp), capi.ptr(q), capi.ptr(p))
    return bool(ok), q, p


def write_pcd_binary(path: str, xyzi: np.ndarray):
    """pcl::PCDWriter::writeBinary of PointXYZINormal points {x, y, z, intensity} (the other fields 0), host code."""
    a = np.ascontiguousarray(xyzi, np.float32).reshape(-1, 4)
    rc = capi.load().malio_write_pcd_binary(os.fsencode(path), capi.ptr(a), a.shape[0])
    if rc != capi.OK:
        raise capi.MalioError(rc, f"malio_write_pcd_binary({path!r})")


def read_pcd(path: str) -> np.ndarray:
    """A binary PCD file as this library (and pcl::PCDWriter::writeBinary) writes it: float32 (n, 4) {x, y, z, intensity}
    (intensity 0 when the file has none).  Host code (malio_read_pcd)."""
    lib = capi.load()
    n = C.c_uint64(0)
    rc = lib.malio_read_pcd(os.fsencode(path), None, 0, C.byref(n))
    if rc != capi.OK:
        raise capi.MalioError(rc, f"malio_read_pcd({path!r})")
    out = np.zeros((n.value, 4), np.float32)
    if n.value:
        rc = lib.malio_read_pcd(os.fsencode(path), capi.ptr(out), n.value, C.byref(n))
        if rc != capi.OK:
            raise capi.MalioError(rc, f"malio_read_pcd({path!r})")
    return out


def pos_lid(s: "capi.State") -> np.ndarray:
    """pos_lid = state.pos + state.rot * extrinsic_trans[0] (laserMapping.cpp:1056) in float64, the quaternion applied as Eigen's
    _transformVector: v + w uv + qv x uv, uv = 2 (qv x v)."""
    q = np.array(s.rot[:], np.float64)
    v = np.array(s.ext[0].t[:], np.float64)
    qv = q[1:]
    uv = np.cross(qv, v)
    uv = uv + uv
    r = v + q[0] * uv + np.cross(qv, uv)
    return np.array(s.pos[:], np.float64) + r


# Defaults of the carve and the keep rule (malio_world_voxel_accumulate_carve), chosen with tests/carve_ref.py on the street
# scene of synth.street_scan (DESIGN.md, "Clearing moving objects"): rays followed 100 m; no voxel entered within 4 m of a ray's
# end counts as passed (grazing rays over the ground and along façades); a voxel is dropped after at least 2 scans passed it
# and more than twice as many scans passed it as hit it.
CARVE_MAX_RANGE = 100.0
CARVE_END_MARGIN = 4.0
KEEP_MIN_MISS = 2
KEEP_MAX_MISS_PER_HIT = 2.0
# The hits a seeded voxel starts with (malio_world_voxel_seed), chosen with tests/world_seed_ref.py on the two-session street
# scene (DESIGN.md, "Keeping a saved map current").
SEED_HITS = 2
# Defaults of the occupancy grid (malio_grid_build_device), chosen with tests/grid_ref.py on the carved street and the sloped
# scene of tests/test_grid_cpu.py (DESIGN.md, "A 2-D occupancy grid for navigation"): 0.1 m cells, the ground taken over
# +-1 m around a cell, an obstacle band 0.3-2.0 m above it, one band point for an obstacle (a voxel map holds one centroid per
# voxel, so a box's roof gives one band point per column).
GRID_RES = 0.1
GRID_GROUND_HALFWIDTH = 10
GRID_H_LO = 0.3
GRID_H_HI = 2.0
GRID_MIN_OBSTACLE_POINTS = 1
# Defaults of the loop closure (malio_scan_store_match, close_loops), chosen on the synthetic ray-cast drives of
# tests/test_gpu_loop.py (DESIGN.md, "Closing loops over the scan store"): three levels from 2 m to 0.5 m voxels, a submap of the
# anchor +- 10 stored scans, an edge accepted at fitness >= 0.3, rms <= 0.1 m and a per-inlier constraint (accept_edge) >= ACCEPT_CONSTRAINT.
MATCH_LEAF = (2.0, 1.0, 0.5)
MATCH_GATE = (1.0, 0.5, 0.25)
MATCH_MAX_ITER = 30
MATCH_EPS_ROT = 1e-6
MATCH_EPS_POS = 1e-5
MATCH_MIN_POINTS = 5
MATCH_PLANARITY = 0.1
MATCH_SIGMA = 0.05
MATCH_HALF_WINDOW = 10
ACCEPT_FITNESS = 0.3
ACCEPT_RMS = 0.1
# eig_min * sigma^2 / n_inliers: the smallest eigenvalue of the mean J^T J per inlier, independent of the scan's size and of
# sigma (a corridor gave 0.006, the drive around a block 0.041-0.047, a street corner 0.073)
ACCEPT_CONSTRAINT = 0.02
POSE_GRAPH_SIGMA_ROT = 0.01
POSE_GRAPH_SIGMA_POS = 0.1
GRID_SOURCES = {"points": capi.GRID_POINTS, "voxel_map": capi.GRID_VOXEL_MAP, "prior": capi.GRID_PRIOR}


def match_args(target_first: int = 0, target_count: int = 1, leaf=MATCH_LEAF, gate=MATCH_GATE, max_iter: int = MATCH_MAX_ITER,
               eps_rot: float = MATCH_EPS_ROT, eps_pos: float = MATCH_EPS_POS, min_points: int = MATCH_MIN_POINTS,
               planarity: float = MATCH_PLANARITY, sigma: float = MATCH_SIGMA) -> capi.MatchArgs:
    """malio_match_args; leaf and gate: one value per level, coarse to fine (at most MATCH_MAX_LEVELS)."""
    leaf, gate = [float(v) for v in np.atleast_1d(leaf)], [float(v) for v in np.atleast_1d(gate)]
    if len(leaf) != len(gate) or not 0 < len(leaf) <= capi.MATCH_MAX_LEVELS:
        raise ValueError(f"leaf and gate: one value each per level, 1..{capi.MATCH_MAX_LEVELS} levels")
    a = capi.MatchArgs()
    a.target_first, a.target_count, a.n_levels = int(target_first), int(target_count), len(leaf)
    for l, (f, g) in enumerate(zip(leaf, gate)):
        a.leaf[l], a.gate[l] = f, g
    a.max_iter, a.eps_rot, a.eps_pos = int(max_iter), float(eps_rot), float(eps_pos)
    a.min_points, a.planarity, a.sigma = int(min_points), float(planarity), float(sigma)
    return a


def pose_graph_optimize(states, edges, sigma_rot: float = POSE_GRAPH_SIGMA_ROT, sigma_pos: float = POSE_GRAPH_SIGMA_POS,
                        max_iter: int = 50, eps_rot: float = 1e-9, eps_pos: float = 1e-8) -> tuple:
    """The odometry chain of `states` (capi.PassState / capi.State, node 0 fixed) plus loop `edges` (capi.PoseEdge, or dicts
    with a, b, rel_rot, rel_pos, info as close_loops accepts them) optimized on the host (malio_pose_graph_optimize).
    Returns (corrected capi.PassState list, per-loop chi^2 array, report dict)."""
    lib = capi.load()
    states = [s.pass_state() if isinstance(s, capi.State) else s for s in states]
    n, m = len(states), len(edges)
    odo = (capi.PassState * max(n, 1))(*states)
    loops = (capi.PoseEdge * max(m, 1))()
    for i, e in enumerate(edges):
        if isinstance(e, capi.PoseEdge):
            loops[i] = e
            continue
        loops[i].a, loops[i].b = int(e["a"]), int(e["b"])
        loops[i].rot[:] = [float(v) for v in e["rel_rot"]]
        loops[i].pos[:] = [float(v) for v in e["rel_pos"]]
        loops[i].info[:] = [float(v) for v in np.asarray(e["info"], np.float64).reshape(36)]
    a = capi.PoseGraphArgs(float(sigma_rot), float(sigma_pos), int(max_iter), float(eps_rot), float(eps_pos))
    out = (capi.PassState * max(n, 1))()
    chi = np.zeros(max(m, 1))
    rep = capi.PoseGraphReport()
    rc = lib.malio_pose_graph_optimize(odo, n, loops if m else None, m, C.byref(a), out, capi.ptr(chi), C.byref(rep))
    if rc != capi.OK:
        raise capi.MalioError(rc, "malio_pose_graph_optimize: invalid argument")
    return ([out[k] for k in range(n)], chi[:m].copy(),
            dict(iterations=int(rep.iterations), converged=bool(rep.converged), chi2_odo=rep.chi2_odo, chi2_loop=rep.chi2_loop,
                 chi2_loop_before=rep.chi2_loop_before, ms=rep.ms))


def loop_candidates(records, radius: float, min_gap: int, stride: int = 1) -> list:
    """(i, j) pairs: for every stride-th stored scan j, the scan i <= j - min_gap whose stored position is nearest to j's,
    when it lies within radius (first index on ties).  records: capi.StoredScan (or capi.PassState) list."""
    pos = np.array([list((r.state if hasattr(r, "state") else r).pos) for r in records], np.float64).reshape(-1, 3)
    out = []
    for j in range(0, len(pos), max(int(stride), 1)):
        if j - min_gap < 0:
            continue
        d = np.linalg.norm(pos[:j - min_gap + 1] - pos[j], axis=1)
        i = int(np.argmin(d))
        if d[i] <= radius:
            out.append((i, j))
    return out


def constraint(rep: dict) -> float:
    """eig_min * sigma^2 / n_inliers of a match report: how well the weakest direction of the edge is held, per inlier (0 for
    no inlier).  Unlike eig_min it does not grow with the scan's size or the chosen sigma."""
    return rep["eig_min"] * rep["sigma"] ** 2 / rep["n_inliers"] if rep["n_inliers"] else 0.0


def accept_edge(rep: dict, fitness: float = ACCEPT_FITNESS, rms: float = ACCEPT_RMS, min_constraint: float = ACCEPT_CONSTRAINT) -> bool:
    """The acceptance rule of close_loops: a match whose finest level converged, with fitness, rms and constraint(rep) on the
    right side of the thresholds."""
    return bool(rep["converged"] and rep["fitness"] >= fitness and rep["rms"] <= rms and constraint(rep) >= min_constraint)


def close_loops(model: "MeasurementModel", radius: float = 10.0, min_gap: int = 30, stride: int = 1,
                half_window: int = MATCH_HALF_WINDOW, accept: dict | None = None, graph: dict | None = None, **match) -> dict:
    """Loop closure over the model's scan store: loop_candidates, each candidate's source matched against its anchor
    +- half_window (scan_store_match from the source's stored state), the edges accept_edge keeps, then pose_graph_optimize
    of the stored states with them.  Returns dict(states = the corrected capi.PassState list (for voxel_map_rebuild),
    edges = the accepted match reports the pose graph used (with a = anchor, b = source; more accepted edges than
    capi.POSE_GRAPH_MAX_LOOPS are thinned evenly along the drive), reports = every match report (accepted, used), graph = the
    pose graph's report)."""
    recs = model.scan_store_records()
    reports, edges = [], []
    for i, j in loop_candidates(recs, radius, min_gap, stride):
        first = max(i - half_window, 0)
        count = min(i + half_window + 1, j - min_gap + 1, len(recs)) - first
        r = model.scan_store_match(j, i, target_first=first, target_count=count, **match)
        r["accepted"] = accept_edge(r, **(accept or {}))
        reports.append(r)
        if r["accepted"]:
            edges.append(dict(r, a=i, b=j))
    if len(edges) > capi.POSE_GRAPH_MAX_LOOPS:   # thinned evenly along the drive to what the pose graph takes
        keep = np.unique(np.linspace(0, len(edges) - 1, capi.POSE_GRAPH_MAX_LOOPS).round().astype(int))
        edges = [edges[k] for k in keep]
    used = {(e["a"], e["b"]) for e in edges}
    for r in reports:
        r["used"] = (r["anchor"], r["source"]) in used
    states = [r.state for r in recs]
    if edges:
        states, _, g = pose_graph_optimize(states, edges, **(graph or {}))
    else:
        g = dict(iterations=0, converged=True, chi2_odo=0.0, chi2_loop=0.0, chi2_loop_before=0.0, ms=0.0)
    return dict(states=states, edges=edges, reports=reports, graph=g)


def carve_args(max_range: float = CARVE_MAX_RANGE, end_margin: float = CARVE_END_MARGIN) -> capi.CarveArgs:
    a = capi.CarveArgs()
    a.max_range, a.end_margin = float(max_range), float(end_margin)
    return a


def carve_keep(min_miss: int = KEEP_MIN_MISS, max_miss_per_hit: float = KEEP_MAX_MISS_PER_HIT) -> capi.CarveKeep:
    k = capi.CarveKeep()
    k.min_miss, k.max_miss_per_hit = int(min_miss), float(max_miss_per_hit)
    return k


def _as_carve(carve) -> capi.CarveArgs | None:
    """None, True (the defaults), a capi.CarveArgs, or a dict of carve_args' keywords."""
    if carve is None or carve is False:
        return None
    if carve is True:
        return carve_args()
    return carve if isinstance(carve, capi.CarveArgs) else carve_args(**carve)


def _as_keep(keep) -> capi.CarveKeep | None:
    """None (every voxel), True (the defaults), a capi.CarveKeep, or a dict of carve_keep's keywords."""
    if keep is None or keep is False:
        return None
    if keep is True:
        return carve_keep()
    return keep if isinstance(keep, capi.CarveKeep) else carve_keep(**keep)


def grid_args(res: float = GRID_RES, i0: int = 0, j0: int = 0, nx: int = 0, ny: int = 0, ground_halfwidth: int = GRID_GROUND_HALFWIDTH,
              h_lo: float = GRID_H_LO, h_hi: float = GRID_H_HI, min_obstacle_points: int = GRID_MIN_OBSTACLE_POINTS) -> capi.GridArgs:
    """malio_grid_args with the library's defaults; the region (i0, j0, nx, ny) in cells of res (nx = ny = 0: to be filled, e.g.
    by MeasurementModel.grid from the source's extent)."""
    a = capi.GridArgs()
    a.res, a.i0, a.j0, a.nx, a.ny = float(res), int(i0), int(j0), int(nx), int(ny)
    a.ground_halfwidth, a.h_lo, a.h_hi, a.min_obstacle_points = int(ground_halfwidth), float(h_lo), float(h_hi), int(min_obstacle_points)
    return a


def save_grid(stem: str, cls, args: capi.GridArgs):
    """Write <stem>.pgm and <stem>.yaml, the map_server pair navigation stacks load, from a class raster (ny, nx) u8 (numpy or a
    tensor) of the region in args (malio_write_grid_pgm, host code).  Returns the two paths."""
    c = np.ascontiguousarray(cls.cpu().numpy() if hasattr(cls, "cpu") else cls, np.uint8)
    if c.ndim != 2 or c.shape != (args.ny, args.nx):
        raise ValueError(f"cls: shape {c.shape}, expected ({args.ny}, {args.nx})")
    pgm, yaml = stem + ".pgm", stem + ".yaml"
    rc = capi.load().malio_write_grid_pgm(os.fsencode(pgm), os.fsencode(yaml), capi.ptr(c), args.nx, args.ny, C.c_float(args.res),
                                          args.i0, args.j0)
    if rc != capi.OK:
        raise capi.MalioError(rc, f"malio_write_grid_pgm({pgm!r}, {yaml!r})")
    return pgm, yaml


def _grid_report(r: capi.GridReport) -> dict:
    return {f: int(getattr(r, f)) for f, _ in capi.GridReport._fields_}


class PcdSaver:
    """The pcd_save_en branch of publish_frame_world (laserMapping.cpp:466-488) and the map save at shutdown (:1083-1091) over
    a MeasurementModel: the library keeps pcl_wait_save on the device; the scan counter and the file names live here.
    leaf (m, optional): keep the saved map as a voxel map of that leaf instead of the dense cloud (MeasurementModel.voxel_map_*):
    the files hold one centroid per voxel; the names and the interval logic are the same.
    carve / keep (with leaf): count free-space evidence while accumulating and save only the voxels the keep rule keeps (True
    for the defaults, or CarveArgs / CarveKeep); see MeasurementModel.voxel_map_accumulate."""

    def __init__(self, model: "MeasurementModel", directory: str, pcd_save_interval: int, leaf: float | None = None,
                 carve=None, keep=None):
        self.model, self.directory, self.interval = model, directory, int(pcd_save_interval)
        self.leaf = None if leaf is None else _check_leaf(leaf)
        self.carve, self.keep = _as_carve(carve), _as_keep(keep)
        if self.leaf is None and (self.carve is not None or self.keep is not None):
            raise ValueError("carve and keep need the voxel map (leaf)")
        self.scan_wait_num = 0
        self.pcd_index = 0
        self.n_wait_save = 0

    def _accumulate(self, s, slot_tag) -> int:
        if self.leaf is None:
            return self.model.pcd_accumulate(s, slot_tag)
        if self.carve is None:
            return self.model.voxel_map_accumulate(s, slot_tag, self.leaf)
        return self.model.voxel_map_accumulate(s, slot_tag, self.leaf, carve=self.carve)

    def _save(self, path, clear):
        if self.leaf is None:
            self.model.pcd_save(path, clear=clear)
        elif self.keep is None:
            self.model.voxel_map_save(path, clear=clear)
        else:
            self.model.voxel_map_save(path, clear=clear, keep=self.keep)

    def after_update(self, s, slot_tag) -> str | None:
        """Once per scan after the update.  Returns the path written, if any."""
        self.n_wait_save = self._accumulate(s, slot_tag)                                   # :475
        self.scan_wait_num += 1
        if self.n_wait_save > 0 and self.interval > 0 and self.scan_wait_num > self.interval:   # :478
            self.pcd_index += 1
            path = os.path.join(self.directory, f"scans_{self.pcd_index}.pcd")
            self._save(path, clear=True)                                                   # :484-485
            self.n_wait_save = 0
            self.scan_wait_num = 0
            return path
        return None

    def finish(self) -> str | None:
        """At shutdown: result.pcd with whatever is still waiting (:1083-1091); nothing when the cloud is empty."""
        if self.n_wait_save == 0:
            return None
        path = os.path.join(self.directory, "result.pcd")
        self._save(path, clear=False)
        return path


class MeasurementModel:
    """One handle = one GPU.  Mirrors the life cycle of one scan in laserMapping.cpp:935-1082."""

    def __init__(self, n_lidar: int = 3, device: int = 0, sort_queries: bool = True, params: capi.Params | None = None,
                 knn_cell_size: float = 0.0):
        """knn_cell_size: edge of the k-NN fast path's cell-list index (0 automatic, < 0 off = ikd-Tree traversal only)."""
        self.lib = capi.load()
        cfg = capi.Config()
        cfg.params = params if params is not None else capi.default_params(n_lidar)
        cfg.params.n_lidar = n_lidar
        cfg.device = device
        self.device = device
        cfg.sort_queries = 1 if sort_queries else 0
        cfg.knn_cell_size = float(knn_cell_size)
        self.n_lidar = n_lidar
        self.n_dof = 17 + 6 * n_lidar
        self.n_cols = 6 * (n_lidar + 1)
        self._h = C.c_void_p()
        rc = self.lib.malio_create(C.byref(self._h), C.byref(cfg))
        if rc != capi.OK:
            raise capi.MalioError(rc, self.lib.malio_last_error(None).decode())
        self.n_points = 0
        self._slot_rows = {}   # rows of the last undistort*() per LiDAR slot (voxel_grid_tensor sizes its output by them)
        self._keep = []   # host buffers must outlive the (synchronous) calls only; kept for clarity

    def close(self):
        if self._h:
            self.lib.malio_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, allow=()):
        if rc != capi.OK and rc not in allow:
            raise capi.MalioError(rc, self.lib.malio_last_error(self._h).decode())
        return rc

    # ---- multi-GPU plumbing
    @staticmethod
    def nccl_unique_id() -> np.ndarray:
        uid = np.zeros(capi.NCCL_UNIQUE_ID_BYTES, dtype=np.uint8)
        rc = capi.load().malio_get_nccl_unique_id(capi.ptr(uid))
        if rc != capi.OK:
            raise capi.MalioError(rc, "malio_get_nccl_unique_id")
        return uid

    def comm_init(self, uid: np.ndarray, rank: int, world: int):
        uid = np.ascontiguousarray(uid, dtype=np.uint8)
        self._check(self.lib.malio_comm_init(self._h, capi.ptr(uid), rank, world))

    # ---- per scan
    def upload_map(self, snap: MapSnapshot):
        nodes = np.ascontiguousarray(snap.nodes)
        cov = np.ascontiguousarray(snap.node_cov, dtype=np.float32)
        self._check(self.lib.malio_upload_map(self._h, capi.ptr(nodes), capi.ptr(cov), nodes.shape[0], snap.max_depth))

    def upload_map_compact(self, snap: MapSnapshot, points: np.ndarray | None = None, root_box: np.ndarray | None = None):
        """Same snapshot, 16 bytes per node (point + link) + the weights: the device rebuilds the children's boxes.
        `points` may hold the pre-extracted capi.MAP_POINT array (e.g. in pinned memory); `root_box` the map's bounding
        box {x_min,x_max,y_min,y_max,z_min,z_max} when the caller knows it (the ikd-Tree root's node_range_*)."""
        pts = compact_points(snap.nodes) if points is None else points
        cov = np.ascontiguousarray(snap.node_cov, dtype=np.float32)
        rb = None if root_box is None else np.ascontiguousarray(root_box, dtype=np.float32)
        self._check(self.lib.malio_upload_map_compact(self._h, capi.ptr(pts), capi.ptr(cov), pts.shape[0], snap.max_depth,
                                                      capi.ptr(rb)))

    def download_map_nodes(self, n: int) -> np.ndarray:
        out = np.zeros(n, dtype=capi.MAP_NODE)
        self._check(self.lib.malio_download_map_nodes(self._h, capi.ptr(out), n))
        return out

    def upload_scan(self, pts: np.ndarray, table: np.ndarray, table_off: np.ndarray, temporal_comp: np.ndarray | None):
        pts = np.ascontiguousarray(pts)
        assert pts.dtype == capi.SCAN_PT
        table = np.ascontiguousarray(table)
        assert table.dtype == capi.POSE_ENTRY
        table_off = np.ascontiguousarray(table_off, dtype=np.uint32)
        tc = None if temporal_comp is None else np.ascontiguousarray(temporal_comp)
        self._check(self.lib.malio_upload_scan(self._h, capi.ptr(pts), pts.shape[0], capi.ptr(table),
                                               capi.ptr(table_off), capi.ptr(tc)))
        self.n_points = int(pts.shape[0])

    # ---- the map as a device-resident point set kept in step by deltas (SURVEY.md §8f N1; include/malio_mapsync.hpp)
    @staticmethod
    def _f32(a, cols=None):
        a = np.ascontiguousarray(a, np.float32)
        return a if cols is None else a.reshape(-1, cols)

    def map_build(self, xyz, normal_y, ids=None):
        """KD_TREE::Build: the device-resident map starts as these points (handle switches to device-map mode)."""
        xyz = self._f32(xyz, 3); ny = self._f32(normal_y)
        i = None if ids is None else np.ascontiguousarray(ids, np.int32)
        self._check(self.lib.malio_map_build(self._h, capi.ptr(xyz), capi.ptr(ny), capi.ptr(i), xyz.shape[0]))

    def map_add_points(self, xyz, normal_y, ids=None):
        """Mirror of KD_TREE::Add_Points(points, false)."""
        xyz = self._f32(xyz, 3); ny = self._f32(normal_y)
        i = None if ids is None else np.ascontiguousarray(ids, np.int32)
        self._check(self.lib.malio_map_add_points(self._h, capi.ptr(xyz), capi.ptr(ny), capi.ptr(i), xyz.shape[0]))

    def map_delete_boxes(self, boxes) -> int:
        """Mirror of KD_TREE::Delete_Point_Boxes; boxes: nb x {min3, max3}, half-open.  Returns the points deleted."""
        b = self._f32(boxes, 6)
        n = C.c_uint32(0)
        self._check(self.lib.malio_map_delete_boxes(self._h, capi.ptr(b), b.shape[0], C.byref(n)))
        return int(n.value)

    def map_sync_voxels(self, sync: dict, want_count: bool = True) -> int:
        """After the host tree's Add_Points(points, true): replace the content of every touched voxel box by what
        malio::collect_voxel_sync read back from the tree (dict with boxes, xyz, normal_y, ids).  want_count=False passes
        n_deleted = NULL: the call then returns without waiting for the device (-1 is returned)."""
        b = self._f32(sync["boxes"], 6); xyz = self._f32(sync["xyz"], 3); ny = self._f32(sync["normal_y"])
        i = None if sync.get("ids") is None else np.ascontiguousarray(sync["ids"], np.int32)
        n = C.c_uint32(0)
        self._check(self.lib.malio_map_sync_voxels(self._h, capi.ptr(b) if b.shape[0] else None, b.shape[0],
                                                   capi.ptr(xyz) if xyz.shape[0] else None, capi.ptr(ny) if xyz.shape[0] else None,
                                                   capi.ptr(i) if (i is not None and xyz.shape[0]) else None, xyz.shape[0],
                                                   C.byref(n) if want_count else None))
        return int(n.value) if want_count else -1

    def map_commit(self):
        self._check(self.lib.malio_map_commit(self._h))

    def map_info(self):
        a, b = C.c_uint32(0), C.c_uint32(0)
        self._check(self.lib.malio_map_info(self._h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def map_download(self):
        """Live points of the device-resident map in slot order: dict(xyz, normal_y, ids, slots)."""
        live, _ = self.map_info()
        xyz = np.zeros((live, 3), np.float32); ny = np.zeros(live, np.float32); ids = np.zeros(live, np.int32); sl = np.zeros(live, np.uint32)
        n = C.c_uint32(0)
        self._check(self.lib.malio_map_download(self._h, capi.ptr(xyz), capi.ptr(ny), capi.ptr(ids), capi.ptr(sl), live, C.byref(n)))
        return dict(xyz=xyz, normal_y=ny, ids=ids, slots=sl)

    # ---- the two stages before the path (SURVEY.md §8f N2, N3)
    def undistort(self, lidar: int, pts: np.ndarray, beg_time: float, extrinsic, lt_imu_frame, ctrl_t, ctrl_T, imu_cov_t,
                  cov_pointer: int, want_pose: bool = False):
        """UndistortPcl's per-point loop for one LiDAR (IMU_Processing.hpp:468-508).  pts: capi.RAW_PT[n] sorted by
        curvature; extrinsic / lt_imu_frame: (q wxyz, t).  Returns dict(xyz, idx, ok, pop_point, pose?)."""
        pts = np.ascontiguousarray(pts)
        assert pts.dtype == capi.RAW_PT
        n = pts.shape[0]
        a, cv, _keep = _undistort_args(beg_time, extrinsic, lt_imu_frame, ctrl_t, ctrl_T, imu_cov_t, cov_pointer)
        xyz = np.zeros((n, 3), np.float32); idx = np.zeros(n, np.int32); ok = np.zeros(n, np.uint8)
        pop = np.full(max(cv.shape[0], 1), -1, np.int32); npop = C.c_uint32(0)
        pose = np.zeros((n, 7)) if want_pose else None
        self._check(self.lib.malio_undistort(self._h, lidar, capi.ptr(pts), n, C.byref(a), capi.ptr(xyz), capi.ptr(idx), capi.ptr(ok),
                                             capi.ptr(pop), C.byref(npop), capi.ptr(pose)))
        self._slot_rows[lidar] = n
        return dict(xyz=xyz, idx=idx, ok=ok, pop_point=pop[: npop.value], pose=pose)

    def voxel_grid(self, lidar: int, pts5: np.ndarray | None, leaf: float):
        """pcl::VoxelGrid (laserMapping.cpp:968-983) on the device.  pts5: float32[n,5] {x,y,z,intensity,curvature}, or None to
        take the device-resident output of the last undistort() of this LiDAR slot.  Returns float32[m,5]."""
        n = 0 if pts5 is None else int(pts5.shape[0])
        inp = None if pts5 is None else np.ascontiguousarray(pts5, np.float32)
        m = C.c_uint32(0)
        self._check(self.lib.malio_voxel_grid(self._h, lidar, capi.ptr(inp), n, C.c_float(leaf), None, 0, C.byref(m)))
        out = np.zeros((m.value, 5), np.float32)
        if m.value:   # second call only fetches (the result is device-resident); kept simple: recompute with the output buffer
            self._check(self.lib.malio_voxel_grid(self._h, lidar, capi.ptr(inp), n, C.c_float(leaf), capi.ptr(out), m.value, C.byref(m)))
        return out

    def upload_scan_device(self, table: np.ndarray, table_off: np.ndarray, temporal_comp: np.ndarray | None) -> int:
        """Merge the device-resident down-sampled clouds of all LiDAR slots into the scan (no host bounce)."""
        table = np.ascontiguousarray(table); table_off = np.ascontiguousarray(table_off, dtype=np.uint32)
        tc = None if temporal_comp is None else np.ascontiguousarray(temporal_comp)
        n = C.c_uint32(0)
        self._check(self.lib.malio_upload_scan_device(self._h, capi.ptr(table), capi.ptr(table_off), capi.ptr(tc), C.byref(n)))
        self.n_points = int(n.value)
        return self.n_points

    def scan_uncertainty(self, imu_cov: np.ndarray, extrinsic: np.ndarray, uncertainty: np.ndarray, want_lists: bool = False):
        """The scan's pose-uncertainty lists, temporal compensation and pose_unc table (IMU_Processing.hpp:474-523,
        laserMapping.cpp:1028-1048) on the device, after undistort() has run on every slot 0..L-1.  imu_cov: float64[n_cov,6,6]
        (imu_cov[k].first.second, the list whose times undistort() got); extrinsic: capi.POSE[L] with the extrinsic
        uncertainty; uncertainty: float64[6,6] (kf.getUncertainty()).  Returns dict(table, table_off, temporal_comp capi.POSE[L-1],
        temporal_comp_rigid capi.RIGID[L-1] or None (what upload_scan* take), lidar_unc: list of capi.POSE arrays or None)."""
        L = self.n_lidar
        a, _keep = _scan_unc_args(imu_cov, extrinsic, uncertainty)
        cap = L * capi.MAX_COV
        table = np.zeros(cap, dtype=capi.POSE_ENTRY)
        off = np.zeros(L + 1, np.uint32)
        tc = np.zeros(max(L - 1, 1), dtype=capi.POSE)
        lists = np.zeros(cap, dtype=capi.POSE) if want_lists else None
        counts = np.zeros(L, np.uint32)
        self._check(self.lib.malio_scan_uncertainty(self._h, C.byref(a), capi.ptr(table), cap, capi.ptr(off), capi.ptr(tc),
                                                    capi.ptr(lists), capi.ptr(counts)))
        tc = tc[: L - 1]
        rigid = _rigid_of(tc)
        lu = None
        if want_lists:
            ends = np.cumsum(counts)
            lu = [lists[e - c:e].copy() for c, e in zip(counts.astype(np.int64), ends.astype(np.int64))]
        return dict(table=table[: off[L]].copy(), table_off=off, temporal_comp=tc, temporal_comp_rigid=rigid, lidar_unc=lu)

    # ---- after the update: publish_frame_world and the saved map (laserMapping.cpp:448-489)
    def publish_frame_world(self, s: capi.PassState | capi.State, dense: bool, slot_tag=None) -> np.ndarray:
        """The registered cloud of publish_frame_world (scan_pub_en) with the updated state: float32[n,4] {x, y, z, intensity}.
        dense=True: the undistorted clouds of slots 0..L-1 (feats_undistort), slot_tag[l] = the raw points' normal_y of slot l;
        dense=False: the down-sampled scan in caller order, intensity = normal_y of the last pass."""
        ps = s.pass_state() if isinstance(s, capi.State) else s
        src = capi.WORLD_DENSE if dense else capi.WORLD_DOWNSAMPLED
        tag = None if slot_tag is None else np.ascontiguousarray(slot_tag, np.float32)
        n = C.c_uint32(0)
        self._check(self.lib.malio_world_register(self._h, C.byref(ps), src, capi.ptr(tag), None, 0, C.byref(n)))
        out = np.zeros((n.value, 4), np.float32)
        if n.value:
            self._check(self.lib.malio_world_register(self._h, C.byref(ps), src, capi.ptr(tag), capi.ptr(out), n.value, C.byref(n)))
        return out

    def pcd_accumulate(self, s: capi.PassState | capi.State, slot_tag) -> int:
        """pcl_wait_save += the registered dense cloud (laserMapping.cpp:468-475), kept on the device.  Returns its size."""
        ps = s.pass_state() if isinstance(s, capi.State) else s
        tag = np.ascontiguousarray(slot_tag, np.float32)
        n = C.c_uint64(0)
        self._check(self.lib.malio_world_accumulate(self._h, C.byref(ps), capi.ptr(tag), C.byref(n)))
        return int(n.value)

    def pcd_save(self, path: str, clear: bool):
        """pcd_writer.writeBinary(path, *pcl_wait_save) (:484, :1090); clear=True also empties the cloud (:485)."""
        self._check(self.lib.malio_world_save_pcd(self._h, os.fsencode(path), 1 if clear else 0))

    # ---- the saved map as a voxel map (malio_world_voxel_*): pcl::VoxelGrid of the accumulated dense cloud, kept per voxel
    def voxel_map_accumulate(self, s: capi.PassState | capi.State, slot_tag, leaf: float, carve=None) -> int:
        """Fold the registered dense cloud into the device's voxel map (leaf in m, fixed by the first call after creation or a
        clearing save).  carve (None, True for the defaults, capi.CarveArgs or a dict of carve_args' keywords): also count this
        scan's hits and the voxels its rays pass (malio_world_voxel_accumulate_carve).  Returns the number of voxels."""
        leaf = _check_leaf(leaf)
        tag = np.ascontiguousarray(slot_tag, np.float32).reshape(-1)
        if tag.shape[0] != self.n_lidar:
            raise ValueError(f"slot_tag: {tag.shape[0]} values, expected one per LiDAR slot ({self.n_lidar})")
        ps = s.pass_state() if isinstance(s, capi.State) else s
        n = C.c_uint64(0)
        a = _as_carve(carve)
        if a is None:
            self._check(self.lib.malio_world_voxel_accumulate(self._h, C.byref(ps), capi.ptr(tag), C.c_float(leaf), C.byref(n)))
        else:
            self._check(self.lib.malio_world_voxel_accumulate_carve(self._h, C.byref(ps), capi.ptr(tag), C.c_float(leaf), C.byref(a),
                                                                    C.byref(n)))
        return int(n.value)

    def voxel_map_tensor(self, keep=None):
        """The voxel map's centroids as a CUDA tensor float32 (n, 4) {x, y, z, intensity} in ascending (z, y, x) voxel order,
        allocated on the current stream.  Returns once the sort and the copy are enqueued.  keep (None, True for the defaults,
        capi.CarveKeep or a dict of carve_keep's keywords): only the voxels the keep rule keeps (the call waits for their count)."""
        import torch
        n = C.c_uint64(0)
        st = torch.cuda.current_stream(self.device)
        self._check(self.lib.malio_world_voxel_download_device(self._h, None, 0, C.byref(n), st.cuda_stream))
        out = self._empty((n.value, 4), torch.float32)
        k = _as_keep(keep)
        if k is not None:
            cap = n.value
            self._check(self.lib.malio_world_voxel_download_kept_device(self._h, C.byref(k), _dptr(out) if cap else None, cap, C.byref(n),
                                                                        st.cuda_stream))
            return out[: n.value]
        if n.value:
            self._check(self.lib.malio_world_voxel_download_device(self._h, _dptr(out), n.value, C.byref(n), st.cuda_stream))
        return out

    def voxel_map_evidence_tensor(self):
        """The (hit, miss) counters as a CUDA tensor int32 (n, 2) (the u32 bits; a counter stays below 2^31 for 2^31 scans) in the
        order of voxel_map_tensor(), allocated on the current stream.  Zeros for a map that was never carved."""
        import torch
        n = C.c_uint64(0)
        st = torch.cuda.current_stream(self.device)
        self._check(self.lib.malio_world_voxel_evidence_device(self._h, None, 0, C.byref(n), st.cuda_stream))
        out = self._empty((n.value, 2), torch.int32)
        if n.value:
            self._check(self.lib.malio_world_voxel_evidence_device(self._h, _dptr(out), n.value, C.byref(n), st.cuda_stream))
        return out

    def voxel_map_save(self, path: str, clear: bool, keep=None):
        """The voxel map as a binary PCD file (the writer of pcd_save); clear=True also empties it, releases its leaf and resets
        the counters.  keep (as voxel_map_tensor): only the voxels the keep rule keeps."""
        k = _as_keep(keep)
        if k is None:
            self._check(self.lib.malio_world_voxel_save_pcd(self._h, os.fsencode(path), 1 if clear else 0))
        else:
            self._check(self.lib.malio_world_voxel_save_pcd_kept(self._h, os.fsencode(path), C.byref(k), 1 if clear else 0))

    def voxel_map_seed(self, xyzi, leaf: float, seed_hits: int = SEED_HITS) -> int:
        """Start the empty voxel map from saved points (float32 (n, 4) {x, y, z, intensity}, e.g. read_pcd of a kept file): the map
        one voxel_map_accumulate of these points would hold, each voxel starting at hit = seed_hits, miss = 0.  The seeded voxels
        are what voxel_map_changes compares against.  Returns the number of voxels."""
        leaf = _check_leaf(leaf)
        x = self._f32(xyzi, 4)
        n = C.c_uint64(0)
        self._check(self.lib.malio_world_voxel_seed(self._h, capi.ptr(x), x.shape[0], C.c_float(leaf), int(seed_hits), C.byref(n)))
        return int(n.value)

    def voxel_map_seed_tensor(self, xyzi, leaf: float, seed_hits: int = SEED_HITS) -> int:
        """voxel_map_seed from a contiguous float32 CUDA tensor (n, 4) on the handle's device, read in place, ordered on
        torch.cuda.current_stream().  Returns once the seed is done (its voxel count)."""
        import torch
        leaf = _check_leaf(leaf)
        _check_tensor(xyzi, "xyzi", torch.float32, 4, self.device)
        n = C.c_uint64(0)
        st = torch.cuda.current_stream(xyzi.device)
        self._check(self.lib.malio_world_voxel_seed_device(self._h, _dptr(xyzi), xyzi.shape[0], C.c_float(leaf), int(seed_hits),
                                                           C.byref(n), st.cuda_stream))
        return int(n.value)

    def voxel_map_changes(self, keep=True):
        """(removed, added) as CUDA tensors float32 (n, 4) in the order of voxel_map_tensor(): the seeded voxels the keep rule
        drops and the voxels not seeded that it keeps (keep as voxel_map_tensor's, the defaults when True), allocated on the
        current stream.  The call waits for the two counts."""
        import torch
        k = _as_keep(keep) or carve_keep()
        nr, na = C.c_uint64(0), C.c_uint64(0)
        st = torch.cuda.current_stream(self.device)
        self._check(self.lib.malio_world_voxel_changes_device(self._h, C.byref(k), None, 0, C.byref(nr), None, 0, C.byref(na),
                                                              st.cuda_stream))
        rem, add = self._empty((nr.value, 4), torch.float32), self._empty((na.value, 4), torch.float32)
        if nr.value or na.value:
            self._check(self.lib.malio_world_voxel_changes_device(self._h, C.byref(k), _dptr(rem), nr.value, C.byref(nr), _dptr(add),
                                                                  na.value, C.byref(na), st.cuda_stream))
        return rem, add

    def voxel_map_save_changes(self, removed_path: str | None, added_path: str | None, keep=True) -> tuple:
        """voxel_map_changes as two binary PCD files (None skips a file; an empty set writes none).  The map is not cleared.
        Returns (n_removed, n_added)."""
        k = _as_keep(keep) or carve_keep()
        nr, na = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.malio_world_voxel_save_changes_pcd(self._h, C.byref(k), None if removed_path is None else os.fsencode(removed_path),
                                                                None if added_path is None else os.fsencode(added_path),
                                                                C.byref(nr), C.byref(na)))
        return int(nr.value), int(na.value)

    def voxel_map_info(self) -> dict:
        """Voxels in use, entry capacity and the device bytes the voxel map holds."""
        v, c, b = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.malio_world_voxel_info(self._h, C.byref(v), C.byref(c), C.byref(b)))
        return dict(n_voxels=int(v.value), capacity=int(c.value), device_bytes=int(b.value))

    # ---- the scan store and the voxel map's rebuild from it (malio_scan_store_*, malio_world_voxel_rebuild)
    def scan_store_add(self, s: capi.PassState | capi.State, slot_tag, time: float = 0.0) -> int:
        """Keep the current dense cloud (the rows voxel_map_accumulate folds, LiDAR frame) on the device with state s, slot_tag
        and the caller's time stamp, so that a later voxel_map_rebuild can fold it again.  Returns the number of stored scans."""
        tag = np.ascontiguousarray(slot_tag, np.float32).reshape(-1)
        if tag.shape[0] != self.n_lidar:
            raise ValueError(f"slot_tag: {tag.shape[0]} values, expected one per LiDAR slot ({self.n_lidar})")
        ps = s.pass_state() if isinstance(s, capi.State) else s
        n = C.c_uint64(0)
        self._check(self.lib.malio_scan_store_add(self._h, C.byref(ps), capi.ptr(tag), C.c_double(time), C.byref(n)))
        return int(n.value)

    def scan_store_put(self, record: capi.StoredScan, xyz) -> int:
        """Append a stored scan: its record and its points, float32 (n, 3) with n = sum(record.n_points).  Returns the number of
        stored scans."""
        x = self._f32(xyz, 3)
        if x.shape[0] != sum(record.n_points):
            raise ValueError(f"xyz: {x.shape[0]} points, the record counts {sum(record.n_points)}")
        n = C.c_uint64(0)
        self._check(self.lib.malio_scan_store_put(self._h, C.byref(record), capi.ptr(x) if x.shape[0] else None, C.byref(n)))
        return int(n.value)

    def scan_store_get(self, k: int) -> tuple:
        """(record, xyz float32 (n, 3)) of stored scan k."""
        rec, n = capi.StoredScan(), C.c_uint64(0)
        self._check(self.lib.malio_scan_store_get(self._h, int(k), C.byref(rec), None, 0, C.byref(n)))
        xyz = np.zeros((n.value, 3), np.float32)
        if n.value:
            self._check(self.lib.malio_scan_store_get(self._h, int(k), None, capi.ptr(xyz), n.value, C.byref(n)))
        return rec, xyz

    def scan_store_records(self) -> list:
        """Every stored scan's record (copies: edit their states and pass them, or theirs, to voxel_map_rebuild)."""
        out = []
        for k in range(self.scan_store_info()["n_scans"]):
            rec, n = capi.StoredScan(), C.c_uint64(0)
            self._check(self.lib.malio_scan_store_get(self._h, k, C.byref(rec), None, 0, C.byref(n)))
            out.append(rec)
        return out

    def scan_store_register_tensor(self, k: int, state: capi.PassState | capi.State | None = None):
        """Stored scan k registered with `state` (None: its stored state) as a CUDA tensor float32 (n, 4) {x, y, z, slot_tag},
        the bits publish_frame_world(dense=True) gave for it; allocated and ordered on the current stream."""
        import torch
        ps = None if state is None else (state.pass_state() if isinstance(state, capi.State) else state)
        sp = None if ps is None else C.byref(ps)
        n = C.c_uint64(0)
        st = torch.cuda.current_stream(self.device)
        self._check(self.lib.malio_scan_store_register_device(self._h, int(k), sp, None, 0, C.byref(n), st.cuda_stream))
        out = self._empty((n.value, 4), torch.float32)
        if n.value:
            self._check(self.lib.malio_scan_store_register_device(self._h, int(k), sp, _dptr(out), n.value, C.byref(n), st.cuda_stream))
        return out

    def scan_store_info(self) -> dict:
        """Stored scans, stored points and the device bytes of the store's blocks."""
        s, p, b = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.malio_scan_store_info(self._h, C.byref(s), C.byref(p), C.byref(b)))
        return dict(n_scans=int(s.value), n_points=int(p.value), device_bytes=int(b.value))

    def scan_store_clear(self):
        """Release every stored scan."""
        self._check(self.lib.malio_scan_store_clear(self._h))

    def voxel_map_rebuild(self, leaf: float, states=None, first: int = 0, count: int | None = None, carve=None) -> int:
        """Fold stored scans [first, first + count) into the voxel map again, as voxel_map_accumulate of each in index order
        would, each under states[k - first] (capi.PassState or capi.State; None: the stored states) with its stored slot tags
        and temporal compensation.  count None: every scan from first on.  carve as voxel_map_accumulate's.  Clear the map
        first (voxel_map_save(.., clear=True)) for a fresh map.  Returns the number of voxels."""
        leaf = _check_leaf(leaf)
        if count is None:
            count = max(self.scan_store_info()["n_scans"] - int(first), 0)
        arr = None
        if states is not None:
            states = list(states)
            if len(states) != count:
                raise ValueError(f"states: {len(states)} states for {count} scans")
            arr = (capi.PassState * max(count, 1))()
            for i, s in enumerate(states):
                arr[i] = s.pass_state() if isinstance(s, capi.State) else s
        a = _as_carve(carve)
        n = C.c_uint64(0)
        self._check(self.lib.malio_world_voxel_rebuild(self._h, int(first), int(count), arr, C.c_float(leaf),
                                                       None if a is None else C.byref(a), C.byref(n)))
        return int(n.value)

    def scan_store_match(self, source: int, anchor: int, guess: capi.PassState | capi.State | None = None, **args) -> dict:
        """Register stored scan `source` against a submap of stored scans on the device (malio_scan_store_match), starting from
        guess (None: the source's stored state).  args: match_args' keywords (target_first / target_count default to anchor
        +- half_window).  Returns the report as a dict: rot, pos, rel_rot, rel_pos (the loop edge T_anchor^-1 T_est), info
        (6 x 6), rms, fitness, eig_min, n_points, n_inliers, iterations, converged, target_points, target_voxels, device_bytes,
        and the call's source, anchor and sigma."""
        half = int(args.pop("half_window", MATCH_HALF_WINDOW))
        if "target_first" not in args:
            n = self.scan_store_info()["n_scans"]
            args["target_first"] = max(int(anchor) - half, 0)
            args["target_count"] = min(int(anchor) + half + 1, n) - args["target_first"]
        a = match_args(**args)
        ps = None if guess is None else (guess.pass_state() if isinstance(guess, capi.State) else guess)
        rep = capi.MatchReport()
        self._check(self.lib.malio_scan_store_match(self._h, int(source), int(anchor), None if ps is None else C.byref(ps), C.byref(a),
                                                    C.byref(rep)))
        L = a.n_levels
        return dict(rot=np.array(rep.rot[:]), pos=np.array(rep.pos[:]), rel_rot=np.array(rep.rel_rot[:]), rel_pos=np.array(rep.rel_pos[:]),
                    info=np.array(rep.info[:]).reshape(6, 6), rms=rep.rms, fitness=rep.fitness, eig_min=rep.eig_min,
                    n_points=int(rep.n_points), n_inliers=int(rep.n_inliers), iterations=[int(v) for v in rep.iterations[:L]],
                    converged=bool(rep.converged), target_points=int(rep.target_points),
                    target_voxels=[int(v) for v in rep.target_voxels[:L]], device_bytes=int(rep.device_bytes),
                    source=int(source), anchor=int(anchor), sigma=float(a.sigma))

    # ---- a 2-D occupancy grid for navigation (malio_grid_*)
    def _grid_source(self, source, xyzi, keep):
        """(source code, device pointer, rows, CarveKeep or None, the current stream) of grid / grid_extent's arguments."""
        import torch
        if source not in GRID_SOURCES:
            raise ValueError(f"source: {source!r}, expected one of {sorted(GRID_SOURCES)}")
        src = GRID_SOURCES[source]
        if (xyzi is not None) != (src == capi.GRID_POINTS):
            raise ValueError("xyzi is the 'points' source's input and only its")
        if keep is not None and src != capi.GRID_VOXEL_MAP:
            raise ValueError("keep applies to the 'voxel_map' source only")
        if xyzi is not None:
            _check_tensor(xyzi, "xyzi", torch.float32, 4, self.device)
        k = _as_keep(keep)
        return src, _dptr(xyzi), 0 if xyzi is None else xyzi.shape[0], k, torch.cuda.current_stream(self.device)

    def grid_extent(self, source: str = "voxel_map", xyzi=None, keep=None, res: float = GRID_RES) -> tuple:
        """(imin, jmin, imax, jmax): the column indices floorf(x / res) of the source's finite points ((0, 0, -1, -1) when there are
        none).  source: "points" (xyzi a float32 CUDA tensor (n, 4)), "voxel_map" (keep as voxel_map_tensor's) or "prior"."""
        src, p, n, k, st = self._grid_source(source, xyzi, keep)
        ext = np.zeros(4, np.int32)
        self._check(self.lib.malio_grid_extent_device(self._h, src, p, n, None if k is None else C.byref(k), C.c_float(res),
                                                      capi.ptr(ext), st.cuda_stream))
        return tuple(int(v) for v in ext)

    def grid(self, source: str = "voxel_map", xyzi=None, keep=None, args: capi.GridArgs | None = None):
        """The occupancy grid of a source on the device: (cls, ground, report).  cls uint8 (ny, nx) (GRID_FREE / GRID_OCCUPIED /
        GRID_UNKNOWN, row r at cell row j0 + r), ground float32 (ny, nx) (NaN where no point lies within the ground window), both
        CUDA tensors on the current stream; report a dict of malio_grid_report.  source and keep as grid_extent's; args from
        grid_args, or None for the defaults over the whole extent of the source (with nx or ny 0 the extent fills the region)."""
        import torch
        src, p, n, k, st = self._grid_source(source, xyzi, keep)
        a = grid_args() if args is None else args
        if a.nx == 0 or a.ny == 0:
            lo_i, lo_j, hi_i, hi_j = self.grid_extent(source, xyzi, keep, a.res)
            if hi_i < lo_i:
                raise ValueError("the source has no finite point: give the region in args")
            a = grid_args(a.res, lo_i, lo_j, hi_i - lo_i + 1, hi_j - lo_j + 1, a.ground_halfwidth, a.h_lo, a.h_hi, a.min_obstacle_points)
        cls, ground = self._empty((a.ny, a.nx), torch.uint8), self._empty((a.ny, a.nx), torch.float32)
        rep = capi.GridReport()
        self._check(self.lib.malio_grid_build_device(self._h, src, p, n, None if k is None else C.byref(k), C.byref(a), _dptr(cls),
                                                     _dptr(ground), st.cuda_stream, C.byref(rep)))
        r = _grid_report(rep)
        r["args"] = a
        return cls, ground, r

    def grid_host(self, xyzi, args: capi.GridArgs, want_ground: bool = True):
        """malio_grid_build: the grid of host points (float32 (n, 4)) into numpy arrays (cls, ground or None, report)."""
        x = self._f32(xyzi, 4)
        cls = np.empty((args.ny, args.nx), np.uint8)
        ground = np.empty((args.ny, args.nx), np.float32) if want_ground else None
        rep = capi.GridReport()
        self._check(self.lib.malio_grid_build(self._h, capi.ptr(x), x.shape[0], C.byref(args), capi.ptr(cls), capi.ptr(ground), C.byref(rep)))
        return cls, ground, _grid_report(rep)

    # ---- localization in a saved map (malio_prior_map_*): the prior on the device and lasermap_fov_segment's window over it
    def prior_map_load(self, xyz, normal_y=0.001, ids=None):
        """Load the prior map (replaces the previous one and ends the window).  xyz float32 (n, 3); normal_y a scalar (the map-side
        weight build_static_snapshot uses by default) or (n,); ids int32 (n,) or None (0..n-1)."""
        xyz = self._f32(xyz, 3)
        n = xyz.shape[0]
        ny = np.full(n, normal_y, np.float32) if np.isscalar(normal_y) else self._f32(normal_y)
        if ny.shape[0] != n:
            raise ValueError(f"normal_y: {ny.shape[0]} values for {n} points")
        i = None if ids is None else np.ascontiguousarray(ids, np.int32)
        if i is not None and i.shape[0] != n:
            raise ValueError(f"ids: {i.shape[0]} values for {n} points")
        self._check(self.lib.malio_prior_map_load(self._h, capi.ptr(xyz), capi.ptr(ny), capi.ptr(i), n))

    def prior_map_load_tensor(self, xyz, normal_y, ids=None):
        """prior_map_load from CUDA tensors (as map_build_tensor), read in place, ordered on torch.cuda.current_stream()."""
        self._map_tensor("malio_prior_map_load_device", xyz, normal_y, ids)

    def prior_map_window(self, pos_or_state, cube_len: float = 1000.0, det_range: float = 100.0) -> dict:
        """lasermap_fov_segment (laserMapping.cpp:171-224) on the device map over the prior.  pos_or_state: pos_lid (3 floats) or a
        capi.State (pos_lid computed as at :1056).  Returns the report as a dict: initialized, moved, cube float32 (6,), boxes
        float32 (n_boxes, 6), n_killed, n_entered, n_live."""
        p = pos_lid(pos_or_state) if isinstance(pos_or_state, capi.State) else np.ascontiguousarray(pos_or_state, np.float64).reshape(3)
        p = np.ascontiguousarray(p, np.float64)
        rep = capi.WindowReport()
        self._check(self.lib.malio_prior_map_window(self._h, capi.ptr(p), C.c_double(cube_len), C.c_float(det_range), C.byref(rep)))
        return dict(initialized=bool(rep.initialized), moved=bool(rep.moved), cube=np.array(rep.cube[:], np.float32),
                    boxes=np.array(rep.boxes[:6 * rep.n_boxes], np.float32).reshape(-1, 6),
                    n_killed=int(rep.n_killed), n_entered=int(rep.n_entered), n_live=int(rep.n_live))

    def prior_map_info(self) -> dict:
        """Points and occupied tiles of the prior, and the device bytes the prior and its window's scratch hold."""
        n, t, b = C.c_uint64(0), C.c_uint32(0), C.c_uint64(0)
        self._check(self.lib.malio_prior_map_info(self._h, C.byref(n), C.byref(t), C.byref(b)))
        return dict(n_points=int(n.value), n_tiles=int(t.value), device_bytes=int(b.value))

    def prior_map_clear(self):
        """Release the prior; the device map keeps its points."""
        self._check(self.lib.malio_prior_map_clear(self._h))

    def prior_map_extend(self, state: capi.PassState | capi.State, filter_size_map: float = 0.5) -> dict:
        """malio_prior_map_extend: map_incremental in localization mode, with the state after the update.  The scan's candidates
        whose voxel box holds no live point of the window are folded and added to the session (and to the window where they lie
        inside the cube).  Returns the report as a dict: n_candidates, n_admitted, n_inserted, n_session."""
        ps = state.pass_state() if isinstance(state, capi.State) else state
        rep = capi.ExtendReport()
        self._check(self.lib.malio_prior_map_extend(self._h, C.byref(ps), C.c_double(filter_size_map), C.byref(rep)))
        return dict(n_candidates=int(rep.n_candidates), n_admitted=int(rep.n_admitted), n_inserted=int(rep.n_inserted),
                    n_session=int(rep.n_session))

    def prior_map_session(self) -> np.ndarray:
        """The session's points as float32 (n, 4) {x, y, z, normal_y} in session order (point k has id -1 - k)."""
        n = C.c_uint64(0)
        self._check(self.lib.malio_prior_map_session_download(self._h, None, 0, C.byref(n)))
        out = np.zeros((n.value, 4), np.float32)
        if n.value:
            self._check(self.lib.malio_prior_map_session_download(self._h, capi.ptr(out), n.value, C.byref(n)))
        return out

    def relocalize(self, guess: capi.State | capi.PassState, res: float, half_xy: int, half_z: int, n_yaw: int = 360,
                   yaw_lo: float = 0.0, yaw_step: float | None = None) -> dict:
        """malio_relocalize: the best of n_yaw yaws (yaw_lo + k * yaw_step, default step 2 pi / n_yaw) about the prior's z axis after
        guess.rot, and of the integer voxel offsets (a, b) in [-half_xy, half_xy]^2, c in [-half_z, half_z] (steps of res metres)
        around guess.pos, scored against the loaded prior with the resident scan.  Returns the report's fields as a dict and
        `state`: a copy of guess with rot and pos replaced, ready for prior_map_window and update_iterated_dyn_share_modified."""
        ps = guess.pass_state() if isinstance(guess, capi.State) else guess
        a = capi.RelocArgs()
        a.n_yaw = int(n_yaw)
        a.yaw_lo = float(yaw_lo)
        a.yaw_step = 2.0 * math.pi / max(a.n_yaw, 1) if yaw_step is None else float(yaw_step)
        a.res, a.half_xy, a.half_z = float(res), int(half_xy), int(half_z)
        rep = capi.RelocReport()
        self._check(self.lib.malio_relocalize(self._h, C.byref(ps), C.byref(a), C.byref(rep)))
        state = type(guess)()
        C.memmove(C.byref(state), C.byref(guess), C.sizeof(guess))
        state.rot[:] = rep.rot[:]
        state.pos[:] = rep.pos[:]
        return dict(rot=np.array(rep.rot[:]), pos=np.array(rep.pos[:]), yaw_index=int(rep.yaw_index),
                    offset=tuple(int(v) for v in rep.offset), score=int(rep.score), n_points=int(rep.n_points),
                    n_candidates=int(rep.n_candidates), nodes_bounded=int(rep.nodes_bounded),
                    leaves_scored=int(rep.leaves_scored), device_bytes=int(rep.device_bytes), state=state)

    @staticmethod
    def place_args(sensor_height: float, cell: float = 1.0, step: float = 1.0, r_max: float = 60.0, n_ring: int = 20,
                   n_sector: int = 72, z_lo: float | None = None, dz: float = 1.0, fov_up: float = math.pi / 2,
                   block_level: int = 2) -> capi.PlaceArgs:
        """malio_place_args with the defaults of the header; z_lo defaults to -sensor_height + 0.5 (the ground is empty), fov_up
        to no cap."""
        a = capi.PlaceArgs()
        a.cell, a.step, a.r_max, a.n_ring, a.n_sector = float(cell), float(step), float(r_max), int(n_ring), int(n_sector)
        a.sensor_height = float(sensor_height)
        a.z_lo = -float(sensor_height) + 0.5 if z_lo is None else float(z_lo)
        a.dz, a.fov_up, a.block_level = float(dz), float(fov_up), int(block_level)
        return a

    def place_db_build(self, sensor_height: float | None = None, args: capi.PlaceArgs | None = None, **kw) -> dict:
        """malio_place_db_build: describe every lattice position of the loaded prior (place_args(sensor_height, **kw), or args).
        Returns the report's fields as a dict."""
        a = args if args is not None else self.place_args(sensor_height, **kw)
        rep = capi.PlaceDbReport()
        self._check(self.lib.malio_place_db_build(self._h, C.byref(a), C.byref(rep)))
        return {f: int(getattr(rep, f)) for f, _ in capi.PlaceDbReport._fields_}

    def place_db_info(self) -> dict:
        n, b = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.malio_place_db_info(self._h, C.byref(n), C.byref(b)))
        return dict(n_positions=int(n.value), device_bytes=int(b.value))

    def place_db_download(self, n_ring: int, n_sector: int) -> dict:
        """The database (test / debug): cols (n, 2), z_s (n,), nibbles (n, bytes per position), ring_keys (n, n_ring)."""
        n = C.c_uint64(0)
        self._check(self.lib.malio_place_db_download(self._h, None, None, None, None, 0, C.byref(n)))
        m = int(n.value)
        cols, zs = np.zeros((m, 2), np.int32), np.zeros(m, np.float64)
        nib, rk = np.zeros((m, (n_ring * n_sector + 1) // 2), np.uint8), np.zeros((m, n_ring), np.uint16)
        self._check(self.lib.malio_place_db_download(self._h, capi.ptr(cols), capi.ptr(zs), capi.ptr(nib), capi.ptr(rk), m, C.byref(n)))
        return dict(cols=cols, z_s=zs, nibbles=nib, ring_keys=rk)

    def relocalize_global(self, guess: capi.State | capi.PassState, k1: int = 256, k2: int = 8, yaw_step: float = math.radians(1.0),
                          res: float = 0.5, half_xy: int | None = None, half_z: int = 2, step: float = 1.0) -> dict:
        """malio_relocalize_global: the resident scan against the place database, the k2 best places each checked by
        malio_relocalize.  guess supplies the tilt and the extrinsics (its position and yaw do not matter); half_xy defaults to
        ceil(step / (2 res)) + 2 with step the database's lattice step.  Returns the report's fields as a dict, the candidates as a
        list of dicts, and `state`: a copy of guess with rot and pos replaced, ready for prior_map_window and the update."""
        ps = guess.pass_state() if isinstance(guess, capi.State) else guess
        a = capi.GlobalArgs()
        a.k1, a.k2, a.yaw_step, a.res = int(k1), int(k2), float(yaw_step), float(res)
        a.half_xy = int(math.ceil(step / (2 * res)) + 2) if half_xy is None else int(half_xy)
        a.half_z = int(half_z)
        rep = capi.GlobalReport()
        self._check(self.lib.malio_relocalize_global(self._h, C.byref(ps), C.byref(a), C.byref(rep)))
        state = type(guess)()
        C.memmove(C.byref(state), C.byref(guess), C.sizeof(guess))
        state.rot[:] = rep.rot[:]
        state.pos[:] = rep.pos[:]
        cand = []
        for c in rep.cand[:rep.n_candidates]:
            cand.append(dict(position=int(c.position), shift=int(c.shift), d1=int(c.d1), d2=int(c.d2), col=tuple(c.col[:]),
                             z_s=float(c.z_s), guess_rot=np.array(c.guess_rot[:]), guess_pos=np.array(c.guess_pos[:]),
                             rot=np.array(c.rot[:]), pos=np.array(c.pos[:]), score=int(c.score), n_points=int(c.n_points)))
        v = rep.verify
        return dict(rot=np.array(rep.rot[:]), pos=np.array(rep.pos[:]), score=int(rep.score), n_points=int(rep.n_points),
                    best_rank=int(rep.best_rank), n_candidates=int(rep.n_candidates), n_stage1=int(rep.n_stage1),
                    verify=dict(yaw_lo=v.yaw_lo, yaw_step=v.yaw_step, n_yaw=int(v.n_yaw), res=v.res, half_xy=int(v.half_xy),
                                half_z=int(v.half_z)),
                    cand=cand, stage1=np.array(rep.stage1[:rep.n_stage1], np.int64),
                    stage1_d1=np.array(rep.stage1_d1[:rep.n_stage1], np.int64), query=np.array(rep.query[:], np.uint8),
                    ms_rank=float(rep.ms_rank), ms_verify=float(rep.ms_verify), device_bytes=int(rep.device_bytes), state=state)

    def rearm_scan(self):
        """Reset the per-scan state of the scan already resident on the device (no host copy)."""
        self._check(self.lib.malio_rearm_scan(self._h))

    def set_timing(self, enable: bool):
        """Per-pass CUDA-event timing (PassStats.ms_*, Counters.knn_ms); on by default."""
        self._check(self.lib.malio_set_timing(self._h, 1 if enable else 0))

    def counters(self) -> capi.Counters:
        c = capi.Counters()
        self._check(self.lib.malio_get_counters(self._h, C.byref(c)))
        return c

    def h_share_model(self, s: capi.PassState | capi.State, converge: bool):
        """One measurement pass.  Returns (valid, HTH[c,c], HTh[c], stats)."""
        ps = s.pass_state() if isinstance(s, capi.State) else s
        c = self.n_cols
        HTH = np.zeros((c, c))
        HTh = np.zeros(c)
        st = capi.PassStats()
        rc = self._check(self.lib.malio_measure(self._h, C.byref(ps), 1 if converge else 0, capi.ptr(HTH),
                                                capi.ptr(HTh), C.byref(st)), allow=(capi.ERR_NO_EFFECTIVE_POINTS,))
        return rc == capi.OK, HTH, HTh, st

    def rows(self, cap: int | None = None):
        cap = capi.MAX_DOF if cap is None else cap
        hx = np.zeros((cap, self.n_cols))
        hv = np.zeros(cap)
        n = C.c_uint32(0)
        self._check(self.lib.malio_download_rows(self._h, capi.ptr(hx), capi.ptr(hv), cap, C.byref(n)))
        return hx[: n.value], hv[: n.value]

    def aux(self, normal_y=True, nn_idx=True, nn_sqdist=True, selected=True, world=True, out: dict | None = None):
        """Side outputs of the last pass in caller order.  `out` may carry pre-allocated (e.g. pinned) arrays under the
        same keys; missing ones are allocated."""
        n = self.n_points
        if out is not None:
            self._check(self.lib.malio_download_aux(self._h, capi.ptr(out.get("normal_y")), capi.ptr(out.get("nn_idx")),
                                                    capi.ptr(out.get("nn_sqdist")), capi.ptr(out.get("selected")),
                                                    capi.ptr(out.get("world"))))
            return out
        o_ny = np.zeros(n, np.float32) if normal_y else None
        o_idx = np.zeros((n, capi.K), np.uint32) if nn_idx else None
        o_d2 = np.zeros((n, capi.K), np.float32) if nn_sqdist else None
        o_sel = np.zeros(n, np.uint8) if selected else None
        o_w = np.zeros((n, 3), np.float32) if world else None
        self._check(self.lib.malio_download_aux(self._h, capi.ptr(o_ny), capi.ptr(o_idx), capi.ptr(o_d2),
                                                capi.ptr(o_sel), capi.ptr(o_w)))
        return dict(normal_y=o_ny, nn_idx=o_idx, nn_sqdist=o_d2, selected=o_sel, world=o_w)

    def map_incremental(self, s: capi.PassState | capi.State, filter_size_map: float = 0.5, ekf_inited: bool = True,
                        world: bool = True):
        """map_incremental's per-point decision (laserMapping.cpp:398-446) with the state after the update.
        Returns (cls uint8[N] with capi.MAP_* codes, feats_down_world float32[N,3] or None)."""
        ps = s.pass_state() if isinstance(s, capi.State) else s
        cls = np.zeros(self.n_points, np.uint8)
        w = np.zeros((self.n_points, 3), np.float32) if world else None
        self._check(self.lib.malio_map_incremental(self._h, C.byref(ps), C.c_double(filter_size_map), 1 if ekf_inited else 0,
                                                   capi.ptr(cls), capi.ptr(w)))
        return cls, w

    def update_iterated_dyn_share_modified(self, x: capi.State, P: np.ndarray, max_iter: int, R: float = 0.001):
        """IESKF update; x and P are updated in place.  Returns the report (status in report.last_status)."""
        assert P.shape == (self.n_dof, self.n_dof) and P.dtype == np.float64 and P.flags["C_CONTIGUOUS"]
        rep = capi.UpdateReport()
        rc = self.lib.malio_ieskf_update(self._h, C.byref(x), capi.ptr(P), max_iter, R, C.byref(rep))
        self._check(rc, allow=(capi.ERR_NO_EFFECTIVE_POINTS,))
        return rep

    # ---- stand-alone k-NN (BASELINE config C5)
    def Nearest_Search(self, queries: np.ndarray):
        q = np.ascontiguousarray(queries, dtype=np.float32)
        n = q.shape[0]
        idx = np.zeros((n, capi.K), np.uint32)
        d2 = np.zeros((n, capi.K), np.float32)
        ms = C.c_float(0)
        self._check(self.lib.malio_knn(self._h, capi.ptr(q), n, capi.ptr(idx), capi.ptr(d2), C.byref(ms)))
        return idx, d2, float(ms.value)

    # ---- the same on torch CUDA tensors: no host copy, ordered on torch.cuda.current_stream() (malio_knn_device & co.)
    def knn_tensor(self, q):
        """Nearest_Search on a contiguous float32 CUDA tensor (n, 3) on the handle's device.  Returns (idx int32 (n, 5), sqdist
        float32 (n, 5)), allocated on and ordered with the current stream; idx holds the bits of the uint32 indices, so a missing
        neighbour reads -1.  Returns once the search is enqueued; a traversal fault is reported by the next call on the model."""
        import torch
        _check_tensor(q, "q", torch.float32, 3, self.device)
        n = q.shape[0]
        idx = torch.empty((n, capi.K), dtype=torch.int32, device=q.device)
        d2 = torch.empty((n, capi.K), dtype=torch.float32, device=q.device)
        st = torch.cuda.current_stream(q.device)
        self._check(self.lib.malio_knn_device(self._h, _dptr(q), n, _dptr(idx), _dptr(d2), st.cuda_stream))
        return idx, d2

    def map_build_tensor(self, xyz, normal_y, ids=None):
        """map_build from CUDA tensors: xyz float32 (n, 3), normal_y float32 (n,), ids int32 (n,) or None, contiguous, on the
        handle's device; read in place, ordered on torch.cuda.current_stream()."""
        self._map_tensor("malio_map_build_device", xyz, normal_y, ids)

    def map_add_points_tensor(self, xyz, normal_y, ids=None):
        """map_add_points from CUDA tensors (as map_build_tensor); returns once the append is enqueued."""
        self._map_tensor("malio_map_add_points_device", xyz, normal_y, ids)

    def _map_tensor(self, name, xyz, normal_y, ids):
        import torch
        _check_tensor(xyz, "xyz", torch.float32, 3, self.device)
        n = xyz.shape[0]
        _check_tensor(normal_y, "normal_y", torch.float32, None, self.device, n)
        if ids is not None:
            _check_tensor(ids, "ids", torch.int32, None, self.device, n)
        st = torch.cuda.current_stream(xyz.device)
        self._check(getattr(self.lib, name)(self._h, _dptr(xyz), _dptr(normal_y), _dptr(ids), n, st.cuda_stream))

    # ---- the measurement path on torch CUDA tensors: the scan in, the per-point outputs out, ordered on
    # torch.cuda.current_stream() (malio_upload_scan_from_device & co.)
    def upload_scan_tensor(self, pts, table: np.ndarray, table_off: np.ndarray, temporal_comp: np.ndarray | None):
        """upload_scan from a contiguous int32 CUDA tensor (n, 4) of malio_scan_pt records (pack_scan_tensor builds them) on the
        handle's device; table / table_off / temporal_comp are host arrays as for upload_scan.  The records are copied into the
        handle, so pts may be reused afterwards.  Waits until the current stream has reached the call (a record with
        lidar >= n_lidar is rejected before the resident scan changes)."""
        import torch
        _check_tensor(pts, "pts", torch.int32, 4, self.device)
        table = np.ascontiguousarray(table)
        assert table.dtype == capi.POSE_ENTRY
        table_off = np.ascontiguousarray(table_off, dtype=np.uint32)
        tc = None if temporal_comp is None else np.ascontiguousarray(temporal_comp)
        n = pts.shape[0]
        st = torch.cuda.current_stream(pts.device)
        self._check(self.lib.malio_upload_scan_from_device(self._h, _dptr(pts), n, capi.ptr(table), capi.ptr(table_off),
                                                           capi.ptr(tc), st.cuda_stream))
        self.n_points = int(n)

    def _empty(self, shape, dtype, want=True):
        import torch
        return torch.empty(shape, dtype=dtype, device=torch.device("cuda", self.device)) if want else None

    def aux_tensor(self, normal_y=True, nn_idx=True, nn_sqdist=True, selected=True, world=True):
        """aux() into CUDA tensors allocated on the current stream: normal_y float32 (n,), nn_idx int32 (n, 5) (the bits of the
        uint32 indices: a missing neighbour reads -1), nn_sqdist float32 (n, 5), selected uint8 (n,), world float32 (n, 3); the
        ones not asked for are None.  Returns once the scatter is enqueued."""
        import torch
        n = self.n_points
        o = dict(normal_y=self._empty((n,), torch.float32, normal_y), nn_idx=self._empty((n, capi.K), torch.int32, nn_idx),
                 nn_sqdist=self._empty((n, capi.K), torch.float32, nn_sqdist), selected=self._empty((n,), torch.uint8, selected),
                 world=self._empty((n, 3), torch.float32, world))
        st = torch.cuda.current_stream(self.device)
        self._check(self.lib.malio_download_aux_device(self._h, _dptr(o["normal_y"]), _dptr(o["nn_idx"]), _dptr(o["nn_sqdist"]),
                                                       _dptr(o["selected"]), _dptr(o["world"]), st.cuda_stream))
        return o

    def map_incremental_tensor(self, s: capi.PassState | capi.State, filter_size_map: float = 0.5, ekf_inited: bool = True,
                               world: bool = True):
        """map_incremental() into CUDA tensors: (cls uint8 (n,) with capi.MAP_* codes, feats_down_world float32 (n, 3) or None).
        Returns once the kernel is enqueued on the current stream."""
        import torch
        ps = s.pass_state() if isinstance(s, capi.State) else s
        cls = self._empty((self.n_points,), torch.uint8)
        w = self._empty((self.n_points, 3), torch.float32, world)
        st = torch.cuda.current_stream(self.device)
        self._check(self.lib.malio_map_incremental_device(self._h, C.byref(ps), C.c_double(filter_size_map), 1 if ekf_inited else 0,
                                                          _dptr(cls), _dptr(w), st.cuda_stream))
        return cls, w

    def publish_frame_world_tensor(self, s: capi.PassState | capi.State, dense: bool, slot_tag=None):
        """publish_frame_world() into a CUDA tensor float32 (n, 4) {x, y, z, intensity}, allocated on the current stream.  Returns
        once the registration is enqueued."""
        import torch
        ps = s.pass_state() if isinstance(s, capi.State) else s
        src = capi.WORLD_DENSE if dense else capi.WORLD_DOWNSAMPLED
        tag = None if slot_tag is None else np.ascontiguousarray(slot_tag, np.float32)
        n = C.c_uint32(0)
        st = torch.cuda.current_stream(self.device)
        self._check(self.lib.malio_world_register_device(self._h, C.byref(ps), src, capi.ptr(tag), None, 0, C.byref(n), st.cuda_stream))
        out = self._empty((n.value, 4), torch.float32)
        if n.value:
            self._check(self.lib.malio_world_register_device(self._h, C.byref(ps), src, capi.ptr(tag), _dptr(out), n.value, C.byref(n),
                                                             st.cuda_stream))
        return out

    # ---- the front half of a scan on torch CUDA tensors: raw clouds in, the pose table kept on the device, ordered on
    # torch.cuda.current_stream() (malio_undistort_device & co.)
    UNDISTORT_OUTPUTS = ("cloud", "idx", "ok", "pop_point", "pose")

    def undistort_tensor(self, lidar: int, pts, beg_time: float, extrinsic, lt_imu_frame, ctrl_t, ctrl_T, imu_cov_t, cov_pointer: int,
                         want=UNDISTORT_OUTPUTS):
        """undistort() of a contiguous float32 CUDA tensor (n, 4) {x, y, z, curvature} on the handle's device, sorted by
        curvature and read in place; the other arguments are host values as for undistort().  Returns a dict with n_pops and the
        tensors named in `want`: cloud float32 (n, 5) {x, y, z, idx as float (0 where untouched), curvature} — the rows
        voxel_grid_tensor takes —, idx int32 (n,), ok uint8 (n,), pop_point int32 (n_pops,), pose float64 (n, 7).  Waits once, at
        its end, for the pop count and the time-order check; an unordered cloud raises MalioError (ERR_INVALID_ARG) and leaves
        the slot without a result until it is undistorted again."""
        import torch
        _check_tensor(pts, "pts", torch.float32, 4, self.device)
        unknown = set(want) - set(self.UNDISTORT_OUTPUTS)
        if unknown:
            raise ValueError(f"want: unknown outputs {sorted(unknown)}")
        n = pts.shape[0]
        a, cv, _keep = _undistort_args(beg_time, extrinsic, lt_imu_frame, ctrl_t, ctrl_T, imu_cov_t, cov_pointer)
        o = dict(cloud=self._empty((n, 5), torch.float32, "cloud" in want), idx=self._empty((n,), torch.int32, "idx" in want),
                 ok=self._empty((n,), torch.uint8, "ok" in want), pop_point=self._empty((cv.shape[0],), torch.int32, "pop_point" in want),
                 pose=self._empty((n, 7), torch.float64, "pose" in want))
        npop = C.c_uint32(0)
        st = torch.cuda.current_stream(pts.device)
        self._check(self.lib.malio_undistort_device(self._h, lidar, _dptr(pts), n, C.addressof(a), _dptr(o["cloud"]), _dptr(o["idx"]),
                                                    _dptr(o["ok"]), _dptr(o["pop_point"]), _dptr(o["pose"]), C.addressof(npop),
                                                    st.cuda_stream))
        self._slot_rows[lidar] = n
        out = {k: v for k, v in o.items() if k in want}
        if "pop_point" in want:
            out["pop_point"] = o["pop_point"][: npop.value]   # (an empty cloud writes nothing: no pop, an empty slice)
        out["n_pops"] = int(npop.value)
        return out

    def voxel_grid_tensor(self, lidar: int, pts5, leaf: float):
        """voxel_grid() of a contiguous float32 CUDA tensor (n, 5) {x, y, z, intensity, curvature}, read in place, or with None of
        the slot's undistorted cloud.  Returns float32 (n_out, 5), a view of a buffer allocated on the current stream; the result
        is enqueued, not waited for.  The filter returns at most one row per input row, so the buffer is allocated with the input's
        rows and sliced: the filter runs once, where the size-query protocol of voxel_grid() runs it twice.  For the slot's cloud
        the rows are those of this model's last undistort*() on the slot; if the slot holds more (it was filled through the
        C-ABI directly), a second call with the full size fetches the rest."""
        import torch
        if pts5 is not None:
            _check_tensor(pts5, "pts5", torch.float32, 5, self.device)
        rows = self._slot_rows.get(lidar, 0) if pts5 is None else pts5.shape[0]
        st = torch.cuda.current_stream(self.device)
        m = C.c_uint32(0)
        call = lambda out, cap: self._check(self.lib.malio_voxel_grid_device(
            self._h, lidar, _dptr(pts5), 0 if pts5 is None else pts5.shape[0], C.c_float(leaf), _dptr(out), cap, C.addressof(m), st.cuda_stream))
        out = self._empty((rows, 5), torch.float32)
        call(out, rows)
        if m.value > rows:
            out = self._empty((m.value, 5), torch.float32)
            call(out, m.value)
        return out[: m.value]

    def scan_uncertainty_resident(self, imu_cov: np.ndarray, extrinsic: np.ndarray, uncertainty: np.ndarray):
        """scan_uncertainty() with the table left on the device for upload_scan_resident().  Returns (table_off uint32[L+1],
        temporal_comp capi.POSE[L-1])."""
        L = self.n_lidar
        a, _keep = _scan_unc_args(imu_cov, extrinsic, uncertainty)
        off = np.zeros(L + 1, np.uint32)
        tc = np.zeros(max(L - 1, 1), dtype=capi.POSE)
        self._check(self.lib.malio_scan_uncertainty_resident(self._h, C.addressof(a), capi.ptr(off), capi.ptr(tc)))
        return off, tc[: L - 1]

    def upload_scan_resident(self) -> int:
        """upload_scan_device() with the table, offsets and temporal compensations of the last scan_uncertainty*()."""
        n = C.c_uint32(0)
        self._check(self.lib.malio_upload_scan_resident(self._h, C.addressof(n)))
        self.n_points = int(n.value)
        return self.n_points


STORED_SCAN = np.dtype([("time", "<f8"), ("rot", "<f8", 4), ("pos", "<f8", 3), ("ext", capi.RIGID, capi.MAX_LIDAR),
                        ("temporal_comp", capi.RIGID, capi.MAX_LIDAR - 1), ("slot_tag", "<f4", capi.MAX_LIDAR),
                        ("n_points", "<u4", capi.MAX_LIDAR)])   # malio_stored_scan as a numpy record
assert STORED_SCAN.itemsize == C.sizeof(capi.StoredScan)
SCAN_STORE_FORMAT = 1


def write_scan_store_npz(path: str, records: np.ndarray, xyz: np.ndarray):
    """A scan store as one .npz: records (STORED_SCAN, one per scan) and every scan's points concatenated in index order
    (float32 (sum of n_points, 3)).  ValueError when the counts do not add up."""
    records = np.ascontiguousarray(records, STORED_SCAN)
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    if int(records["n_points"].astype(np.int64).sum()) != xyz.shape[0]:
        raise ValueError(f"xyz: {xyz.shape[0]} points, the records count {int(records['n_points'].astype(np.int64).sum())}")
    with open(path, "wb") as f:
        np.savez(f, format=np.int64(SCAN_STORE_FORMAT), records=records, xyz=xyz)


def read_scan_store_npz(path: str) -> tuple:
    """(records, list of each scan's float32 (n, 3) points) of a file write_scan_store_npz wrote."""
    with np.load(path, allow_pickle=False) as z:
        if int(z["format"]) != SCAN_STORE_FORMAT:
            raise ValueError(f"{path}: scan store format {int(z['format'])}, expected {SCAN_STORE_FORMAT}")
        records = np.ascontiguousarray(z["records"], STORED_SCAN)
        xyz = np.ascontiguousarray(z["xyz"], np.float32).reshape(-1, 3)
    ends = np.cumsum(records["n_points"].astype(np.int64).sum(axis=1))
    if (ends[-1] if ends.shape[0] else 0) != xyz.shape[0]:
        raise ValueError(f"{path}: {xyz.shape[0]} points, the records count {int(ends[-1]) if ends.shape[0] else 0}")
    starts = np.concatenate([[0], ends[:-1]]).astype(np.int64)
    return records, [xyz[a:b] for a, b in zip(starts, ends)]


def save_scan_store(model: MeasurementModel, path: str):
    """Every scan model stores, records and points, into one .npz (write_scan_store_npz), so that a later process can correct
    the states and rebuild the map (load_scan_store, then MeasurementModel.voxel_map_rebuild)."""
    recs, pts = [], []
    for k in range(model.scan_store_info()["n_scans"]):
        rec, xyz = model.scan_store_get(k)
        recs.append(np.frombuffer(bytes(rec), STORED_SCAN)[0])
        pts.append(xyz)
    records = np.array(recs, STORED_SCAN) if recs else np.zeros(0, STORED_SCAN)
    write_scan_store_npz(path, records, np.concatenate(pts) if pts else np.zeros((0, 3), np.float32))


def load_scan_store(model: MeasurementModel, path: str) -> int:
    """Append the scans of a save_scan_store file to model's store.  Returns the number of stored scans."""
    records, pts = read_scan_store_npz(path)
    n = model.scan_store_info()["n_scans"]
    for r, xyz in zip(records, pts):
        n = model.scan_store_put(capi.StoredScan.from_buffer_copy(r.tobytes()), xyz)
    return n


def _undistort_args(beg_time, extrinsic, lt_imu_frame, ctrl_t, ctrl_T, imu_cov_t, cov_pointer):
    """capi.UndistortArgs over host arrays: (args, the imu_cov times, the arrays the struct points into: keep them alive)."""
    ct = np.ascontiguousarray(ctrl_t, np.float64)
    cT = np.ascontiguousarray(ctrl_T, np.float64).reshape(-1, 16)
    cv = np.ascontiguousarray(imu_cov_t, np.float64)
    a = capi.UndistortArgs()
    a.beg_time = float(beg_time)
    a.extrinsic.q[:] = list(map(float, extrinsic[0])); a.extrinsic.t[:] = list(map(float, extrinsic[1]))
    a.lt_imu_frame.q[:] = list(map(float, lt_imu_frame[0])); a.lt_imu_frame.t[:] = list(map(float, lt_imu_frame[1]))
    a.ctrl_t = ct.ctypes.data; a.ctrl_T = cT.ctypes.data; a.n_ctrl = ct.shape[0]
    a.imu_cov_t = cv.ctypes.data if cv.shape[0] else None; a.n_cov = cv.shape[0]; a.cov_pointer = int(cov_pointer)
    return a, cv, (ct, cT)


def _scan_unc_args(imu_cov, extrinsic, uncertainty):
    """capi.ScanUncArgs over host arrays: (args, the arrays the struct points into: keep them alive)."""
    cov = np.ascontiguousarray(imu_cov, np.float64).reshape(-1, 36)
    ext = np.ascontiguousarray(extrinsic, dtype=capi.POSE)
    unc0 = np.ascontiguousarray(uncertainty, np.float64).reshape(36)
    a = capi.ScanUncArgs()
    a.imu_cov = cov.ctypes.data if cov.shape[0] else None
    a.n_cov = cov.shape[0]
    a.extrinsic = ext.ctypes.data
    a.uncertainty = unc0.ctypes.data
    return a, (cov, ext, unc0)


def _rigid_of(tc):
    """capi.POSE[k] -> capi.RIGID[k] (what upload_scan* take as temporal_comp); None for k == 0."""
    if tc.shape[0] == 0:
        return None
    rigid = np.zeros(tc.shape[0], dtype=capi.RIGID)
    rigid["q"], rigid["t"] = tc["q"], tc["t"]
    return rigid


def pack_scan_tensor(xyz, lidar, table_idx):
    """malio_scan_pt records built with torch ops, on the inputs' device: int32 (n, 4), words 0..2 the bits of xyz (float32
    (n, 3)), word 3 = lidar | table_idx << 16 (integer tensors (n,)).  Raises ValueError for an id outside [0, 65535]; that
    check reads the ids' range back to the host (one synchronisation)."""
    import torch
    if not isinstance(xyz, torch.Tensor) or xyz.dtype != torch.float32 or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError(f"xyz: expected a float32 tensor (n, 3), got {getattr(xyz, 'dtype', type(xyz).__name__)} "
                         f"{tuple(getattr(xyz, 'shape', ()))}")
    n = xyz.shape[0]
    ids = []
    for name, t in (("lidar", lidar), ("table_idx", table_idx)):
        if not isinstance(t, torch.Tensor) or t.dim() != 1 or t.shape[0] != n:
            raise ValueError(f"{name}: expected a tensor ({n},)")
        if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
            raise ValueError(f"{name}: dtype {t.dtype}, expected an integer dtype")
        if t.device != xyz.device:
            raise ValueError(f"{name}: on {t.device}, xyz on {xyz.device}")
        ids.append(t.to(torch.int64))
    if n:
        lo_l, hi_l, lo_t, hi_t = torch.stack([ids[0].min(), ids[0].max(), ids[1].min(), ids[1].max()]).tolist()
        for name, lo, hi in (("lidar", lo_l, hi_l), ("table_idx", lo_t, hi_t)):
            if lo < 0 or hi > 0xFFFF:
                raise ValueError(f"{name}: values in [{lo}, {hi}], outside [0, 65535]")
    out = torch.empty((n, 4), dtype=torch.int32, device=xyz.device)
    out[:, :3] = xyz.contiguous().view(torch.int32)
    w = ids[0] | (ids[1] << 16)
    out[:, 3] = torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32)   # the uint32 word's bits
    return out


def _check_leaf(leaf) -> float:
    """A voxel leaf size in m: a finite number > 0 (ValueError otherwise), as a float32 value."""
    try:
        with np.errstate(over="ignore"):
            v = float(np.float32(leaf))
    except (TypeError, ValueError):
        raise ValueError(f"leaf: expected a number, got {type(leaf).__name__}") from None
    if not (np.isfinite(v) and v > 0.0):
        raise ValueError(f"leaf: {leaf!r}, expected a finite size > 0")
    return v


def _dptr(t):
    """Device address of a tensor for the C-ABI (None for None or an empty tensor: the calls take NULL with n == 0)."""
    return None if t is None or t.numel() == 0 else t.data_ptr()


def _check_tensor(t, name, dtype, cols, device, rows=None):
    """Raise ValueError unless t is a contiguous CUDA tensor of dtype on cuda:device with shape (rows, cols) — (rows,) when cols
    is None; rows None = any."""
    import torch
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name}: expected a torch.Tensor, got {type(t).__name__}")
    if t.dtype != dtype:
        raise ValueError(f"{name}: dtype {t.dtype}, expected {dtype}")
    shape_ok = (t.dim() == 1) if cols is None else (t.dim() == 2 and t.shape[1] == cols)
    if not shape_ok or (rows is not None and t.shape[0] != rows):
        want = f"({rows if rows is not None else 'n'},)" if cols is None else f"({rows if rows is not None else 'n'}, {cols})"
        raise ValueError(f"{name}: shape {tuple(t.shape)}, expected {want}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: not contiguous")
    if t.device.type != "cuda" or t.device.index != device:
        raise ValueError(f"{name}: on {t.device}, expected cuda:{device} (the handle's device)")
