"""numpy restatement of malio_world_voxel_rebuild (include/malio_b200.h): the contract as a loop over the existing restatements.
Each stored scan k = first .. first + count - 1, in index order: its stored points registered with world_ref.register_world
under states[k - first] (or its stored state) and its stored temporal compensation, slot by slot with the stored slot tags,
then folded with VoxelMapRef.accumulate_fast, or with CarveMapRef.accumulate_carve and the slots' origins.

A stored scan here is a dict: state (capi.PassState), temporal_comp (capi.RIGID[MAX_LIDAR - 1]), slot_tag (float32[L]),
n_points (int[L]) and xyz (float32 (sum n_points, 3), slots in order)."""
import numpy as np

import world_ref as W
from malio_b200 import capi

F = np.float32


def scan_of(record, xyz, L):
    """The dict of a capi.StoredScan record and its points."""
    tc = np.frombuffer(bytes(record.temporal_comp), capi.RIGID).copy()
    return dict(state=record.state, temporal_comp=tc, slot_tag=np.array(record.slot_tag[:L], F),
                n_points=[int(v) for v in record.n_points[:L]], xyz=np.asarray(xyz, F).reshape(-1, 3))


def slots(scan):
    """Each slot's (l, float32 (m_l, 3)) points."""
    at = 0
    for l, m in enumerate(scan["n_points"]):
        yield l, scan["xyz"][at:at + m]
        at += m


def register(scan, state=None):
    """float32 (n, 4): the scan registered as malio_world_register(.., MALIO_WORLD_DENSE, ..) registers it."""
    s = scan["state"] if state is None else state
    parts = [W.register_world(s, scan["temporal_comp"], xyz, l, scan["slot_tag"][l]) for l, xyz in slots(scan)]
    return np.concatenate(parts).reshape(-1, 4) if parts else np.zeros((0, 4), F)


def origins(scan, state=None):
    """float32 (L, 3): each slot's origin, body_to_world of (0, 0, 0)."""
    s = scan["state"] if state is None else state
    return np.concatenate([W.register_world(s, scan["temporal_comp"], np.zeros((1, 3), F), l, 0.0)[:, :3]
                           for l in range(len(scan["n_points"]))])


def rebuild(ref, scans, leaf, states=None, carve=None):
    """The rebuild of `scans` into ref (world_voxel_ref.VoxelMapRef, or carve_ref.CarveMapRef with carve = dict(max_range,
    end_margin)).  Returns the voxel count."""
    n = len(ref.sums)
    for k, sc in enumerate(scans):
        s = None if states is None else states[k]
        cloud = register(sc, s)
        if carve is None:
            n = ref.accumulate_fast(cloud, leaf) if not hasattr(ref, "hit") else ref.accumulate(cloud, leaf)
        else:
            n = ref.accumulate_carve(cloud, sc["n_points"], origins(sc, s), leaf, **carve)
    return n
