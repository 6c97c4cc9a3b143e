"""Test infrastructure for publish_frame_world and the saved map (laserMapping.cpp:448-489): a host restatement of
RGBpointBodyToWorld, an independent scipy version of the same transform, and a numpy reader of the binary PCD files."""
import numpy as np

from malio_b200 import capi, synth

PCD_HEADER = ("# .PCD v0.7 - Point Cloud Data file format\n"
              "VERSION 0.7\n"
              "FIELDS x y z intensity normal_x normal_y normal_z curvature\n"
              "SIZE 4 4 4 4 4 4 4 4\n"
              "TYPE F F F F F F F F\n"
              "COUNT 1 1 1 1 1 1 1 1\n"
              "WIDTH {n}\n"
              "HEIGHT 1\n"
              "VIEWPOINT 0 0 0 1 0 0 0\n"
              "POINTS {n}\n"
              "DATA binary\n")
PCD_FIELDS = ("x", "y", "z", "intensity", "normal_x", "normal_y", "normal_z", "curvature")
PCD_RECORD = np.dtype([(f, "<f4") for f in PCD_FIELDS])


def pcd_header(n: int) -> bytes:
    return PCD_HEADER.format(n=n).encode()


def read_pcd(path):
    """A binary PCD file of PointXYZINormal -> (header bytes, records as PCD_RECORD[n]).  Checks the header's shape."""
    data = open(path, "rb").read()
    end = data.index(b"DATA binary\n") + len(b"DATA binary\n")
    hdr = data[:end]
    n = int(hdr.split(b"POINTS ")[1].split(b"\n")[0])
    assert hdr == pcd_header(n), hdr
    assert len(data) == end + 32 * n, (len(data), end, n)
    return hdr, np.frombuffer(data[end:], PCD_RECORD).copy()


def xyzi(rec) -> np.ndarray:
    """PCD records -> float32[n,4] {x, y, z, intensity}."""
    return np.stack([rec[f] for f in PCD_FIELDS[:4]], axis=1)


def _qrot(q, v):
    """Eigen's QuaternionBase::_transformVector, v + w uv + qv x uv with uv = 2 qv x v, in its operation order (float64)."""
    w, x, y, z = (float(c) for c in q)
    v0, v1, v2 = v[:, 0], v[:, 1], v[:, 2]
    a0, a1, a2 = y * v2 - z * v1, z * v0 - x * v2, x * v1 - y * v0
    u0, u1, u2 = a0 + a0, a1 + a1, a2 + a2
    c0, c1, c2 = y * u2 - z * u1, z * u0 - x * u2, x * u1 - y * u0
    return np.stack([(v0 + w * u0) + c0, (v1 + w * u1) + c1, (v2 + w * u2) + c2], axis=1)


def _pass_parts(s):
    ps = s.pass_state() if isinstance(s, capi.State) else s
    rot, pos = np.array(ps.rot[:]), np.array(ps.pos[:])
    ext = [(np.array(ps.ext[l].q[:]), np.array(ps.ext[l].t[:])) for l in range(capi.MAX_LIDAR)]
    return rot, pos, ext


def register_world(s, temporal_comp, xyz, lid, normal_y):
    """RGBpointBodyToWorld (laserMapping.cpp:149-163) over a host cloud, restated in the reference's operation order:
    lid = int(intensity); p_w = rot (q_E[0] p + t_E[0]) + pos for lid 0, rot (q_C[lid-1] (q_E[lid] p + t_E[lid]) + t_C[lid-1]) + pos
    otherwise, in float64, stored as float32; intensity = normal_y.  s: capi.State / PassState (the updated state, extrinsics
    from it); temporal_comp: capi.RIGID[L-1] or None.  Returns float32[n,4]."""
    rot, pos, ext = _pass_parts(s)
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    n = xyz.shape[0]
    lid = np.broadcast_to(np.asarray(lid, np.int64), (n,))
    out = np.zeros((n, 4), np.float32)
    out[:, 3] = np.broadcast_to(np.asarray(normal_y, np.float32), (n,))
    for l in np.unique(lid):
        m = lid == l
        a = _qrot(ext[l][0], xyz[m].astype(np.float64)) + ext[l][1]
        if l != 0:
            a = _qrot(temporal_comp[l - 1]["q"], a) + temporal_comp[l - 1]["t"]
        out[m, :3] = (_qrot(rot, a) + pos).astype(np.float32)
    return out


def register_world_scipy(s, temporal_comp, xyz, lid):
    """The same transform, independently: scipy rotation matrices in float64, p_w = R (R_C (R_E p + t_E) + t_C) + pos."""
    from scipy.spatial.transform import Rotation
    R = lambda q: Rotation.from_quat(np.asarray(q, np.float64)[[1, 2, 3, 0]]).as_matrix()
    rot, pos, ext = _pass_parts(s)
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3).astype(np.float64)
    lid = np.broadcast_to(np.asarray(lid, np.int64), (xyz.shape[0],))
    out = np.zeros_like(xyz)
    for l in np.unique(lid):
        m = lid == l
        a = xyz[m] @ R(ext[l][0]).T + ext[l][1]
        if l != 0:
            a = a @ R(temporal_comp[l - 1]["q"]).T + temporal_comp[l - 1]["t"]
        out[m] = a @ R(rot).T + pos
    return out


def far_state(L, seed):
    """An updated state 1e4 m from the origin with non-identity extrinsics, and the scan's temporal compensation."""
    rng = np.random.default_rng(seed)
    extq = [synth.q_exp(synth.rand_unit(rng) * 0.4) for _ in range(L)]
    extt = [rng.normal(0, 0.5, 3) for _ in range(L)]
    s = synth.make_state([1.0e4, -0.7e4, 35.0], synth.q_exp(synth.rand_unit(rng) * 2.5), extq, extt)
    tc = np.zeros(max(L - 1, 0), capi.RIGID)
    for l in range(1, L):
        tc[l - 1]["q"] = synth.q_exp(synth.rand_unit(rng) * 0.05)
        tc[l - 1]["t"] = rng.normal(0, 0.3, 3)
    return s, (tc if L > 1 else None)
