"""publish_frame_world and the saved map without a GPU: the PCD file the library writes (malio_write_pcd_binary, the same code as
malio_world_save_pcd), the host restatement of RGBpointBodyToWorld the GPU tests hold the device to, and the save-interval
bookkeeping of plugin.PcdSaver (laserMapping.cpp:448-489, :1083-1091)."""
import os

import numpy as np
import pytest

import helpers as H
import world_ref as W
from malio_b200 import capi, plugin, synth


def _cloud(n, seed=0):
    rng = np.random.default_rng(seed)
    a = rng.normal(0, 50, (n, 4)).astype(np.float32)
    a[:, 3] = rng.integers(0, 3, n).astype(np.float32)
    if n > 3:
        a[0] = [-0.0, np.inf, -np.inf, np.nan]          # non-finite and signed-zero bit patterns go through untouched
        a[1, 0] = np.float32(1e-45)                     # a denormal
    return a


@pytest.mark.parametrize("n", [1, 100_000])
def test_pcd_binary_layout(tmp_path, n):
    pts = _cloud(n, seed=n)
    path = str(tmp_path / "cloud.pcd")
    plugin.write_pcd_binary(path, pts)
    data = open(path, "rb").read()
    hdr = W.pcd_header(n)
    assert data[: len(hdr)] == hdr
    assert len(data) == len(hdr) + 32 * n
    _, rec = W.read_pcd(path)
    assert W.xyzi(rec).tobytes() == pts.tobytes()       # bit for bit, NaN payloads and -0 included
    for f in ("normal_x", "normal_y", "normal_z", "curvature"):
        assert rec[f].view(np.uint32).max() == 0         # +0.0 exactly


def test_pcd_binary_refuses_without_leaving_a_file(tmp_path):
    lib = capi.load()
    pts = _cloud(10)
    p0 = tmp_path / "empty.pcd"
    assert lib.malio_write_pcd_binary(os.fsencode(str(p0)), capi.ptr(pts), 0) == capi.ERR_INVALID_ARG
    assert not p0.exists()
    assert lib.malio_write_pcd_binary(None, capi.ptr(pts), 10) == capi.ERR_INVALID_ARG
    p1 = tmp_path / "null.pcd"
    assert lib.malio_write_pcd_binary(os.fsencode(str(p1)), None, 10) == capi.ERR_INVALID_ARG
    assert not p1.exists()
    p2 = tmp_path / "no_such_dir" / "x.pcd"
    assert lib.malio_write_pcd_binary(os.fsencode(str(p2)), capi.ptr(pts), 10) == capi.ERR_INVALID_ARG
    assert not p2.exists() and not p2.parent.exists()
    assert sorted(os.listdir(tmp_path)) == []
    with pytest.raises(capi.MalioError):
        plugin.write_pcd_binary(str(p2), pts)


@pytest.mark.parametrize("L", [1, 2, 3])
def test_register_world_against_scipy(L):
    s, tc = W.far_state(L, seed=10 + L)
    rng = np.random.default_rng(L)
    n = 20000
    xyz = rng.uniform(-80, 80, (n, 3)).astype(np.float32)
    lid = rng.integers(0, L, n)
    ny = rng.uniform(0, 3, n).astype(np.float32)
    got = W.register_world(s, tc, xyz, lid, ny)
    ref = W.register_world_scipy(s, tc, xyz, lid)
    assert np.abs(ref).max() > 9e3
    assert H.ulp_diff(got[:, :3], ref.astype(np.float32)) <= 1.0
    assert got[:, 3].tobytes() == ny.tobytes()
    if L > 1:   # the temporal compensation is applied to LiDARs 1.. only
        plain = W.register_world_scipy(s, None, xyz[lid == 0], 0)
        assert H.ulp_diff(got[lid == 0, :3], plain.astype(np.float32)) <= 1.0


def test_register_world_equals_oracle_map_incremental():
    """pointBodyToWorld (:134-147) and RGBpointBodyToWorld (:149-163) share their xyz expression: the restatement is
    bit-equal to the oracle's map_incremental world output on every point that function does not skip."""
    case = synth.make_case("world-3L", 3000, 40000, 3, 3, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    orc = H.make_oracle(case, snap)
    x, P = case.x_prop.copy(), case.P_prop.copy()
    orc.update_iterated(x, P, case.max_iter)
    cls, w = orc.map_incremental(x, 0.5, True)
    ny = orc.aux()["normal_y"]
    got = W.register_world(x, case.temporal_comp, case.pts["xyz"], case.pts["lidar"], ny)
    keep = cls != capi.MAP_SKIP
    assert keep.sum() > 1000 and len(np.unique(case.pts["lidar"][keep])) == 3
    assert got[keep, :3].tobytes() == w[keep].tobytes()
    assert got[:, 3].tobytes() == ny.tobytes()


class _FakeModel:
    """Stands in for MeasurementModel: records pcd_accumulate / pcd_save as the library would see them."""

    def __init__(self, sizes):
        self.sizes, self.k, self.n, self.saved = list(sizes), 0, 0, []

    def pcd_accumulate(self, s, slot_tag):
        self.n += self.sizes[self.k]
        self.k += 1
        return self.n

    def pcd_save(self, path, clear):
        assert self.n > 0
        self.saved.append((os.path.basename(path), self.n))
        if clear:
            self.n = 0


@pytest.mark.parametrize("interval", [0, 1, 3])
def test_pcd_saver_interval(interval):
    """scan_wait_num > pcd_save_interval (:478): a file after every interval + 1 scans, numbered from 1; result.pcd at the end
    with what is left; never an empty cloud."""
    sizes = [5, 0, 7, 3, 0, 0, 0, 0, 2, 4]
    m = _FakeModel(sizes)
    saver = plugin.PcdSaver(m, "/nonexistent", interval)
    written = [saver.after_update(None, [0.0]) for _ in sizes]
    final = saver.finish()
    exp, wait, pending, k = [], 0, 0, 0
    for sz in sizes:
        pending += sz
        wait += 1
        if pending > 0 and interval > 0 and wait > interval:
            k += 1
            exp.append((f"scans_{k}.pcd", pending))
            pending, wait = 0, 0
    if pending:
        exp.append(("result.pcd", pending))
    assert m.saved == exp
    assert [os.path.basename(p) for p in written if p] == [e[0] for e in exp if e[0] != "result.pcd"]
    assert (final is not None) == (pending > 0)
    # scans 1-4; 5-8 add nothing, so the counter runs on until scan 9 brings points; scan 10 is left for result.pcd
    hand = {0: [("result.pcd", 21)], 3: [("scans_1.pcd", 15), ("scans_2.pcd", 2), ("result.pcd", 4)]}
    if interval in hand:
        assert m.saved == hand[interval]
