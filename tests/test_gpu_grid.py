"""The 2-D occupancy grid on the device (malio_grid_build_device & co.), exactly against tests/grid_ref.py:
  - raster, ground and report byte-identical to the restatement at every argument edge of tests/test_grid_cpu.py and at
    several million points; the host entry equals the device entry;
  - the voxel map in place (with and without a keep rule) equals the points of the matching download; the prior equals its
    points followed by its session's; four quadrants stitched equal one region; the extent equals the restatement's;
  - every refusal leaves sentinel-filled outputs untouched; the call is ordered on the caller's stream; the handle's device
    bytes are the same after the call;
  - on the carved street: parked boxes occupied, the road and the car's lane free; without carving the lane is occupied."""
import ctypes as C

import numpy as np
import pytest
import torch

import grid_ref as G
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu
F = np.float32
Q_ID = np.array([1.0, 0.0, 0.0, 0.0])
EDGES = [   # res, i0, j0, nx, ny, w, h_lo, h_hi, m (tests/test_grid_cpu.py's, and wider ones)
    (0.1, -5, -4, 9, 7, 0, 0.3, 2.0, 1),
    (0.1, -5, -4, 9, 7, 1, 0.3, 2.0, 2),
    (0.25, 3, -2, 6, 5, 5, 0.3, 2.0, 1),
    (0.1, 2, 3, 1, 1, 1, 0.2, 0.2, 1),
    (0.1, 0, 0, 1, 6, 5, 0.5, 0.5, 1),
    (0.2, -1, 0, 7, 1, 0, 0.1, 1.0, 3),
    (0.05, -300, -200, 600, 400, 10, 0.3, 2.0, 2),
]


@pytest.fixture(scope="module")
def model():
    m = plugin.MeasurementModel(1)
    yield m
    m.close()


def _cloud(rng, n, res, i0, j0, nx, ny, w):
    lo = np.array([(i0 - w - 2) * res, (j0 - w - 2) * res])
    hi = np.array([(i0 + nx + w + 2) * res, (j0 + ny + w + 2) * res])
    xy = rng.uniform(lo, hi, (n, 2))
    k = n // 4
    xy[:k] = np.round(xy[:k] / res) * res
    xy[k] = [(i0 - w) * res, (j0 - w) * res]
    xy[k + 1] = [(i0 + nx + w) * res, (j0 + ny + w) * res]
    z = rng.choice(np.array([0.0, 0.1, 0.3, 0.5, 1.2, 2.0, 2.5], F), n) + F(0.01) * rng.integers(0, 3, n).astype(F)
    z[: n // 8] = rng.choice(np.array([-0.0, 0.0], F), n // 8)
    pts = np.concatenate([xy.astype(F), z[:, None].astype(F), rng.uniform(0, 1, (n, 1)).astype(F)], axis=1)
    pts[-1, 0], pts[-2, 1], pts[-3, 2] = np.nan, np.inf, -np.inf
    return pts


def _args(res, i0, j0, nx, ny, w, h_lo, h_hi, m):
    return plugin.grid_args(res, i0, j0, nx, ny, w, h_lo, h_hi, m)


def _same_as_ref(cls, ground, rep, pts, edge):
    rc, rg, rr = G.grid(pts, *edge)
    assert np.array_equal(cls.cpu().numpy() if hasattr(cls, "cpu") else cls, rc)
    g = ground.cpu().numpy() if hasattr(ground, "cpu") else ground
    assert g.tobytes() == rg.tobytes()
    for key in ("n_used", "n_nonfinite", "n_outside", "n_occupied", "n_free", "n_unknown", "device_bytes"):
        assert rep[key] == rr[key], key


@pytest.mark.parametrize("edge", EDGES)
def test_device_equals_the_restatement_at_every_edge(model, edge):
    rng = np.random.default_rng(edge[3] * 13 + edge[5])
    pts = _cloud(rng, 5000 if edge[3] < 100 else 400000, *edge[:6])
    x = torch.from_numpy(pts).cuda()
    cls, ground, rep = model.grid("points", x, args=_args(*edge))
    _same_as_ref(cls, ground, rep, pts, edge)
    hc, hg, hr = model.grid_host(pts, _args(*edge))
    assert np.array_equal(hc, cls.cpu().numpy()) and hg.tobytes() == ground.cpu().numpy().tobytes()
    assert {k: v for k, v in hr.items() if k != "device_bytes"} == {k: v for k, v in rep.items() if k not in ("device_bytes", "args")}


def test_millions_of_points_host_and_device(model):
    """6 M points over a 40 m x 30 m region at 0.05 m: the host entry stages them in two chunks."""
    rng = np.random.default_rng(11)
    edge = (0.05, -400, -300, 800, 600, 10, 0.3, 2.0, 2)
    pts = _cloud(rng, 6_000_000, *edge[:6])
    cls, ground, rep = model.grid("points", torch.from_numpy(pts).cuda(), args=_args(*edge))
    _same_as_ref(cls, ground, rep, pts, edge)
    hc, hg, _ = model.grid_host(pts, _args(*edge))
    assert np.array_equal(hc, cls.cpu().numpy()) and hg.tobytes() == ground.cpu().numpy().tobytes()


def test_quadrants_stitch_into_one_region(model):
    rng = np.random.default_rng(5)
    edge = (0.1, -100, -80, 200, 160, 7, 0.3, 2.0, 2)
    x = torch.from_numpy(_cloud(rng, 300000, *edge[:6])).cuda()
    whole, wg, _ = model.grid("points", x, args=_args(*edge))
    cls, gr = torch.empty_like(whole), torch.empty_like(wg)
    for i0, nx in ((-100, 90), (-10, 110)):
        for j0, ny in ((-80, 75), (-5, 85)):
            c, g, _ = model.grid("points", x, args=_args(0.1, i0, j0, nx, ny, 7, 0.3, 2.0, 2))
            cls[j0 + 80: j0 + 80 + ny, i0 + 100: i0 + 100 + nx] = c
            gr[j0 + 80: j0 + 80 + ny, i0 + 100: i0 + 100 + nx] = g
    assert torch.equal(cls, whole) and gr.cpu().numpy().tobytes() == wg.cpu().numpy().tobytes()


def test_extent_equals_the_restatement(model):
    rng = np.random.default_rng(2)
    pts = _cloud(rng, 20000, 0.1, -50, -30, 100, 60, 3)
    x = torch.from_numpy(pts).cuda()
    assert model.grid_extent("points", x, res=0.1) == G.extent(pts, 0.1)
    assert model.grid_extent("points", x, res=0.37) == G.extent(pts, 0.37)
    nan = torch.full((4, 4), float("nan"), device="cuda")
    assert model.grid_extent("points", nan) == (0, 0, -1, -1)
    far = torch.tensor([[2e6, 0.0, 0.0, 0.0]], device="cuda")
    with pytest.raises(capi.MalioError) as e:
        model.grid_extent("points", far, res=0.1)
    assert e.value.status == capi.ERR_CAPACITY
    # the whole extent as the default region
    cls, _, rep = model.grid("points", x)
    e4 = G.extent(pts, plugin.GRID_RES)
    assert tuple(cls.shape) == (e4[3] - e4[1] + 1, e4[2] - e4[0] + 1) and rep["args"].i0 == e4[0]


def _plant(m, xyz):
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    pts = np.zeros(xyz.shape[0], capi.RAW_PT)
    pts["xyz"] = xyz
    ctrl_t = np.array([-10.0, -9.0, -8.0, -7.0])
    m.undistort(0, pts, 0.0, (Q_ID, np.zeros(3)), (Q_ID, np.zeros(3)), ctrl_t, np.tile(np.eye(4), (4, 1, 1)), np.zeros(0), -1)


def _street_map(carve, leaf=0.1, n_scans=20):
    st = synth.Street()
    m = plugin.MeasurementModel(1)
    for k in range(n_scans):
        sc = synth.street_scan(st, k)
        _plant(m, sc["body"][0])
        m.voxel_map_accumulate(sc["state"], np.zeros(1, F), leaf, carve=True if carve else None)
    return st, m


def test_voxel_map_and_prior_sources_equal_their_downloads(model):
    st, m = _street_map(True, leaf=0.2, n_scans=12)
    try:
        a = plugin.grid_args(0.1, -150, -100, 700, 200)
        downs = {keep: m.voxel_map_tensor(keep) for keep in (None, True)}   # a download keeps its sort area until a save
        info0 = m.voxel_map_info()
        for keep in (None, True):
            down = downs[keep]
            c1, g1, r1 = m.grid("voxel_map", keep=keep, args=a)
            c2, g2, r2 = m.grid("points", down, args=a)
            assert torch.equal(c1, c2) and g1.cpu().numpy().tobytes() == g2.cpu().numpy().tobytes()
            assert {k: r1[k] for k in ("n_used", "n_outside", "n_nonfinite")} == {k: r2[k] for k in ("n_used", "n_outside", "n_nonfinite")}
            _same_as_ref(c1, g1, r1, down.cpu().numpy(), (0.1, -150, -100, 700, 200, a.ground_halfwidth, a.h_lo, a.h_hi, a.min_obstacle_points))
            assert m.grid_extent("voxel_map", keep=keep) == G.extent(down.cpu().numpy(), 0.1)
        assert m.voxel_map_info() == info0
        kept = downs[True].cpu().numpy()
        m.prior_map_load(kept[:, :3])
        p0 = m.prior_map_info()
        sess = m.prior_map_session()
        both = np.concatenate([np.concatenate([kept[:, :3], np.full((kept.shape[0], 1), 0.001, F)], 1), sess]).astype(F)
        c1, g1, r1 = m.grid("prior", args=a)
        c2, g2, _ = m.grid("points", torch.from_numpy(both).cuda(), args=a)
        assert torch.equal(c1, c2) and g1.cpu().numpy().tobytes() == g2.cpu().numpy().tobytes() and r1["n_used"] > 0
        assert m.prior_map_info() == p0 and m.voxel_map_info() == info0
    finally:
        m.close()


def test_states_refused(model):
    m = plugin.MeasurementModel(1)
    try:
        for src in ("voxel_map", "prior"):
            with pytest.raises(capi.MalioError) as e:
                m.grid(src, args=plugin.grid_args(nx=4, ny=4))
            assert e.value.status == capi.ERR_STATE
    finally:
        m.close()


def _raw(model, src, x, n, k, a, cls, ground, stream=None):
    return model.lib.malio_grid_build_device(model._h, src, None if x is None else x.data_ptr(), n, k, C.byref(a),
                                             None if cls is None else cls.data_ptr(), None if ground is None else ground.data_ptr(),
                                             stream, None)


def test_refusals_leave_the_outputs_untouched(model):
    rng = np.random.default_rng(9)
    x = torch.from_numpy(_cloud(rng, 1000, 0.1, 0, 0, 8, 8, 1)).cuda()
    good = dict(res=0.1, i0=0, j0=0, nx=8, ny=8, ground_halfwidth=1, h_lo=0.3, h_hi=2.0, min_obstacle_points=1)
    bads = [dict(res=0.0), dict(res=float("inf")), dict(nx=0), dict(ny=0), dict(h_lo=0.0), dict(h_lo=3.0), dict(h_hi=float("nan")),
            dict(min_obstacle_points=0), dict(i0=(1 << 24) - 8, ground_halfwidth=1), dict(j0=-(1 << 24), ground_halfwidth=1)]
    cls = torch.full((8, 8), 7, dtype=torch.uint8, device="cuda")
    ground = torch.full((8, 8), 3.5, device="cuda")
    for b in bads:
        a = plugin.grid_args(**{**good, **b})
        assert _raw(model, capi.GRID_POINTS, x, 1000, None, a, cls, ground) == capi.ERR_INVALID_ARG, b
    a = plugin.grid_args(**good)
    host = torch.zeros(64, dtype=torch.uint8).pin_memory()
    assert _raw(model, capi.GRID_POINTS, x, 1000, None, a, host, ground) == capi.ERR_INVALID_ARG
    assert _raw(model, capi.GRID_POINTS, x[:, 1:].contiguous()[1:], 999, None, a, cls, ground) == capi.ERR_INVALID_ARG   # misaligned
    assert _raw(model, 7, x, 1000, None, a, cls, ground) == capi.ERR_INVALID_ARG
    assert _raw(model, capi.GRID_VOXEL_MAP, None, 0, None, a, cls, ground) == capi.ERR_STATE
    big = plugin.grid_args(**{**good, "nx": 1 << 20, "ny": 1 << 20})
    assert _raw(model, capi.GRID_POINTS, x, 1000, None, big, cls, ground) == capi.ERR_CAPACITY
    assert "bytes" in model.lib.malio_last_error(model._h).decode()
    torch.cuda.synchronize()
    assert torch.all(cls == 7) and torch.all(ground == 3.5)


def test_ordered_on_the_callers_stream(model):
    """The points are written on a side stream after a long kernel; the grid reads them there and its outputs are read on the
    same stream without a host synchronisation in between."""
    rng = np.random.default_rng(4)
    edge = (0.1, -40, -40, 80, 80, 5, 0.3, 2.0, 2)
    pts = _cloud(rng, 200000, *edge[:6])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        big = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            big = big @ big / 64.0
        x = torch.from_numpy(pts).pin_memory().cuda(non_blocking=True)
        cls, ground, rep = model.grid("points", x, args=_args(*edge))
        out_c, out_g = cls.cpu(), ground.cpu()
    _same_as_ref(out_c, out_g, rep, pts, edge)


def test_device_bytes_unchanged(model):
    st, m = _street_map(False, leaf=0.2, n_scans=3)
    try:
        v0 = m.voxel_map_info()
        m.grid("voxel_map", args=plugin.grid_args(0.1, -100, -100, 500, 200))
        m.grid("voxel_map")
        assert m.voxel_map_info() == v0
    finally:
        m.close()


def test_street_parked_boxes_occupied_and_lanes_free(tmp_path):
    """The kept map of 20 carved scans at a 0.2 m leaf, gridded at 0.2 m with the other defaults: the parked boxes' footprints
    occupied, the observed road free, and the lane the car drove along free; without carving part of its trail is an obstacle.
    The device equals the restatement on the download, and the thresholds are the restatement's numbers on the same scene
    (DESIGN.md's table: 0.569 / 1.0 / 0.042, and 0.129 of the lane occupied without carving)."""
    fr = {}
    for carve in (True, False):
        st, m = _street_map(carve, leaf=0.2)
        try:
            keep = True if carve else None
            lo_i, lo_j, hi_i, hi_j = m.grid_extent("voxel_map", keep=keep, res=0.2)
            a = plugin.grid_args(0.2, lo_i, lo_j, hi_i - lo_i + 1, hi_j - lo_j + 1)
            cls, ground, rep = m.grid("voxel_map", keep=keep, args=a)
            down = m.voxel_map_tensor(keep).cpu().numpy()
            _same_as_ref(cls, ground, rep, down, (a.res, a.i0, a.j0, a.nx, a.ny, a.ground_halfwidth, a.h_lo, a.h_hi, a.min_obstacle_points))
            c = cls.cpu().numpy()
            fr[carve] = G.street_fractions(st, c, a.res, a.i0, a.j0, a.nx, a.ny)
            if carve:
                pgm, yaml = plugin.save_grid(str(tmp_path / "street"), cls, a)
                body = np.frombuffer(open(pgm, "rb").read()[len(f"P5\n{a.nx} {a.ny}\n255\n"):], np.uint8).reshape(a.ny, a.nx)
                y = dict(l.split(": ", 1) for l in open(yaml).read().splitlines())
                assert np.array_equal(G.decode(body, float(y["occupied_thresh"]), float(y["free_thresh"])), c)
        finally:
            m.close()
    print("street fractions", fr)
    assert fr[True]["parked"] >= 0.55 and fr[True]["road"] >= 0.99 and fr[True]["lane_occupied"] <= 0.05, fr
    assert fr[False]["lane_occupied"] >= 0.12, fr
