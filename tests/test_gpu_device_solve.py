"""The iterated update with the IESKF step taken ON THE DEVICE (malio_solve.cu: one enqueued kernel sequence per scan, no host
round trip per pass) against the host loop (malio_host.cpp, MALIO_DEVICE_SOLVE=0) and the CPU oracle: same passes and
searches, same N_eff, state and covariance to FP64 rounding, for L = 1..3, max_iteration 1..5, a scan whose first pass is
invalid, and the degenerate n > N_eff branch (which the device path hands back to the host loop)."""
import numpy as np
import pytest

import helpers as H
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu


def _pair(case, snap, monkeypatch):
    monkeypatch.setenv("MALIO_DEVICE_SOLVE", "1")     # opt-in experiment, see DESIGN.md
    dev = H.make_model(case, snap)
    monkeypatch.setenv("MALIO_DEVICE_SOLVE", "0")
    host = H.make_model(case, snap)
    monkeypatch.delenv("MALIO_DEVICE_SOLVE")
    return dev, host


@pytest.mark.parametrize("L,max_iter", [(1, 3), (2, 3), (3, 3), (3, 5), (3, 1), (3, 2)])
def test_device_side_update_equals_host_loop_and_oracle(L, max_iter, monkeypatch):
    case = synth.make_case(f"ds-{L}", 20000, 200000, L, max_iter, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    dev, host = _pair(case, snap, monkeypatch)
    orc = H.make_oracle(case, snap)
    xd, Pd = case.x_prop.copy(), case.P_prop.copy()
    xh, Ph = case.x_prop.copy(), case.P_prop.copy()
    xo, Po = case.x_prop.copy(), case.P_prop.copy()
    c0 = dev.counters()
    rd = dev.update_iterated_dyn_share_modified(xd, Pd, max_iter)
    c1 = dev.counters()
    rh = host.update_iterated_dyn_share_modified(xh, Ph, max_iter)
    rc, _, _, ro = orc.update_iterated(xo, Po, max_iter, nthreads=4)
    assert rd.ms_host_solve == 0.0 and rh.ms_host_solve > 0.0          # the two paths really are different
    assert rd.passes == rh.passes == ro.passes and rd.searches == rh.searches == ro.searches
    assert rd.n_eff_last == rh.n_eff_last == ro.n_eff_last and rd.converged_count == rh.converged_count
    vd, vh, vo = (synth.state_to_vec(s, L) for s in (xd, xh, xo))
    assert np.abs(vd - vh).max() < 1e-9 and np.abs(vd - vo).max() < 1e-8   # summation orders differ (warp-level solves)
    assert H.rel_err(Pd, Ph) < 1e-8 and H.rel_err(Pd, Po) < 1e-6
    n = case.n_dof
    np.testing.assert_allclose(np.array(rd.dx_last[:n]), np.array(rh.dx_last[:n]), atol=1e-9)
    ad, ah = dev.aux(), host.aux()
    for k in ("selected", "nn_idx", "world", "normal_y"):
        assert np.array_equal(ad[k], ah[k]), k
    # a second scan on the same handle (sequence numbers / parities carried over), then a single legacy pass after it
    dev.rearm_scan(); host.rearm_scan()
    xd2, Pd2 = case.x_prop.copy(), case.P_prop.copy()
    xh2, Ph2 = case.x_prop.copy(), case.P_prop.copy()
    dev.update_iterated_dyn_share_modified(xd2, Pd2, max_iter); host.update_iterated_dyn_share_modified(xh2, Ph2, max_iter)
    assert np.array_equal(synth.state_to_vec(xd2, L), vd) and np.abs(synth.state_to_vec(xh2, L) - vd).max() < 1e-9
    ok1, H1, h1, s1 = dev.h_share_model(case.x_true, True)
    ok2, H2, h2, s2 = host.h_share_model(case.x_true, True)
    assert ok1 and ok2 and np.array_equal(H1, H2) and s1.n_eff == s2.n_eff
    dev.close(); host.close(); orc.close()


def test_degenerate_and_invalid_scans_through_the_device_path(monkeypatch):
    case = synth.make_case("ds-deg", 4000, 40000, 3, 3)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    dev, host = _pair(case, snap, monkeypatch)
    # (a) fewer effective points than state dimensions: the device path hands the scan back to the host loop
    few = np.ascontiguousarray(case.pts[::160][:22])
    for m in (dev, host):
        m.upload_scan(few, case.table, case.table_off, case.temporal_comp)
    xd, Pd = case.x_prop.copy(), case.P_prop.copy()
    xh, Ph = case.x_prop.copy(), case.P_prop.copy()
    rd = dev.update_iterated_dyn_share_modified(xd, Pd, 3)
    rh = host.update_iterated_dyn_share_modified(xh, Ph, 3)
    assert 0 < rd.n_eff_last < 35 and rd.passes == rh.passes
    assert np.array_equal(synth.state_to_vec(xd, 3), synth.state_to_vec(xh, 3)) and np.array_equal(Pd, Ph)
    # (b) a scan far away from the map: every pass invalid, state untouched, covariance = the propagated one
    far = case.pts.copy()
    far["xyz"] += np.float32(5000.0)
    for m in (dev, host):
        m.upload_scan(far, case.table, case.table_off, case.temporal_comp)
    xd, Pd = case.x_prop.copy(), case.P_prop.copy()
    xh, Ph = case.x_prop.copy(), case.P_prop.copy()
    rd = dev.update_iterated_dyn_share_modified(xd, Pd, 3)
    rh = host.update_iterated_dyn_share_modified(xh, Ph, 3)
    assert rd.passes == rh.passes == 4 and rd.last_status == rh.last_status == capi.ERR_NO_EFFECTIVE_POINTS
    assert np.array_equal(synth.state_to_vec(xd, 3), synth.state_to_vec(case.x_prop, 3)) and np.array_equal(Pd, Ph)
    dev.close(); host.close()


@pytest.mark.parametrize("env", [{"MALIO_PIPELINE": "1"}, {"MALIO_KNN_DIRECT": "1"}, {"MALIO_PIPELINE": "1", "MALIO_KNN_DIRECT": "1"}])
def test_optional_execution_variants_give_the_default_result(env, monkeypatch):
    """Opt-in variants of HOW the same update is executed — the pipelined host loop (next pass enqueued ahead, waiting on the
    device for the host's decision; only active with per-pass timing off) and the direct-load 3x3x3 k-NN scan — must give
    the default path's result: neighbour lists and gates identical, state bit-identical."""
    case = synth.make_case("variants", 30000, 300000, 3, 3, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    ref = H.make_model(case, snap)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    var = H.make_model(case, snap)
    for k in env:
        monkeypatch.delenv(k)
    ref.set_timing(False); var.set_timing(False)
    for rnd in range(3):
        xr, Pr = case.x_prop.copy(), case.P_prop.copy()
        xv, Pv = case.x_prop.copy(), case.P_prop.copy()
        ref.rearm_scan(); var.rearm_scan()
        rr = ref.update_iterated_dyn_share_modified(xr, Pr, 3)
        rv = var.update_iterated_dyn_share_modified(xv, Pv, 3)
        assert rr.passes == rv.passes and rr.searches == rv.searches and rr.n_eff_last == rv.n_eff_last
        assert np.array_equal(synth.state_to_vec(xr, 3), synth.state_to_vec(xv, 3)) and np.array_equal(Pr, Pv)
        ar, av = ref.aux(), var.aux()
        for k in ("selected", "nn_idx", "nn_sqdist", "world", "normal_y"):
            assert np.array_equal(ar[k], av[k]), k
    # a 1-iteration update (the pipelined loop cancels nothing / one pass) and a direct single pass afterwards
    xr, Pr = case.x_prop.copy(), case.P_prop.copy(); xv, Pv = case.x_prop.copy(), case.P_prop.copy()
    ref.rearm_scan(); var.rearm_scan()
    ref.update_iterated_dyn_share_modified(xr, Pr, 1); var.update_iterated_dyn_share_modified(xv, Pv, 1)
    assert np.array_equal(synth.state_to_vec(xr, 3), synth.state_to_vec(xv, 3))
    ok1, H1, h1, s1 = ref.h_share_model(case.x_true, True); ok2, H2, h2, s2 = var.h_share_model(case.x_true, True)
    assert ok1 and ok2 and np.array_equal(H1, H2)
    ref.close(); var.close()
