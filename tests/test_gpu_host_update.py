"""The iterated update (malio_host.cpp: the IESKF step on the host, one pass kernel per iteration) against the CPU oracle:
same passes and searches, same N_eff, state and covariance to FP64 rounding, for L = 1..3, max_iteration 1..5, a scan on
the same handle after it, the degenerate n > N_eff branch, and a scan whose every pass is invalid.  The environment
switches of the execution experiments that were removed from the library must leave the result untouched."""
import numpy as np
import pytest

import helpers as H
from malio_b200 import capi, plugin, synth

pytestmark = pytest.mark.gpu

RETIRED_SWITCHES = {"MALIO_DEVICE_SOLVE": "1", "MALIO_PIPELINE": "1", "MALIO_KNN_DIRECT": "0", "MALIO_KNN_KEYS": "0",
                    "MALIO_TAU_INLINE": "1", "MALIO_COOP_LAUNCH": "0"}


@pytest.mark.parametrize("L,max_iter", [(1, 3), (2, 3), (3, 3), (3, 5), (3, 1), (3, 2)])
def test_host_update_against_oracle(L, max_iter):
    case = synth.make_case(f"ds-{L}", 20000, 200000, L, max_iter, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    model = H.make_model(case, snap)
    orc = H.make_oracle(case, snap)
    xh, Ph = case.x_prop.copy(), case.P_prop.copy()
    xo, Po = case.x_prop.copy(), case.P_prop.copy()
    rh = model.update_iterated_dyn_share_modified(xh, Ph, max_iter)
    rc, _, _, ro = orc.update_iterated(xo, Po, max_iter, nthreads=4)
    assert rc == 0 and rh.last_status == 0 and rh.ms_host_solve > 0.0
    assert rh.passes == ro.passes and rh.searches == ro.searches
    assert rh.n_eff_last == ro.n_eff_last and rh.converged_count == ro.converged_count
    vh = synth.state_to_vec(xh, L)
    assert np.abs(vh - synth.state_to_vec(xo, L)).max() < 1e-8
    assert H.rel_err(Ph, Po) < 1e-6
    # a second scan on the same handle (sequence numbers / parities carried over), then a single pass after it
    model.rearm_scan()
    xh2, Ph2 = case.x_prop.copy(), case.P_prop.copy()
    model.update_iterated_dyn_share_modified(xh2, Ph2, max_iter)
    assert np.array_equal(synth.state_to_vec(xh2, L), vh) and np.array_equal(Ph2, Ph)
    ok_g, HTH, HTh, st = model.h_share_model(case.x_true, True)
    ok_o = orc.h_share_model(case.x_true, True, nthreads=4)
    assert ok_g and ok_o and st.n_eff == orc.stats().n_eff
    assert np.array_equal(model.aux()["selected"], orc.aux()["selected"])
    HTH_o, HTh_o = orc.reduce()
    assert H.rel_err(HTH, HTH_o) < 1e-9 and H.rel_err(HTh, HTh_o) < 1e-9
    model.close(); orc.close()


def test_degenerate_and_invalid_scans():
    case = synth.make_case("ds-deg", 4000, 40000, 3, 3)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    model = H.make_model(case, snap)
    orc = H.make_oracle(case, snap)
    # (a) fewer effective points than state dimensions: the degenerate branch with the dense rows
    few = np.ascontiguousarray(case.pts[::160][:22])
    model.upload_scan(few, case.table, case.table_off, case.temporal_comp)
    orc.set_scan(few, case.table, case.table_off, case.temporal_comp)
    xh, Ph = case.x_prop.copy(), case.P_prop.copy()
    xo, Po = case.x_prop.copy(), case.P_prop.copy()
    rh = model.update_iterated_dyn_share_modified(xh, Ph, 3)
    _, _, _, ro = orc.update_iterated(xo, Po, 3, nthreads=4)
    assert 0 < rh.n_eff_last < 35 and rh.passes == ro.passes
    # (b) a scan far away from the map: every pass invalid, state untouched, covariance = the propagated one
    far = case.pts.copy()
    far["xyz"] += np.float32(5000.0)
    model.upload_scan(far, case.table, case.table_off, case.temporal_comp)
    orc.set_scan(far, case.table, case.table_off, case.temporal_comp)
    xh, Ph = case.x_prop.copy(), case.P_prop.copy()
    xo, Po = case.x_prop.copy(), case.P_prop.copy()
    rh = model.update_iterated_dyn_share_modified(xh, Ph, 3)
    orc.update_iterated(xo, Po, 3, nthreads=4)
    assert rh.passes == 4 and rh.last_status == capi.ERR_NO_EFFECTIVE_POINTS
    assert np.array_equal(synth.state_to_vec(xh, 3), synth.state_to_vec(case.x_prop, 3)) and np.array_equal(Ph, Po)
    model.close(); orc.close()


def test_retired_switches_are_inert(monkeypatch):
    """The switches of the removed execution experiments (device-side IESKF step, pipelined host loop, staged k-NN scan,
    forced scan kernel, inline covariance traces, plain pass launch) are no longer read: a handle created with all of
    them set runs the host loop and gives the default handle's neighbour lists, gates, state and covariance bit for bit."""
    case = synth.make_case("variants", 30000, 300000, 3, 3, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    ref = H.make_model(case, snap)
    for k, v in RETIRED_SWITCHES.items():
        monkeypatch.setenv(k, v)
    var = H.make_model(case, snap)
    for k in RETIRED_SWITCHES:
        monkeypatch.delenv(k)
    ref.set_timing(False); var.set_timing(False)
    for rnd in range(3):
        xr, Pr = case.x_prop.copy(), case.P_prop.copy()
        xv, Pv = case.x_prop.copy(), case.P_prop.copy()
        ref.rearm_scan(); var.rearm_scan()
        rr = ref.update_iterated_dyn_share_modified(xr, Pr, 3)
        rv = var.update_iterated_dyn_share_modified(xv, Pv, 3)
        assert rv.ms_host_solve > 0.0
        assert rr.passes == rv.passes and rr.searches == rv.searches and rr.n_eff_last == rv.n_eff_last
        assert np.array_equal(synth.state_to_vec(xr, 3), synth.state_to_vec(xv, 3)) and np.array_equal(Pr, Pv)
        ar, av = ref.aux(), var.aux()
        for k in ("selected", "nn_idx", "nn_sqdist", "world", "normal_y"):
            assert np.array_equal(ar[k], av[k]), k
    # a 1-iteration update and a single pass afterwards
    xr, Pr = case.x_prop.copy(), case.P_prop.copy(); xv, Pv = case.x_prop.copy(), case.P_prop.copy()
    ref.rearm_scan(); var.rearm_scan()
    ref.update_iterated_dyn_share_modified(xr, Pr, 1)
    rv = var.update_iterated_dyn_share_modified(xv, Pv, 1)
    assert rv.ms_host_solve > 0.0
    assert np.array_equal(synth.state_to_vec(xr, 3), synth.state_to_vec(xv, 3)) and np.array_equal(Pr, Pv)
    ok1, H1, h1, s1 = ref.h_share_model(case.x_true, True); ok2, H2, h2, s2 = var.h_share_model(case.x_true, True)
    assert ok1 and ok2 and np.array_equal(H1, H2) and np.array_equal(h1, h2)
    ar, av = ref.aux(), var.aux()
    for k in ("selected", "nn_idx", "nn_sqdist", "world", "normal_y"):
        assert np.array_equal(ar[k], av[k]), k
    ref.close(); var.close()
