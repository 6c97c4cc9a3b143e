"""The product's HOST code without a GPU.  malio_host.cpp (malio_ieskf_update = esekfom.hpp:495-721 with the one-factorisation
algebra, the degenerate branch, manifold operators) is linked against tests/hoststub/malio_dev_stub.cpp, a stand-in for the
CUDA translation unit whose measure() calls back into this test; the callback answers with the ORACLE's reduced system
for the state it is given.  The product's iterated update must then reproduce the oracle's own
update_iterated_dyn_share_modified: same passes, same searches, same state and covariance."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import helpers as H
from malio_b200 import capi, plugin, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUB_DIR = os.path.join(ROOT, "tests", "hoststub")


@pytest.fixture(scope="module")
def stub():
    lib = os.path.join(STUB_DIR, "libmalio_hoststub.so")
    srcs = [os.path.join(ROOT, "ma-lio_b200", "csrc", "malio_host.cpp"), os.path.join(STUB_DIR, "malio_dev_stub.cpp")]
    if not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs):
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-I" + os.path.join(ROOT, "include"),
                        "-I" + os.path.join(ROOT, "ma-lio_b200", "csrc"), *srcs, "-o", lib], check=True)
    L = C.CDLL(lib)
    L.malio_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p]
    L.malio_destroy.argtypes = [C.c_void_p]
    L.malio_ieskf_update.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_void_p]
    L.malio_last_error.restype = C.c_char_p
    L.malio_last_error.argtypes = [C.c_void_p]
    return L


MEASURE_FN = C.CFUNCTYPE(C.c_int, C.POINTER(capi.PassState), C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double),
                         C.POINTER(capi.PassStats))
ROWS_FN = C.CFUNCTYPE(C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_uint32, C.POINTER(C.c_uint32))


def _run(stub, case, snap, max_iter):
    orc_m = H.make_oracle(case, snap)          # answers the product's measure() calls
    orc_u = H.make_oracle(case, snap)          # runs the oracle's own update for comparison
    c = 6 * (case.n_lidar + 1)
    log = []

    def measure(ps, redo, pHTH, pHTh, pst):
        ok = orc_m.h_share_model(ps.contents, bool(redo), 2)
        st = orc_m.stats()
        log.append((bool(redo), ok, st.n_eff))
        C.memmove(pst, C.byref(st), C.sizeof(capi.PassStats))
        if not ok:
            return capi.ERR_NO_EFFECTIVE_POINTS
        HTH, HTh = orc_m.reduce()
        C.memmove(pHTH, HTH.ctypes.data, 8 * c * c)
        C.memmove(pHTh, HTh.ctypes.data, 8 * c)
        return capi.OK

    def rows(phx, ph, cap, pn):
        hx, h, _ = orc_m.dense()
        w = orc_m.stats().loc_weight
        n = min(hx.shape[0], cap)
        hx = np.ascontiguousarray(hx[:n] / w); h = np.ascontiguousarray(h[:n] / w)   # rows come without the localization weight
        C.memmove(phx, hx.ctypes.data, 8 * n * c)
        C.memmove(ph, h.ctypes.data, 8 * n)
        pn[0] = n
        return capi.OK

    mcb, rcb = MEASURE_FN(measure), ROWS_FN(rows)
    stub.malio_stub_set_callbacks(mcb, rcb)
    cfg = capi.Config()
    cfg.params = case.params
    cfg.params.n_lidar = case.n_lidar
    hnd = C.c_void_p()
    assert stub.malio_create(C.byref(hnd), C.byref(cfg)) == capi.OK
    xp, Pp = case.x_prop.copy(), case.P_prop.copy()
    rep = capi.UpdateReport()
    rc = stub.malio_ieskf_update(hnd, C.byref(xp), Pp.ctypes.data_as(C.c_void_p), max_iter, 0.001, C.byref(rep))
    stub.malio_destroy(hnd)
    xo, Po = case.x_prop.copy(), case.P_prop.copy()
    rco, dx_log, flags, rep_o = orc_u.update_iterated(xo, Po, max_iter, nthreads=2)
    return rc, rep, xp, Pp, rco, rep_o, xo, Po, log


@pytest.mark.parametrize("L,max_iter", [(3, 3), (1, 3), (2, 5)])
def test_product_host_ieskf_reproduces_the_oracle_update(stub, L, max_iter):
    case = synth.make_case(f"host{L}", 3000, 40000, L, max_iter, varied_map_cov=True)
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    rc, rep, xp, Pp, rco, rep_o, xo, Po, log = _run(stub, case, snap, max_iter)
    assert rc == capi.OK and rco == 0
    assert rep.passes == rep_o.passes and rep.searches == rep_o.searches and rep.converged_count == rep_o.converged_count
    assert [r for r, _, _ in log].count(True) == rep.searches and log[0][0] is True     # first pass always searches
    n = case.n_dof
    assert np.abs(synth.state_to_vec(xp, L) - synth.state_to_vec(xo, L)).max() < 1e-9
    assert np.abs(np.array(rep.dx_last[:n]) - np.array(rep_o.dx_last[:n])).max() < 1e-9
    assert H.rel_err(Pp, Po) < 1e-7
    assert np.allclose(Pp, Pp.T, rtol=1e-9, atol=1e-15)


@pytest.mark.parametrize("L,tables,mode", [(3, (2, 7, 40), "raw"), (3, (2, 7, 40), "edges"), (1, 5, "raw")])
@pytest.mark.parametrize("ext_en", [0, 1])
def test_product_host_ieskf_frozen_extrinsics_and_uneven_tables(stub, L, tables, mode, ext_en):
    """extrinsic_est_en = 0: the extrinsic columns of every reduced system are exactly zero, so the information block the
    host algebra inverts is rank-deficient there and only the prior holds those states; pose tables of different lengths
    per LiDAR with table indices at and beyond their ends."""
    case = synth.make_case(f"hf{L}", 3000, 40000, L, 3, varied_map_cov=True, table_T=tables, table_idx=mode)
    case.params.extrinsic_est_en = ext_en
    snap = plugin.build_static_snapshot(case.map_xyz, case.map_normal_y)
    orc = H.make_oracle(case, snap)
    assert orc.h_share_model(case.x_prop, True, 2)
    HTH, HTh = orc.reduce()
    ext = np.arange(6, 6 * (L + 1))
    st = orc.stats()
    if ext_en:
        assert np.abs(HTH[np.ix_(ext, ext)]).max() > 0 and st.tau_max > st.tau_min
    else:
        assert not HTH[ext].any() and not HTH[:, ext].any() and not HTh[ext].any()
        assert (st.tau_min, st.tau_max) == (9999.0, 0.0)
    rc, rep, xp, Pp, rco, rep_o, xo, Po, log = _run(stub, case, snap, 3)
    assert rc == capi.OK and rco == 0
    assert rep.passes == rep_o.passes and rep.searches == rep_o.searches and rep.converged_count == rep_o.converged_count
    n = case.n_dof
    assert np.abs(synth.state_to_vec(xp, L) - synth.state_to_vec(xo, L)).max() < 1e-9
    assert np.abs(np.array(rep.dx_last[:n]) - np.array(rep_o.dx_last[:n])).max() < 1e-9
    assert H.rel_err(Pp, Po) < 1e-7
    if not ext_en:   # nothing observes the extrinsics: they keep their prior value, their covariance its prior block
        e = slice(6, 6 + 6 * L)
        v0, v1 = synth.state_to_vec(case.x_prop, L), synth.state_to_vec(xp, L)
        assert np.abs(v1[7:7 + 7 * L] - v0[7:7 + 7 * L]).max() < 1e-12
        assert H.rel_err(Pp[e, e], case.P_prop[e, e]) < 1e-12


def test_product_host_degenerate_and_invalid_branches(stub):
    base = synth.make_case("hb", 3000, 40000, 3, 3, varied_map_cov=True)
    snap = plugin.build_static_snapshot(base.map_xyz, base.map_normal_y)
    # fewer effective points than state DOF: esekfom.hpp:574-582 through the rows callback
    tiny = synth.make_case("ht", 25, 40000, 3, 3, map_xyz=base.map_xyz)
    rc, rep, xp, Pp, rco, rep_o, xo, Po, log = _run(stub, tiny, snap, 3)
    assert rc == capi.OK and 1 <= rep.n_eff_last < 35 and rep.passes == rep_o.passes
    assert np.abs(synth.state_to_vec(xp, 3) - synth.state_to_vec(xo, 3)).max() < 1e-8
    assert H.rel_err(Pp, Po) < 1e-6
    # no effective points at all: every pass invalid, state and covariance untouched (esekfom.hpp:514-517)
    far = plugin.build_static_snapshot(base.map_xyz[:50] + np.float32(1e4))
    rc, rep, xp, Pp, rco, rep_o, xo, Po, log = _run(stub, base, far, 3)
    assert rc == capi.ERR_NO_EFFECTIVE_POINTS and rep.passes == 4 and all(not ok for _, ok, _ in log)
    assert np.array_equal(synth.state_to_vec(xp, 3), synth.state_to_vec(base.x_prop, 3)) and np.array_equal(Pp, base.P_prop)
