"""malio_relocalize without a GPU: the numpy restatement (tests/reloc_ref.py) against a plain loop over candidates and points,
the sliding-OR bound against every leaf under its node, the ctypes layout and signature against the header (compiled with gcc),
and NULL arguments answered with an error code (in a subprocess: a missing check would be a segmentation fault)."""
import ctypes as C
import itertools
import math
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import reloc_ref as RR
from malio_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _instance(seed, L=1, n=40, m=300, span=6.0):
    rng = np.random.default_rng(seed)
    extq = [synth.q_exp(synth.rand_unit(rng) * 0.3) for _ in range(L)]
    extt = [rng.normal(0, 0.3, 3) for _ in range(L)]
    s = synth.make_state(rng.normal(0, 2, 3), synth.q_exp(synth.rand_unit(rng) * 0.2), extq, extt)
    tc = None
    if L > 1:
        tc = np.zeros(L - 1, capi.RIGID)
        for l in range(1, L):
            tc[l - 1]["q"] = synth.q_exp(synth.rand_unit(rng) * 0.05)
            tc[l - 1]["t"] = rng.normal(0, 0.1, 3)
    pts = np.zeros(n, capi.SCAN_PT)
    pts["xyz"] = rng.uniform(-span, span, (n, 3)).astype(np.float32)
    pts["lidar"] = np.arange(n) % L
    prior = rng.uniform(-span - 3, span + 3, (m, 3)).astype(np.float32)
    return s, tc, pts, prior


def _loop_scores(s, tc, pts, prior, res, hxy, hz, n_yaw, yaw_lo, yaw_step):
    """Candidate by candidate, point by point, against a set of occupied voxels."""
    occ = {tuple(v) for v in RR.prior_voxels(prior, res).tolist()}
    best, arg = -1, None
    for k, q in enumerate(RR.candidate_rotations(s.rot[:], yaw_lo, yaw_step, n_yaw)):
        b, _ = RR.base_voxels(s, tc, pts, q, res)
        for c in range(-hz, hz + 1):
            for bb in range(-hxy, hxy + 1):
                for a in range(-hxy, hxy + 1):
                    sc = sum((x + a, y + bb, z + c) in occ for x, y, z in b.tolist())
                    if sc > best:
                        best, arg = sc, (k, (a, bb, c))
    return best, arg


@pytest.mark.parametrize("seed,L,hxy,hz,n_yaw,res", [(1, 1, 1, 0, 1, 1.0), (2, 2, 2, 1, 3, 0.7), (3, 3, 1, 1, 4, 1.3),
                                                     (4, 1, 3, 0, 2, 0.5)])
def test_reference_equals_a_plain_loop(seed, L, hxy, hz, n_yaw, res):
    s, tc, pts, prior = _instance(seed, L)
    r = RR.relocalize(s, tc, pts, prior, res, hxy, hz, n_yaw, 0.3, 2 * math.pi / n_yaw)
    best, (k, off) = _loop_scores(s, tc, pts, prior, res, hxy, hz, n_yaw, 0.3, 2 * math.pi / n_yaw)
    assert r["score"] == best and r["yaw_index"] == k and r["offset"] == off


def test_reference_tie_break_and_empty_prior():
    s, tc, pts, prior = _instance(5)
    r = RR.relocalize(s, tc, pts, np.zeros((0, 3), np.float32), 1.0, 2, 1, 3, 0.0, 1.0)
    assert r["score"] == 0 and r["yaw_index"] == 0 and r["offset"] == (-2, -2, -1)
    # one scan point, one prior voxel: every offset (a, b, c) that maps the point's voxel there scores 1 -> the smallest k, c, b, a
    pts1 = pts[:1]
    b, _ = RR.base_voxels(s, tc, pts1, RR.candidate_rotations(s.rot[:], 0.0, 0.0, 1)[0], 1.0)
    prior1 = (b[0].astype(np.float32) + np.float32(0.5))[None, :]
    r = RR.relocalize(s, tc, pts1, prior1, 1.0, 2, 1, 4, 0.0, 0.0)   # four equal yaws: all tie
    assert r["score"] == 1 and r["yaw_index"] == 0 and r["offset"] == (0, 0, 0)


def test_rotation_order_is_the_header_product():
    rot = synth.q_exp([0.1, -0.2, 0.3])
    for k, q in enumerate(RR.candidate_rotations(rot, -1.0, 0.25, 9)):
        th = -1.0 + k * 0.25
        want = synth.q_mul([math.cos(th / 2), 0, 0, math.sin(th / 2)], rot)
        assert np.allclose(q, want, rtol=0, atol=1e-15)


@pytest.mark.parametrize("seed", range(6))
def test_sliding_or_bound_dominates_every_leaf(seed):
    rng = np.random.default_rng(100 + seed)
    hxy, hz = int(rng.integers(0, 6)), int(rng.integers(0, 3))
    wxy, wz = 2 * hxy + 1, 2 * hz + 1
    n = int(rng.integers(5, 40))
    base = rng.integers(-8, 9, (n, 3))
    rel = base - base.min(axis=0)
    span = rel.max(axis=0)
    levels, dxy, dz = RR.pyramid(np.zeros((1, 1, 1), bool), hxy, hz)
    ext = span + np.array([wxy, wxy, wz]) + np.array([1 << dxy, 1 << dxy, 1 << dz])
    g0 = rng.random(tuple(ext)) < rng.uniform(0.05, 0.5)
    levels, dxy, dz = RR.pyramid(g0, hxy, hz)
    checked = 0
    for l, g in enumerate(levels):
        sx, sz = 1 << min(l, dxy), 1 << min(l, dz)
        for ux, uy, uz in itertools.product(range(0, wxy, sx), range(0, wxy, sx), range(0, wz, sz)):
            bound = RR.node_bound(g, rel, (ux, uy, uz))
            leaves = [RR.node_bound(g0, rel, (x, y, z)) for x in range(ux, min(ux + sx, wxy)) for y in range(uy, min(uy + sx, wxy))
                      for z in range(uz, min(uz + sz, wz))]
            assert bound >= max(leaves), (l, ux, uy, uz)
            if l == 0:
                assert bound == leaves[0]
            checked += 1
    assert checked >= 1
    # the top node's window covers the whole lattice: its bound dominates the best leaf
    assert RR.node_bound(levels[-1], rel, (0, 0, 0)) >= max(RR.node_bound(g0, rel, u) for u in
                                                           itertools.product(range(wxy), range(wxy), range(wz)))


def test_pyramid_level_is_the_or_over_its_window():
    rng = np.random.default_rng(7)
    g0 = rng.random((19, 17, 9)) < 0.1
    levels, dxy, dz = RR.pyramid(g0, 6, 2)
    for l, g in enumerate(levels):
        sx, sz = 1 << min(l, dxy), 1 << min(l, dz)
        for x, y, z in [(0, 0, 0), (3, 5, 1), (18, 16, 8), (10, 2, 4)]:
            assert g[x, y, z] == g0[x:x + sx, y:y + sx, z:z + sz].any()


# ------------------------------------------------------------------ the C-ABI
def _gcc_layout():
    src = textwrap.dedent("""
        #include <stddef.h>
        #include <stdio.h>
        #include "malio_b200.h"
        #define F(T, f) printf(#T "." #f " %zu\\n", offsetof(T, f))
        int main(void) {
          printf("args %zu\\nreport %zu\\n", sizeof(malio_reloc_args), sizeof(malio_reloc_report));
          F(malio_reloc_args, yaw_lo); F(malio_reloc_args, yaw_step); F(malio_reloc_args, n_yaw); F(malio_reloc_args, res);
          F(malio_reloc_args, half_xy); F(malio_reloc_args, half_z);
          F(malio_reloc_report, rot); F(malio_reloc_report, pos); F(malio_reloc_report, yaw_index); F(malio_reloc_report, offset);
          F(malio_reloc_report, score); F(malio_reloc_report, n_points); F(malio_reloc_report, n_candidates);
          F(malio_reloc_report, nodes_bounded); F(malio_reloc_report, leaves_scored); F(malio_reloc_report, device_bytes);
          return 0;
        }""")
    return src


def test_struct_layout_matches_the_header(tmp_path):
    c = tmp_path / "layout.c"
    c.write_text(_gcc_layout())
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.rsplit(" ", 1) for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["args"]) == C.sizeof(capi.RelocArgs)
    assert int(out["report"]) == C.sizeof(capi.RelocReport)
    for T, name in (("malio_reloc_args", capi.RelocArgs), ("malio_reloc_report", capi.RelocReport)):
        for f, _ in name._fields_:
            assert int(out[f"{T}.{f}"]) == getattr(name, f).offset, (T, f)


def test_signature_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    m = re.search(r"\bint\s+malio_relocalize\s*\(([^)]*)\)\s*;", hdr)
    assert m
    args = [a.strip() for a in m.group(1).split(",")]
    assert args == ["malio_handle* h", "const malio_pass_state* s", "const malio_reloc_args* a", "malio_reloc_report* rep"]
    fn = capi.load().malio_relocalize
    assert fn.argtypes == [C.c_void_p] * 4 and fn.restype is C.c_int
    assert "malio_relocalize" in capi.EXPORTS


def test_null_handle_and_null_arguments_return_an_error():
    code = textwrap.dedent("""
        import ctypes as C
        from malio_b200 import capi
        lib = capi.load()
        s, a, r = capi.PassState(), capi.RelocArgs(), capi.RelocReport()
        a.n_yaw, a.res = 1, 1.0
        print("all-null", lib.malio_relocalize(None, None, None, None), flush=True)
        print("no-handle", lib.malio_relocalize(None, C.byref(s), C.byref(a), C.byref(r)), flush=True)
        print("DONE")
    """)
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "ma-lio_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "DONE" and len(lines) == 3
    for l in lines[:-1]:
        assert l.split()[-1] == str(capi.ERR_INVALID_ARG), l
