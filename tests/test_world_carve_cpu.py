"""Clearing moving objects out of the voxel map without a GPU: the DDA of tests/carve_ref.py against an exact segment / box
intersection (fractions), planted mistakes the counters must catch, the keep rule at its boundaries, the C-ABI against the
header (gcc), NULL arguments, and the defaults on the street scene of synth.street_scan."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap
from fractions import Fraction

import numpy as np
import pytest

import carve_ref as CR
import world_ref as W
import world_voxel_ref as V
from malio_b200 import capi, plugin, synth

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
F = np.float32


# ------------------------------------------------------------------ the DDA
def _rays(kind, rng, n=60):
    if kind == "random":
        o = rng.uniform(-3, 3, (n, 3))
        w = o + rng.normal(0, 2.5, (n, 3))
    elif kind == "axis":
        o = rng.uniform(-3, 3, (n, 3))
        w = o.copy()
        ax = rng.integers(0, 3, n)
        w[np.arange(n), ax] += rng.uniform(-6, 6, n)
        w[: n // 2, (ax[: n // 2] + 1) % 3] += rng.uniform(-3, 3, n // 2)   # two axes moving, one fixed
    elif kind == "corner":   # through cell corners of a 0.5 m grid: exact face ties
        c0 = rng.integers(-6, 6, (n, 3)).astype(np.float64) * 0.5 + 0.25
        d = rng.integers(-3, 4, (n, 3)).astype(np.float64) * 0.5
        d[:, 1] = d[:, 0] * rng.choice([-1, 1], n)
        o, w = c0, c0 + d
    elif kind == "zero":
        o = rng.uniform(-3, 3, (n, 3))
        w = o.copy()
    elif kind == "far":
        base = rng.choice([-1e5, 1e5], (n, 3))
        o = base + rng.uniform(-3, 3, (n, 3))
        w = o + rng.normal(0, 2.0, (n, 3))
    else:   # negzero: coordinates at -0.0 and +0.0
        o = rng.uniform(-1, 1, (n, 3))
        w = rng.uniform(-1, 1, (n, 3))
        o[::2, 0] = -0.0
        w[1::2, 1] = -0.0
        w[::3, 2] = 0.0
    return o.astype(F), w.astype(F)


def _clip(a, b, cell, open_):
    """Parameter interval of segment a -> b (fractions) inside the box [cell, cell + 1]^3; open_: its interior."""
    lo, hi = Fraction(0), Fraction(1)
    for ax in range(3):
        d = b[ax] - a[ax]
        c = cell[ax]
        if d == 0:
            inside = (c < a[ax] < c + 1) if open_ else (c <= a[ax] <= c + 1)
            if not inside:
                return None
            continue
        t1, t2 = (c - a[ax]) / d, (c + 1 - a[ax]) / d
        lo, hi = max(lo, min(t1, t2)), min(hi, max(t1, t2))
    return (lo, hi) if (lo < hi if open_ else lo <= hi) else None


@pytest.mark.parametrize("kind", ["random", "axis", "corner", "zero", "far", "negzero"])
@pytest.mark.parametrize("leaf", [0.5, 0.2])
def test_walk_against_exact_segment_box_intersection(kind, leaf):
    rng = np.random.default_rng([ord(ch) for ch in kind] + [int(leaf * 10)])
    o, w = _rays(kind, rng)
    u, e = CR.scaled(o, leaf), CR.scaled(w, leaf)
    ray, cell, t, last = CR.walk(o, w, leaf)
    pr, pc = CR.passed(o, w, leaf, 1e9, 0.0)
    for r in range(o.shape[0]):
        m = ray == r
        cs, ts, ls = cell[m], t[m], last[m]
        start, end = np.floor(u[r]).astype(np.int64), np.floor(e[r]).astype(np.int64)
        assert np.array_equal(cs[0], start) and np.array_equal(cs[-1], end)
        assert cs.shape[0] == 1 + np.abs(end - start).sum()
        assert ls[-1] and not ls[:-1].any()
        step = np.abs(np.diff(cs, axis=0))
        assert np.all(step.sum(axis=1) == 1)                                  # 6-connected
        assert np.all(np.diff(ts) >= 0)                                       # entry parameters never decrease
        a = [Fraction(float(x)) for x in u[r]]
        b = [Fraction(float(x)) for x in e[r]]
        visited = {tuple(c) for c in cs.tolist()}
        for c in pc[pr == r].tolist():                                        # every passed cell meets the segment
            assert _clip(a, b, c, False) is not None, (r, c)
        lo, hi = np.minimum(start, end), np.maximum(start, end)
        if np.prod(hi - lo + 1) <= 4000:
            for c in np.stack(np.meshgrid(*[np.arange(lo[i], hi[i] + 1) for i in range(3)], indexing="ij"), -1).reshape(-1, 3).tolist():
                if _clip(a, b, c, True) is not None:                          # crossed through its interior: visited
                    assert tuple(c) in visited, (r, c)
        if kind == "zero":
            assert cs.shape[0] == 1 and not (pr == r).any()


def test_passed_stops_at_range_and_margin():
    o = np.zeros((1, 3), F)
    w = np.array([[8.0, 0.0, 0.0]], F)
    _, c = CR.passed(o, w, 1.0, 3.0, 0.0)
    assert c[:, 0].tolist() == [0, 1, 2]                                      # entered at 0, 1, 2 m; 3 m is not below 3
    _, c = CR.passed(o, w, 1.0, 3.0, 0.0, variant="le")
    assert c[:, 0].tolist() == [0, 1, 2, 3]
    _, c = CR.passed(o, w, 1.0, 100.0, 2.5)
    assert c[:, 0].tolist() == [0, 1, 2, 3, 4, 5]                             # len - end_margin = 5.5
    _, c = CR.passed(o, w, 1.0, 100.0, 8.0)
    assert c.shape[0] == 0


# ------------------------------------------------------------------ planted mistakes change the counters
def _seed(ref, cells_xyz, leaf):
    """Voxels in the map before the carve (as a plain accumulate of their centres would leave them)."""
    for c in np.unique(np.asarray(cells_xyz, np.int64).reshape(-1, 3), axis=0).tolist():
        k = (c[2], c[1], c[0])
        ref.sums.setdefault(k, np.zeros(4, F))
        ref.cnt.setdefault(k, 1)
        ref.hit.setdefault(k, 0)
        ref.miss.setdefault(k, 0)
    ref.leaf = F(leaf)


def _evidence(o, w, leaf, seed_cells, variant, max_range=100.0, end_margin=0.0):
    ref = CR.CarveMapRef()
    _seed(ref, seed_cells, leaf)
    cloud = np.concatenate([w, np.zeros((w.shape[0], 1), F)], axis=1)
    ref.accumulate_carve(cloud, [w.shape[0]], o[:1], leaf, max_range, end_margin, variant)
    return ref.evidence()


def test_planted_mistakes_change_the_counters():
    rng = np.random.default_rng(5)
    leaf = 0.5
    # ties: one origin, rays through cell corners; the map holds the cells either tie order visits
    o = np.full((40, 3), 0.25, F)
    d = rng.integers(1, 6, 40).astype(F) * F(0.5)
    w = (o + np.stack([d, d, d * rng.integers(0, 2, 40)], axis=1)).astype(F)
    cells = np.concatenate([c for v in ("", "tie_zyx") for c in [CR.walk(o, w, leaf, v)[1]]])
    good = _evidence(o, w, leaf, cells, "")
    assert not np.array_equal(good, _evidence(o, w, leaf, cells, "tie_zyx"))
    # <= in the range test: axis rays whose entry distances hit max_range exactly
    o2 = np.zeros((3, 3), F)
    w2 = np.array([[8.0, 0, 0], [0, 8.0, 0], [0, 0, -8.0]], F)
    c2 = CR.walk(o2, w2, 1.0)[1]
    assert not np.array_equal(_evidence(o2, w2, 1.0, c2, "", 3.0), _evidence(o2, w2, 1.0, c2, "le", 3.0))
    # a float DDA: rays 1e5 m out at 0.1 m
    o3 = np.repeat((np.array([1e5, -1e5, 30.0]) + rng.uniform(-1, 1, 3)).astype(F)[None], 300, axis=0)
    w3 = (o3 + rng.normal(0, 6.0, (300, 3))).astype(F)
    c3 = np.concatenate([CR.walk(o3, w3, 0.1, v)[1] for v in ("", "float")])
    assert not np.array_equal(_evidence(o3, w3, 0.1, c3, ""), _evidence(o3, w3, 0.1, c3, "float"))
    # a miss per ray: two rays through the same voxels
    o4 = np.zeros((2, 3), F)
    w4 = np.array([[5.2, 0.1, 0.1], [5.3, 0.2, 0.1]], F)
    c4 = CR.walk(o4, w4, 1.0)[1]
    e_good, e_ray = _evidence(o4, w4, 1.0, c4, ""), _evidence(o4, w4, 1.0, c4, "per_ray")
    assert e_good[:, 1].max() == 1 and e_ray[:, 1].max() == 2


def test_hits_are_per_scan_and_new_voxels_are_not_missed():
    ref = CR.CarveMapRef()
    o = np.zeros((1, 3), F)
    cloud = np.array([[4.5, 0.5, 0.5, 0], [4.6, 0.5, 0.5, 0], [2.5, 0.5, 0.5, 0], [np.nan, 0, 0, 0]], F)
    ref.accumulate_carve(cloud, [4], o, 1.0, 100.0, 0.0)
    assert ref.hit[(0, 0, 4)] == 1 and ref.hit[(0, 0, 2)] == 1               # two points, one scan: one hit
    assert ref.miss[(0, 0, 2)] == 0                                          # passed by the ray to x = 4.5, but hit
    ref.accumulate(np.array([[1.5, 0.5, 0.5, 0]], F), 1.0)                   # a plain accumulate: starts at 0, 0
    assert ref.hit[(0, 0, 1)] == 0 and ref.miss[(0, 0, 1)] == 0
    ref.accumulate_carve(cloud[:1], [1], o, 1.0, 100.0, 0.0)
    assert ref.miss[(0, 0, 1)] == 1 and ref.miss[(0, 0, 2)] == 1 and ref.hit[(0, 0, 4)] == 2
    with pytest.raises(V.CapacityError):
        ref.accumulate_carve(cloud[:1], [1], np.array([[3e9, 0, 0]], F), 1.0, 100.0, 0.0)
    assert ref.hit[(0, 0, 4)] == 2


@pytest.mark.parametrize("hit,miss,min_miss,ratio,drop", [
    (0, 0, 0, 0.0, False), (0, 1, 1, 0.0, True), (0, 1, 2, 0.0, False), (1, 2, 2, 2.0, False), (1, 3, 2, 2.0, True),
    (2, 4, 2, 2.0, False), (2, 5, 2, 2.0, True), (10, 5, 6, 0.1, False), (3, 1, 1, 0.25, True), (4, 1, 1, 0.25, False),
    (1, 1, 1, 0.999999, True), (1, 1, 1, 1.0, False), (0xFFFFFFFF, 0xFFFFFFFF, 0, 0.99999994, True)])
def test_keep_rule_at_its_boundaries(hit, miss, min_miss, ratio, drop):
    assert CR.dropped(hit, miss, min_miss, ratio) == drop


# ------------------------------------------------------------------ the street scene and the defaults
N_SCANS = 20
RECENT = 9   # trail voxels the car last covered in the final RECENT scans may stay (see the test's docstring)


def test_street_defaults_clear_the_trail_and_keep_the_static_scene():
    """20 scans, one spinning slot of 32 x 128 rays, 0.5 m leaf, the library's defaults.  Trail voxels (hit only by the
    moving car) that the car left before the last RECENT scans are all dropped.  RECENT is 9: a voxel is dropped after more
    than twice as many scans passed it as hit it, the 4.5 m car covers a voxel for up to 3 scans at 1.5 m a scan, and after
    it passes the sensor (scan 13) it drives away behind it, where 128 azimuths leave gaps that later scans fill only in
    part.  Of the façade and ground voxels the defaults keep 98.2 %, short of 99 %: ground voxels beyond about 10 m are hit
    by few scans of this sparse pattern while grazing rays that land farther out pass them in most scans (the 4 m margin
    covers such a ray only for its last 4 m)."""
    st = synth.Street()
    ref = CR.CarveMapRef()
    labels = {}
    for k in range(N_SCANS):
        s = synth.street_scan(st, k)
        cloud = W.register_world(s["state"], None, s["body"][0], 0, 0.0)
        org = W.register_world(s["state"], None, np.zeros((1, 3), F), 0, 0.0)[:, :3]
        ref.accumulate_carve(cloud, [cloud.shape[0]], org, 0.5, plugin.CARVE_MAX_RANGE, plugin.CARVE_END_MARGIN)
        for key, wh in zip(map(tuple, V.voxel_index(cloud[:, :3], 0.5)[0].tolist()), s["what"][0]):
            labels.setdefault(key, set()).add((int(wh), k))
    drop = {k: CR.dropped(ref.hit[k], ref.miss[k], plugin.KEEP_MIN_MISS, plugin.KEEP_MAX_MISS_PER_HIT) for k in ref.sums}
    trail = {k: max(t for _, t in v) for k, v in labels.items() if all(w == 3 for w, _ in v)}
    assert len(trail) > 200
    old = [k for k, last in trail.items() if last < N_SCANS - RECENT]
    assert len(old) > 100 and all(drop[k] for k in old)
    static = [k for k, v in labels.items() if all(w in (0, 1) for w, _ in v)]
    ground = [k for k in static if all(w == 0 for w, _ in labels[k])]
    keep_static = 1.0 - np.mean([drop[k] for k in static])
    keep_ground = 1.0 - np.mean([drop[k] for k in ground])
    assert keep_static >= 0.98 and keep_ground >= 0.94, (keep_static, keep_ground)


def test_street_generator_is_seeded_and_city_sized():
    st = synth.Street()
    a, b = synth.street_scan(st, 3, L=3, cone=500), synth.street_scan(st, 3, L=3, cone=500)
    for x, y in zip(a["body"], b["body"]):
        assert np.array_equal(x, y)
    assert {3} <= set(synth.street_scan(st, 10)["what"][0].tolist())          # the car is in view
    n = sum(x.shape[0] for x in synth.street_scan_city(st, 0)["body"])
    assert n > 150_000


# ------------------------------------------------------------------ the C-ABI
NEW = ("malio_world_voxel_accumulate_carve", "malio_world_voxel_evidence_device", "malio_world_voxel_download_kept_device",
       "malio_world_voxel_save_pcd_kept")
SCALARS = (("uint64_t", C.c_uint64), ("float", C.c_float), ("int", C.c_int))


def _header_args(name):
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    out = []
    for a in (re.sub(r"/\*.*?\*/", "", a).strip() for a in m.group(1).split(",")):
        if a.startswith("const char*"):
            out.append(C.c_char_p)
        elif "*" in a:
            out.append(C.c_void_p)
        else:
            types = [t for word, t in SCALARS if a.split()[0] == word]
            assert len(types) == 1, f"{name}: unexpected argument {a!r}"
            out.append(types[0])
    return out


@pytest.mark.parametrize("name", NEW)
def test_ctypes_signatures_match_the_header(name):
    fn = getattr(capi.load(), name)
    assert fn.argtypes == _header_args(name)
    assert fn.restype is C.c_int
    assert name in capi.EXPORTS


def test_struct_layout_matches_the_header(tmp_path):
    src = textwrap.dedent("""
        #include <stddef.h>
        #include <stdio.h>
        #include "malio_b200.h"
        #define F(T, f) printf(#T "." #f " %zu\\n", offsetof(T, f))
        int main(void) {
          printf("args %zu\\nkeep %zu\\nbound %.1f\\n", sizeof(malio_carve_args), sizeof(malio_carve_keep), MALIO_CARVE_MAX_RANGE_CELLS);
          F(malio_carve_args, max_range); F(malio_carve_args, end_margin);
          F(malio_carve_keep, min_miss); F(malio_carve_keep, max_miss_per_hit);
          return 0;
        }""")
    c = tmp_path / "layout.c"
    c.write_text(src)
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.rsplit(" ", 1) for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["args"]) == C.sizeof(capi.CarveArgs) and int(out["keep"]) == C.sizeof(capi.CarveKeep)
    assert float(out["bound"]) == 65536.0
    for T, S in (("malio_carve_args", capi.CarveArgs), ("malio_carve_keep", capi.CarveKeep)):
        for f, _ in S._fields_:
            assert int(out[f"{T}.{f}"]) == getattr(S, f).offset, (T, f)


def test_null_handle_and_null_arguments_return_an_error():
    code = textwrap.dedent("""
        import ctypes as C
        from malio_b200 import capi
        lib = capi.load()
        s, t, n = capi.PassState(), (C.c_float * 3)(), C.c_uint64(0)
        a, k = capi.CarveArgs(100.0, 0.5), capi.CarveKeep(2, 2.0)
        print("carve", lib.malio_world_voxel_accumulate_carve(None, None, None, 0.5, None, None), flush=True)
        print("carve-args", lib.malio_world_voxel_accumulate_carve(None, C.addressof(s), C.addressof(t), 0.5, C.addressof(a), C.addressof(n)), flush=True)
        print("evidence", lib.malio_world_voxel_evidence_device(None, None, 0, C.addressof(n), None), flush=True)
        print("kept", lib.malio_world_voxel_download_kept_device(None, C.addressof(k), None, 0, C.addressof(n), None), flush=True)
        print("save", lib.malio_world_voxel_save_pcd_kept(None, b"/nonexistent/x.pcd", C.addressof(k), 1), flush=True)
        print("DONE")
    """)
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "ma-lio_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "DONE" and len(lines) == 6
    for l in lines[:-1]:
        assert l.split()[-1] == str(capi.ERR_INVALID_ARG), l


def test_python_defaults_and_argument_forms():
    a, k = plugin.carve_args(), plugin.carve_keep()
    assert (a.max_range, a.end_margin) == (100.0, 4.0) and (k.min_miss, k.max_miss_per_hit) == (2, 2.0)
    assert plugin._as_carve(None) is None and plugin._as_carve(True).max_range == 100.0
    assert plugin._as_carve(dict(end_margin=1.0)).end_margin == 1.0
    assert plugin._as_keep(dict(min_miss=5)).min_miss == 5 and plugin._as_keep(k) is k
    with pytest.raises(ValueError):
        plugin.PcdSaver(None, "/tmp", 10, carve=True)
