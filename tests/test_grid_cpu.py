"""The 2-D occupancy grid without a GPU: tests/grid_ref.py against a direct per-cell loop at the argument edges (ties, -0.0,
non-finite rows, points on region and pad borders, w in {0, 1, 5}, one-cell regions, h_lo == h_hi), the tiling property,
the PGM / YAML writer through the library (bytes, header, row flip, the map_server decode, refusals, no file left behind),
the C-ABI against the header, and the defaults on a sloped scene (a 10 % ramp and a 0.15 m kerb with boxes on them)."""
import ctypes as C
import os
import re
import subprocess
import textwrap

import numpy as np
import pytest

import grid_ref as G
from malio_b200 import capi, plugin

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
F = np.float32


# ------------------------------------------------------------------ the restatement against a direct loop
def _direct(pts, res, i0, j0, nx, ny, w, h_lo, h_hi, m):
    """Per cell, from the definitions, with Python floats made float32 at every step."""
    ir = F(1.0) / F(res)
    cols = {}
    for x, y, z, _ in np.asarray(pts, F):
        if not (np.isfinite(x) and np.isfinite(y) and np.isfinite(z)):
            continue
        fi, fj = F(np.floor(F(x * ir))), F(np.floor(F(y * ir)))
        if i0 - w <= fi < i0 + nx + w and j0 - w <= fj < j0 + ny + w:
            cols.setdefault((int(fi), int(fj)), []).append(F(z))

    def lowest(zs):   # the key order: -0.0 below +0.0
        return min(zs, key=lambda v: (float(v), not np.signbit(v)))

    zmin = {c: lowest(v) for c, v in cols.items()}
    cls = np.zeros((ny, nx), np.uint8)
    ground = np.zeros((ny, nx), F)
    for r in range(ny):
        for c in range(nx):
            i, j = i0 + c, j0 + r
            win = [zmin[(a, b)] for a in range(i - w, i + w + 1) for b in range(j - w, j + w + 1) if (a, b) in zmin]
            g = lowest(win) if win else F(np.nan)
            ground[r, c] = g
            band = floor = 0
            for z in cols.get((i, j), []):
                d = F(z - g)
                band += F(h_lo) <= d <= F(h_hi)
                floor += d < F(h_lo)
            cls[r, c] = G.OCCUPIED if band >= m else (G.FREE if floor else G.UNKNOWN)
    return cls, ground


def _cloud(rng, n, res, i0, j0, nx, ny, w):
    """Points over and around the padded region, with exact cell borders, ties, -0.0 and non-finite rows."""
    lo = np.array([(i0 - w - 2) * res, (j0 - w - 2) * res])
    hi = np.array([(i0 + nx + w + 2) * res, (j0 + ny + w + 2) * res])
    xy = rng.uniform(lo, hi, (n, 2))
    k = n // 4
    xy[:k] = np.round(xy[:k] / res) * res                                  # on cell faces, pad and region borders included
    xy[k] = [(i0 - w) * res, (j0 - w) * res]
    xy[k + 1] = [(i0 + nx + w) * res, (j0 + ny + w) * res]
    xy[k + 2] = [i0 * res, (j0 + ny) * res]
    z = rng.choice(np.array([0.0, 0.1, 0.3, 0.5, 1.2, 2.0, 2.5], F), n) + F(0.01) * rng.integers(0, 3, n).astype(F)
    z[: n // 8] = rng.choice(np.array([-0.0, 0.0], F), n // 8)            # ties and signed zeros
    pts = np.concatenate([xy.astype(F), z[:, None].astype(F), rng.uniform(0, 1, (n, 1)).astype(F)], axis=1)
    pts[-1, 0], pts[-2, 1], pts[-3, 2] = np.nan, np.inf, -np.inf
    return pts


EDGES = [   # res, i0, j0, nx, ny, w, h_lo, h_hi, m
    (0.1, -5, -4, 9, 7, 0, 0.3, 2.0, 1),
    (0.1, -5, -4, 9, 7, 1, 0.3, 2.0, 2),
    (0.25, 3, -2, 6, 5, 5, 0.3, 2.0, 1),
    (0.1, 2, 3, 1, 1, 1, 0.2, 0.2, 1),
    (0.1, 0, 0, 1, 6, 5, 0.5, 0.5, 1),
    (0.2, -1, 0, 7, 1, 0, 0.1, 1.0, 3),
]


@pytest.mark.parametrize("edge", EDGES)
def test_restatement_equals_a_direct_loop(edge):
    res, i0, j0, nx, ny, w, h_lo, h_hi, m = edge
    rng = np.random.default_rng(nx * 31 + ny * 7 + w)
    pts = _cloud(rng, 400, res, i0, j0, nx, ny, w)
    cls, ground, rep = G.grid(pts, res, i0, j0, nx, ny, w, h_lo, h_hi, m)
    dc, dg = _direct(pts, res, i0, j0, nx, ny, w, h_lo, h_hi, m)
    assert np.array_equal(cls, dc)
    assert ground.tobytes() == np.where(np.isnan(dg), np.frombuffer(G.GROUND_NAN.tobytes(), F)[0], dg).astype(F).tobytes()
    assert rep["n_nonfinite"] == 3 and rep["n_used"] + rep["n_outside"] + 3 == pts.shape[0]
    assert rep["n_occupied"] + rep["n_free"] + rep["n_unknown"] == nx * ny


def test_signed_zero_is_the_lower_ground():
    pts = np.array([[0.05, 0.05, 0.0, 0], [0.05, 0.05, -0.0, 0]], F)
    _, ground, _ = G.grid(pts, 0.1, 0, 0, 1, 1, 0, 0.3, 2.0, 1)
    assert np.signbit(ground[0, 0]) and ground[0, 0] == 0


def test_tiling_equals_the_whole_region():
    rng = np.random.default_rng(3)
    args = (0.1, -12, -9, 24, 18)
    w = 4
    pts = _cloud(rng, 3000, *args, w)
    whole_c, whole_g, _ = G.grid(pts, *args, w, 0.3, 2.0, 2)
    for (ci, cj, cnx, cny) in ((-12, -9, 10, 7), (-2, -9, 14, 7), (-12, -2, 10, 11), (-2, -2, 14, 11), (-5, -4, 1, 1)):
        c, g, _ = G.grid(pts, 0.1, ci, cj, cnx, cny, w, 0.3, 2.0, 2)
        sl = (slice(cj + 9, cj + 9 + cny), slice(ci + 12, ci + 12 + cnx))
        assert np.array_equal(c, whole_c[sl]) and g.tobytes() == np.ascontiguousarray(whole_g[sl]).tobytes()


@pytest.mark.parametrize("bad", [
    dict(res=0.0), dict(res=float("nan")), dict(nx=0), dict(ny=0), dict(h_lo=0.0), dict(h_lo=2.5), dict(h_hi=float("inf")),
    dict(m=0), dict(i0=(1 << 24) - 3, w=4), dict(j0=-(1 << 24) + 2, w=3)])
def test_restatement_refusals(bad):
    a = dict(res=0.1, i0=0, j0=0, nx=4, ny=4, w=1, h_lo=0.3, h_hi=2.0, m=1)
    a.update(bad)
    with pytest.raises(G.ArgumentError):
        G.grid(np.zeros((1, 4), F), a["res"], a["i0"], a["j0"], a["nx"], a["ny"], a["w"], a["h_lo"], a["h_hi"], a["m"])


def test_extent_restatement():
    pts = np.array([[0.05, -0.31, 0, 0], [1.0, 2.0, 0, 0], [np.nan, 100, 0, 0], [5, 5, np.inf, 0]], F)
    assert G.extent(pts, 0.1) == (0, -4, 10, 20)
    assert G.extent(pts[2:], 0.1) == (0, 0, -1, -1)
    with pytest.raises(ValueError):
        G.extent(np.array([[2e6, 0, 0, 0]], F), 0.1)


# ------------------------------------------------------------------ the sloped scene and the defaults
def sloped_scene(rng, res=0.05):
    """A 10 % ramp rising along +x over x in [0, 20] m (flat before and after), a 0.15 m kerb along y = 4 m with a pavement
    behind it, and boxes (1 x 1 x 1 m) standing on the ramp and on the pavement.  Points on a res / 2 lattice with 1 cm noise.
    Returns (points float32 (n, 4), boxes [(lo, hi)], ramp_road (x0, x1, y0, y1), kerb y)."""
    def surface(x, y):
        ramp = np.clip(x, 0.0, 20.0) * 0.1
        return ramp + np.where(y >= 4.0, 0.15, 0.0)
    xs, ys = np.meshgrid(np.arange(-5.0, 25.0, res / 2), np.arange(-4.0, 8.0, res / 2), indexing="ij")
    x, y = xs.ravel(), ys.ravel()
    z = surface(x, y) + rng.normal(0, 0.01, x.shape[0])
    pts = [np.stack([x, y, z], 1)]
    boxes = [((5.0, -1.0), 1.0), ((14.0, 1.0), 1.0), ((8.0, 5.5), 1.0)]
    out = []
    for (bx, by), h in boxes:
        base = surface(bx + 0.5, by + 0.5)
        u, v, t = np.meshgrid(np.arange(0, 1.0001, res / 2), np.arange(0, 1.0001, res / 2), np.arange(0, h + 1e-4, res / 2), indexing="ij")
        p = np.stack([bx + u.ravel(), by + v.ravel(), base + t.ravel()], 1)
        shell = (np.isclose(u.ravel(), 0) | np.isclose(u.ravel(), 1.0) | np.isclose(v.ravel(), 0) | np.isclose(v.ravel(), 1.0) |
                 np.isclose(t.ravel(), h))
        pts.append(p[shell])
        out.append((np.array([bx, by]), np.array([bx + 1.0, by + 1.0])))
    p = np.concatenate(pts)
    return np.concatenate([p, np.zeros((p.shape[0], 1))], 1).astype(F), out


def _cells_in(lo, hi, res, i0, j0, nx, ny, inset):
    i = np.arange(nx) + i0
    j = np.arange(ny) + j0
    cx, cy = (i + 0.5) * res, (j + 0.5) * res
    mx = (cx >= lo[0] + inset) & (cx < hi[0] - inset)
    my = (cy >= lo[1] + inset) & (cy < hi[1] - inset)
    return my[:, None] & mx[None, :]


def test_defaults_on_the_sloped_scene():
    """The library's defaults: the box footprints are occupied, the ramp and the kerb (a 0.15 m step, below h_lo) are free, but
    for the kerb's cells on the ramp, where the 1 m ground window reaches 0.1 m down the slope (98.8 % free).  A fixed global
    height band would mark the top of the ramp (2 m above its foot) as obstacle."""
    pts, boxes = sloped_scene(np.random.default_rng(0))
    a = plugin.grid_args()
    res = a.res
    e = G.extent(pts, res)
    i0, j0, nx, ny = e[0], e[1], e[2] - e[0] + 1, e[3] - e[1] + 1
    cls, _, _ = G.grid(pts, res, i0, j0, nx, ny, a.ground_halfwidth, a.h_lo, a.h_hi, a.min_obstacle_points)
    foot = np.zeros_like(cls, bool)
    for lo, hi in boxes:
        m = _cells_in(lo, hi, res, i0, j0, nx, ny, 0.0)
        foot |= _cells_in(lo - 0.3, hi + 0.3, res, i0, j0, nx, ny, 0.0)
        assert np.mean(cls[m] == G.OCCUPIED) >= 0.5, (lo, np.mean(cls[m] == G.OCCUPIED))
    ramp = _cells_in(np.array([-4.0, -3.5]), np.array([24.0, 7.5]), res, i0, j0, nx, ny, 0.0) & ~foot
    assert np.mean(cls[ramp] == G.FREE) >= 0.985, np.mean(cls[ramp] == G.FREE)


# ------------------------------------------------------------------ the writer through the library
def _write(tmp_path, cls, res=0.1, i0=-3, j0=7, stem="map"):
    pgm, yaml = str(tmp_path / f"{stem}.pgm"), str(tmp_path / f"{stem}.yaml")
    c = np.ascontiguousarray(cls, np.uint8)
    rc = capi.load().malio_write_grid_pgm(os.fsencode(pgm), os.fsencode(yaml), capi.ptr(c), c.shape[1], c.shape[0], C.c_float(res), i0, j0)
    return rc, pgm, yaml


def test_writer_bytes_header_flip_and_decode(tmp_path):
    rng = np.random.default_rng(1)
    cls = rng.choice(np.array([G.FREE, G.OCCUPIED, G.UNKNOWN], np.uint8), (5, 7))
    rc, pgm, yaml = _write(tmp_path, cls)
    assert rc == capi.OK
    data = open(pgm, "rb").read()
    hdr = b"P5\n7 5\n255\n"
    assert data[: len(hdr)] == hdr and len(data) == len(hdr) + 35
    body = np.frombuffer(data[len(hdr):], np.uint8).reshape(5, 7)
    assert np.array_equal(body, G.pgm_values(cls))
    assert np.array_equal(body[0], G.pgm_values(cls)[0]) and np.array_equal(body[-1], np.where(cls[0] == 100, 0, np.where(cls[0] == 0, 254, 205)))
    y = dict(l.split(": ", 1) for l in open(yaml).read().splitlines())
    assert y["image"] == "map.pgm" and y["mode"] == "trinary" and y["negate"] == "0"
    assert F(float(y["resolution"])) == F(0.1)                              # the float res, round-trip
    org = [float(v) for v in y["origin"].strip("[]").split(",")]
    assert org == [-3 * float(F(0.1)), 7 * float(F(0.1)), 0.0]
    assert np.array_equal(G.decode(body, float(y["occupied_thresh"]), float(y["free_thresh"])), cls)


def test_plugin_save_grid(tmp_path):
    cls = np.full((3, 4), G.UNKNOWN, np.uint8)
    cls[0, 0], cls[2, 3] = G.OCCUPIED, G.FREE
    a = plugin.grid_args(i0=10, j0=-2, nx=4, ny=3)
    pgm, yaml = plugin.save_grid(str(tmp_path / "g"), cls, a)
    body = np.frombuffer(open(pgm, "rb").read()[len(b"P5\n4 3\n255\n"):], np.uint8).reshape(3, 4)
    assert body[2, 0] == 0 and body[0, 3] == 254 and (body == 205).sum() == 10
    with pytest.raises(ValueError):
        plugin.save_grid(str(tmp_path / "h"), cls[:2], a)


@pytest.mark.parametrize("case", ["bad_value", "yaml_dir", "pgm_dir", "res", "nx"])
def test_writer_refusals_leave_no_file(tmp_path, case):
    cls = np.zeros((2, 3), np.uint8)
    lib = capi.load()
    pgm, yaml = str(tmp_path / "m.pgm"), str(tmp_path / "m.yaml")
    if case == "bad_value":
        cls[1, 2] = 50
    if case == "yaml_dir":
        yaml = str(tmp_path / "missing" / "m.yaml")
    if case == "pgm_dir":
        pgm = str(tmp_path / "missing" / "m.pgm")
    res = 0.0 if case == "res" else 0.1
    nx = 0 if case == "nx" else 3
    rc = lib.malio_write_grid_pgm(os.fsencode(pgm), os.fsencode(yaml), capi.ptr(cls), nx, 2, C.c_float(res), 0, 0)
    assert rc == capi.ERR_INVALID_ARG
    assert os.listdir(tmp_path) == []


# ------------------------------------------------------------------ the C-ABI
NEW = ("malio_grid_build_device", "malio_grid_build", "malio_grid_extent_device", "malio_write_grid_pgm")
SCALARS = (("uint64_t", C.c_uint64), ("uint32_t", C.c_uint32), ("int32_t", C.c_int32), ("float", C.c_float), ("int", C.c_int))


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
          printf("args %zu\\nreport %zu\\nmax %llu\\nbound %d\\nsrc %d %d %d\\ncls %d %d %d\\n", sizeof(malio_grid_args),
                 sizeof(malio_grid_report), MALIO_GRID_MAX_BYTES, MALIO_GRID_MAX_BOUND, MALIO_GRID_POINTS, MALIO_GRID_VOXEL_MAP,
                 MALIO_GRID_PRIOR, MALIO_GRID_FREE, MALIO_GRID_OCCUPIED, MALIO_GRID_UNKNOWN);
          F(malio_grid_args, res); F(malio_grid_args, i0); F(malio_grid_args, j0); F(malio_grid_args, nx); F(malio_grid_args, ny);
          F(malio_grid_args, ground_halfwidth); F(malio_grid_args, h_lo); F(malio_grid_args, h_hi);
          F(malio_grid_args, min_obstacle_points);
          F(malio_grid_report, n_used); F(malio_grid_report, n_nonfinite); F(malio_grid_report, n_outside);
          F(malio_grid_report, n_occupied); F(malio_grid_report, n_free); F(malio_grid_report, n_unknown);
          F(malio_grid_report, device_bytes);
          return 0;
        }""")
    c = tmp_path / "layout.c"
    c.write_text(src)
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split(" ", 1) for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["args"]) == C.sizeof(capi.GridArgs) and int(out["report"]) == C.sizeof(capi.GridReport)
    assert int(out["max"]) == capi.GRID_MAX_BYTES and int(out["bound"]) == capi.GRID_MAX_BOUND == G.MAX_BOUND
    assert out["src"] == f"{capi.GRID_POINTS} {capi.GRID_VOXEL_MAP} {capi.GRID_PRIOR}"
    assert out["cls"] == f"{G.FREE} {G.OCCUPIED} {G.UNKNOWN}" == f"{capi.GRID_FREE} {capi.GRID_OCCUPIED} {capi.GRID_UNKNOWN}"
    for T, S in (("malio_grid_args", capi.GridArgs), ("malio_grid_report", capi.GridReport)):
        for f, _ in S._fields_:
            assert int(out[f"{T}.{f}"]) == getattr(S, f).offset, (T, f)


def test_null_arguments_return_an_error():
    lib = capi.load()
    a = plugin.grid_args(nx=4, ny=4)
    ext = (C.c_int32 * 4)()
    cls = (C.c_uint8 * 16)()
    assert lib.malio_grid_build_device(None, 0, None, 0, None, C.byref(a), cls, None, None, None) == capi.ERR_INVALID_ARG
    assert lib.malio_grid_build(None, None, 0, C.byref(a), cls, None, None) == capi.ERR_INVALID_ARG
    assert lib.malio_grid_extent_device(None, 0, None, 0, None, 0.1, ext, None) == capi.ERR_INVALID_ARG
    assert lib.malio_write_grid_pgm(None, None, None, 0, 0, 0.0, 0, 0) == capi.ERR_INVALID_ARG
    assert lib.malio_write_grid_pgm(b"/nonexistent/a.pgm", b"/nonexistent/a.yaml", cls, 4, 4, 0.1, 0, 0) == capi.ERR_INVALID_ARG


def test_python_defaults():
    a = plugin.grid_args()
    assert (round(a.res, 6), a.ground_halfwidth, round(a.h_lo, 6), round(a.h_hi, 6), a.min_obstacle_points) == (0.1, 10, 0.3, 2.0, 1)
    assert plugin.GRID_SOURCES == {"points": 0, "voxel_map": 1, "prior": 2}
