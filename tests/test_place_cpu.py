"""Place descriptors without a GPU: the numpy restatement (tests/place_ref.py) of the binning table against exact arithmetic and
high-precision angles, its tie rules and quarter-turn invariance, the descriptor's shift under a quarter-turned column grid,
stages 1 and 2 against plain loops (ties included), and the C-ABI: struct layouts against the header (gcc), the signatures,
and NULL arguments answered with an error code (in a subprocess: a missing check would be a segmentation fault)."""
import ctypes as C
import math
import os
import re
import subprocess
import sys
import textwrap
from fractions import Fraction

import numpy as np
import pytest

import place_ref as PR
from malio_b200 import capi, plugin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _args(**kw):
    return PR._args_dict(plugin.MeasurementModel.place_args(1.8, **kw))


# ------------------------------------------------------------------ the binning table
@pytest.mark.parametrize("kw", [{}, dict(n_sector=8, n_ring=4, r_max=12.0), dict(cell=0.5, step=1.5, r_max=20.0, n_sector=36)])
def test_every_stencil_offset_lands_in_one_bin_at_the_exact_ring_and_angle(kw):
    a = _args(**kw)
    t = PR.table(a)
    R, S = t["R"], a["n_sector"]
    want = {(ox, oy) for oy in range(-R, R + 1) for ox in range(-R, R + 1)
            if (ox, oy) != (0, 0) and Fraction(ox * ox + oy * oy) * Fraction(a["cell"]) ** 2 < Fraction(a["r_max"]) ** 2}
    got = list(zip(t["ox"].tolist(), t["oy"].tolist()))
    assert len(got) == len(set(got)) and set(got) == want
    assert np.all((t["bin"] >= 0) & (t["bin"] < a["n_ring"] * S)) and np.array_equal(t["bin"], t["ring"] * S + t["sector"])
    n_boundary = 0
    for ox, oy, ring, sec in zip(t["ox"].tolist(), t["oy"].tolist(), t["ring"].tolist(), t["sector"].tolist()):
        # ring: exact rationals (the radii of these arguments are exact in double)
        r2 = Fraction(ox * ox + oy * oy) * Fraction(a["cell"]) ** 2
        assert ring == sum(1 for k in range(1, a["n_ring"]) if r2 >= (Fraction(a["r_max"]) * k / a["n_ring"]) ** 2)
        # sector: the angle in units of a sector, away from boundaries; on a boundary, the counter-clockwise sector
        u = (math.atan2(oy, ox) % (2 * math.pi)) / (2 * math.pi / S)
        if abs(u - round(u)) > 1e-9:
            assert sec == int(math.floor(u)), (ox, oy, u, sec)
        elif ox == 0 or oy == 0 or abs(ox) == abs(oy):   # exact boundaries: the axes, and the diagonals when 8 | n_sector
            assert sec == round(u) % S, (ox, oy, u, sec)
            n_boundary += 1
    assert n_boundary >= 4


def test_ring_boundaries_go_to_the_outer_ring():
    a = _args()
    assert PR.ring_of(a, 3.0, 0.0) == 1 and PR.ring_of(a, 2.0, 2.0) == 0 and PR.ring_of(a, 0.0, -6.0) == 2
    assert PR.ring_of(a, 59.0, 0.0) == 19


def test_a_quarter_turned_offset_lands_a_quarter_of_the_sectors_on():
    for kw in ({}, dict(n_sector=8, n_ring=4, r_max=12.0), dict(n_sector=36, cell=0.5, step=1.0, r_max=15.0)):
        a = _args(**kw)
        t = PR.table(a)
        S, Q = a["n_sector"], a["n_sector"] // 4
        look = {(ox, oy): (r, s) for ox, oy, r, s in zip(t["ox"].tolist(), t["oy"].tolist(), t["ring"].tolist(), t["sector"].tolist())}
        for (ox, oy), (r, s) in look.items():
            assert look[(-oy, ox)] == (r, (s + Q) % S), (ox, oy)


def test_caps_follow_the_field_of_view():
    a = _args(fov_up=math.radians(15.0))
    c = PR.caps(a)
    assert c[0] == PR.level(0.0, a["z_lo"], a["dz"]) and np.all(np.diff(c) >= 0) and c.max() <= 15 and c.min() >= 1
    assert np.all(PR.caps(_args()) == 15)


# ------------------------------------------------------------------ the descriptor
def test_a_quarter_turned_column_grid_shifts_the_descriptor_by_a_quarter():
    rng = np.random.default_rng(3)
    for kw in ({}, dict(fov_up=math.radians(20.0)), dict(n_sector=8, n_ring=4, r_max=12.0)):
        a = _args(**kw)
        t = PR.table(a)
        R, S = t["R"], a["n_sector"]
        cols = {}
        for _ in range(600):
            cols[(int(rng.integers(-R, R + 1)), int(rng.integers(-R, R + 1)))] = float(rng.uniform(-3, 20))
        turned = {(-y, x): z for (x, y), z in cols.items()}
        h = lambda c: np.array([c.get((ox, oy), np.nan) for ox, oy in zip(t["ox"].tolist(), t["oy"].tolist())])
        d, dt = PR.describe(a, t, h(cols)), PR.describe(a, t, h(turned))
        D, DT = d.reshape(a["n_ring"], S), dt.reshape(a["n_ring"], S)
        assert np.array_equal(DT, np.roll(D, S // 4, axis=1))
        assert np.array_equal(PR.ring_keys(a, d), PR.ring_keys(a, dt))
        assert d.max() <= 15 and d.min() >= 0 and d.any()


def test_levels_and_packing():
    z_lo, dz = -2.5, 1.0
    z = np.array([-2.51, -2.5, -1.5000001, -1.5, 12.0, 1e9, np.nan])
    assert PR.level(z, z_lo, dz).tolist() == [0, 1, 1, 2, 15, 15, 0]
    d = np.random.default_rng(1).integers(0, 16, (5, 1201))
    assert np.array_equal(PR.unpack(PR.pack(d), 1201), d)


def test_database_positions_sit_on_the_lattice_in_row_order():
    rng = np.random.default_rng(4)
    a = _args(r_max=10.0, n_ring=5, n_sector=12, step=3.0)
    prior = np.concatenate([rng.uniform(-20, 20, (400, 3)), np.array([[-3.0, -3.0, 0.25], [-3.0, -3.0, 1.0]])]).astype(np.float32)
    db = PR.database(prior, a)
    assert np.all(db["cols"] % 3 == 0)
    key = db["cols"][:, 1] * 10 ** 6 + db["cols"][:, 0]
    assert np.all(np.diff(key) > 0)
    k = np.flatnonzero((db["cols"][:, 0] == -3) & (db["cols"][:, 1] == -3))
    assert len(k) == 1 and db["z_s"][k[0]] == float(np.float32(0.25)) + 1.8
    assert np.array_equal(db["ring_keys"], db["levels"].reshape(len(key), 5, 12).sum(axis=2))


# ------------------------------------------------------------------ ranking
def _loop_stage1(qk, rk, k1):
    items = []
    for p in range(len(rk)):
        items.append((sum(abs(int(rk[p][r]) - int(qk[r])) for r in range(len(qk))), p))
    items.sort()
    return items[:k1]


def _loop_stage2(q, levels, surv, n_ring, S, k2):
    items = []
    for p in surv:
        best = None
        for s in range(S):
            d = sum(abs(int(q[r * S + c]) - int(levels[p][r * S + (c + s) % S])) for r in range(n_ring) for c in range(S))
            if best is None or d < best[0]:
                best = (d, s)
        items.append((best[0], int(p), best[1]))
    items.sort(key=lambda x: (x[0], x[1]))
    return items[:k2]


@pytest.mark.parametrize("seed", range(4))
def test_stages_one_and_two_equal_plain_loops_ties_included(seed):
    rng = np.random.default_rng(seed)
    n_ring, S = 3, 8
    levels = rng.integers(0, 3, (40, n_ring * S))
    levels[20:30] = levels[0:10]                     # identical copies: stage-1 and stage-2 ties
    levels[30] = np.roll(levels[1].reshape(n_ring, S), 3, axis=1).ravel()   # a turned copy
    q = levels[1].copy()
    rk = levels.reshape(40, n_ring, S).sum(axis=2)
    qk = q.reshape(n_ring, S).sum(axis=1)
    surv, d1 = PR.stage1(qk, rk, 16)
    assert list(zip(d1.tolist(), surv.tolist())) == _loop_stage1(qk, rk, 16)
    a = dict(n_ring=n_ring, n_sector=S)
    p2, d2, sh = PR.stage2(q, levels, surv, a, 6)
    assert list(zip(d2.tolist(), p2.tolist(), sh.tolist())) == _loop_stage2(q, levels, surv.tolist(), n_ring, S, 6)
    assert p2[0] == 1 and d2[0] == 0 and sh[0] == 0


# ------------------------------------------------------------------ the C-ABI
def _gcc_layout():
    fields = {
        "malio_place_args": [f for f, _ in capi.PlaceArgs._fields_],
        "malio_place_db_report": [f for f, _ in capi.PlaceDbReport._fields_],
        "malio_global_args": [f for f, _ in capi.GlobalArgs._fields_],
        "malio_global_candidate": [f for f, _ in capi.GlobalCandidate._fields_],
        "malio_global_report": [f for f, _ in capi.GlobalReport._fields_],
    }
    body = "\n".join(f'printf("{T} %zu\\n", sizeof({T}));' for T in fields)
    body += "\n" + "\n".join(f"F({T}, {f});" for T, fs in fields.items() for f in fs)
    body += textwrap.dedent("""
        printf("MAX %d %d %d %d %d\\n", MALIO_PLACE_MAX_BINS, MALIO_PLACE_MAX_K1, MALIO_PLACE_MAX_K2, MALIO_PLACE_MAX_RADIUS_CELLS, 0);""")
    return ("#include <stddef.h>\n#include <stdio.h>\n#include \"malio_b200.h\"\n"
            "#define F(T, f) printf(#T \".\" #f \" %zu\\n\", offsetof(T, f))\nint main(void) {\n" + body + "\nreturn 0;\n}\n")


def test_struct_layout_matches_the_header(tmp_path):
    c = tmp_path / "layout.c"
    c.write_text(_gcc_layout())
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    out = dict(l.split(" ", 1) for l in lines)
    assert out["MAX"].split()[:3] == [str(capi.PLACE_MAX_BINS), str(capi.PLACE_MAX_K1), str(capi.PLACE_MAX_K2)]
    for T, cls in (("malio_place_args", capi.PlaceArgs), ("malio_place_db_report", capi.PlaceDbReport),
                   ("malio_global_args", capi.GlobalArgs), ("malio_global_candidate", capi.GlobalCandidate),
                   ("malio_global_report", capi.GlobalReport)):
        assert int(out[T]) == C.sizeof(cls), T
        for f, _ in cls._fields_:
            assert int(out[f"{T}.{f}"]) == getattr(cls, f).offset, (T, f)


def test_signatures_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    want = {
        "malio_place_db_build": ["malio_handle* h", "const malio_place_args* a", "malio_place_db_report* rep"],
        "malio_place_db_info": ["malio_handle* h", "uint64_t* n_positions", "uint64_t* device_bytes"],
        "malio_place_db_download": ["malio_handle* h", "int32_t* cols", "double* z_s", "uint8_t* nibbles", "uint16_t* ring_keys",
                                    "uint64_t cap", "uint64_t* n"],
        "malio_relocalize_global": ["malio_handle* h", "const malio_pass_state* s", "const malio_global_args* a",
                                    "malio_global_report* rep"],
    }
    lib = capi.load()
    for name, args in want.items():
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
        assert m, name
        assert [x.strip() for x in m.group(1).replace("\n", " ").split(",")] == args, name
        fn = getattr(lib, name)
        assert len(fn.argtypes) == len(args) and fn.restype is C.c_int and name in capi.EXPORTS


def test_null_handle_and_null_arguments_return_an_error():
    code = textwrap.dedent("""
        import ctypes as C
        from malio_b200 import capi
        lib = capi.load()
        s, pa, pr, ga, gr = capi.PassState(), capi.PlaceArgs(), capi.PlaceDbReport(), capi.GlobalArgs(), capi.GlobalReport()
        n = C.c_uint64(0)
        print("build", lib.malio_place_db_build(None, C.byref(pa), C.byref(pr)), flush=True)
        print("build-null", lib.malio_place_db_build(None, None, None), flush=True)
        print("info", lib.malio_place_db_info(None, C.byref(n), C.byref(n)), flush=True)
        print("download", lib.malio_place_db_download(None, None, None, None, None, 0, C.byref(n)), flush=True)
        print("global", lib.malio_relocalize_global(None, C.byref(s), C.byref(ga), C.byref(gr)), flush=True)
        print("global-null", lib.malio_relocalize_global(None, None, None, None), flush=True)
        print("DONE")
    """)
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "ma-lio_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "DONE" and len(lines) == 7
    for l in lines[:-1]:
        assert l.split()[-1] == str(capi.ERR_INVALID_ARG), l
