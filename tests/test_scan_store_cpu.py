"""CPU tests of the scan store and the voxel map's rebuild (no GPU):
  - tests/scan_store_ref.py against a direct per-point loop (register each point, fold it with VoxelMapRef.accumulate);
  - the chunking argument: several scans folded as one concatenated chunk give the bytes of folding them scan by scan, with
    chunk boundaries inside runs of one voxel;
  - the ctypes declarations (malio_stored_scan's layout, the new entry points' signatures) against the header, compiled;
  - NULL arguments; the .npz writer and reader on plain arrays."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import carve_ref as CR
import scan_store_ref as SR
import world_ref as W
import world_voxel_ref as V
from malio_b200 import capi, plugin

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _state(rng, scale=1.0):
    s = capi.PassState()
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    s.rot[:] = q
    s.pos[:] = rng.uniform(-5, 5, 3) * scale
    for l in range(capi.MAX_LIDAR):
        e = np.array([1.0, *rng.normal(scale=0.05, size=3)])
        s.ext[l].q[:] = e / np.linalg.norm(e)
        s.ext[l].t[:] = rng.uniform(-0.5, 0.5, 3)
    return s


def _scan(rng, L, sizes, lo=-4.0, hi=4.0):
    tc = np.zeros(capi.MAX_LIDAR - 1, capi.RIGID)
    for i in range(capi.MAX_LIDAR - 1):
        q = np.array([1.0, *rng.normal(scale=0.02, size=3)])
        tc[i]["q"], tc[i]["t"] = q / np.linalg.norm(q), rng.uniform(-0.1, 0.1, 3)
    xyz = rng.uniform(lo, hi, (sum(sizes), 3)).astype(F)
    return dict(state=_state(rng), temporal_comp=tc, slot_tag=np.arange(L, dtype=F) + 0.5, n_points=list(sizes), xyz=xyz)


@pytest.mark.parametrize("L", [1, 3])
def test_restatement_matches_a_direct_per_point_loop(L):
    rng = np.random.default_rng(L)
    sizes = {1: [[300], [0], [250]], 3: [[120, 0, 80], [50, 60, 70], [0, 0, 0], [90, 10, 0]]}[L]
    scans = [_scan(rng, L, s) for s in sizes]
    states = [_state(rng) for _ in scans]
    leaf = 0.7
    for st in (None, states):
        fast = V.VoxelMapRef()
        SR.rebuild(fast, scans, leaf, st)
        slow = V.VoxelMapRef()
        for k, sc in enumerate(scans):
            s = sc["state"] if st is None else st[k]
            rows = []
            at = 0
            for l, m in enumerate(sc["n_points"]):
                for p in range(at, at + m):   # one point at a time, in (slot, point) order
                    rows.append(W.register_world(s, sc["temporal_comp"], sc["xyz"][p:p + 1], l, sc["slot_tag"][l])[0])
                at += m
            slow.accumulate(np.array(rows, F).reshape(-1, 4), leaf)
        assert fast.centroids().tobytes() == slow.centroids().tobytes()
        assert fast.keys().tobytes() == slow.keys().tobytes()


def test_carved_restatement_is_the_per_scan_carve():
    rng = np.random.default_rng(5)
    scans = [_scan(rng, 3, s, -10, 10) for s in ([40, 20, 0], [30, 0, 30], [10, 10, 10])]
    carve = dict(max_range=30.0, end_margin=0.5)
    a, b = CR.CarveMapRef(), CR.CarveMapRef()
    SR.rebuild(a, scans, 1.0, carve=carve)
    for sc in scans:
        b.accumulate_carve(SR.register(sc), sc["n_points"], SR.origins(sc), 1.0, **carve)
    assert a.centroids().tobytes() == b.centroids().tobytes() and a.evidence().tobytes() == b.evidence().tobytes()


def _fold_chunks(clouds, bounds, leaf):
    """Fold the concatenated clouds in chunks [bounds[i], bounds[i + 1]) of rows, each chunk as one stable fold."""
    allc = np.concatenate(clouds)
    ref = V.VoxelMapRef()
    for a, b in zip(bounds[:-1], bounds[1:]):
        ref.accumulate_fast(allc[a:b], leaf)
    return ref


def test_chunks_of_concatenated_scans_give_the_per_scan_bytes():
    """The stable fold continues each voxel's sums point by point, so the split of the rows into chunks does not matter: scans
    that share voxels (runs of one voxel crossing every scan boundary and the chunk boundaries) give the same bytes."""
    rng = np.random.default_rng(11)
    leaf = 1.0
    clouds = []
    for k in range(6):
        c = np.zeros((200, 4), F)
        c[:, :3] = rng.uniform(0.0, 3.0, (200, 3)).astype(F) + rng.normal(scale=1e-3, size=(200, 3)).astype(F)
        c[:100, :3] = F(0.5) + rng.uniform(0, 0.4, (100, 3)).astype(F)   # one voxel in every scan
        c[:, 3] = k
        c[7] = (np.nan, 0.0, 0.0, 1.0)                                   # skipped, as the fold skips it
        clouds.append(c)
    per_scan = V.VoxelMapRef()
    for c in clouds:
        per_scan.accumulate_fast(c, leaf)
    n = sum(c.shape[0] for c in clouds)
    for bounds in ([0, n], [0, 200, 400, 600, 800, 1000, n], [0, 50, 333, 901, n], [0, 1, 2, n - 1, n]):
        got = _fold_chunks(clouds, bounds, leaf)
        assert got.centroids().tobytes() == per_scan.centroids().tobytes(), bounds
        assert got.cnt == per_scan.cnt


# ------------------------------------------------------------------ the C-ABI surface
NEW = ["malio_scan_store_add", "malio_scan_store_put", "malio_scan_store_get", "malio_scan_store_register_device",
       "malio_scan_store_info", "malio_scan_store_clear", "malio_world_voxel_rebuild"]


def _prototype(hdr, name):
    m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", hdr)
    assert m, name
    args = re.sub(r"/\*.*?\*/", "", m.group(1)).split(",")
    return [" ".join(a.split()) for a in args]


def _ctype_of(arg):
    if "*" in arg:
        return C.c_void_p
    base = arg.rsplit(" ", 1)[0]
    return {"uint64_t": C.c_uint64, "float": C.c_float, "double": C.c_double, "uint32_t": C.c_uint32, "int": C.c_int}[base]


def test_signatures_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    lib = capi.load()
    for name in NEW:
        assert name in capi.EXPORTS, name
        want = [_ctype_of(a) for a in _prototype(hdr, name)]
        assert list(getattr(lib, name).argtypes) == want, name
    assert int(re.search(r"#define MALIO_STORE_BLOCK_POINTS \(1u << (\d+)\)", hdr).group(1)) == 24
    assert capi.STORE_BLOCK_POINTS == 1 << 24


def test_stored_scan_layout_matches_the_compiled_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "malio_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(malio_stored_scan), offsetof(malio_stored_scan, time), '
                   'offsetof(malio_stored_scan, state), offsetof(malio_stored_scan, temporal_comp), offsetof(malio_stored_scan, slot_tag), '
                   'offsetof(malio_stored_scan, n_points)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-x", "c", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = capi.StoredScan
    assert got == [C.sizeof(S), S.time.offset, S.state.offset, S.temporal_comp.offset, S.slot_tag.offset, S.n_points.offset]
    assert plugin.STORED_SCAN.itemsize == got[0]
    for f in ("time", "temporal_comp", "slot_tag", "n_points"):
        assert plugin.STORED_SCAN.fields[f][1] == getattr(S, f).offset, f
    assert plugin.STORED_SCAN.fields["rot"][1] == S.state.offset


def test_null_arguments_are_refused():
    lib = capi.load()
    rec, n = capi.StoredScan(), C.c_uint64(0)
    assert lib.malio_scan_store_add(None, None, None, 0.0, None) == capi.ERR_INVALID_ARG
    assert lib.malio_scan_store_put(None, C.byref(rec), None, None) == capi.ERR_INVALID_ARG
    assert lib.malio_scan_store_get(None, 0, C.byref(rec), None, 0, C.byref(n)) == capi.ERR_INVALID_ARG
    assert lib.malio_scan_store_register_device(None, 0, None, None, 0, C.byref(n), None) == capi.ERR_INVALID_ARG
    assert lib.malio_scan_store_info(None, C.byref(n), None, None) == capi.ERR_INVALID_ARG
    assert lib.malio_scan_store_clear(None) == capi.ERR_INVALID_ARG
    assert lib.malio_world_voxel_rebuild(None, 0, 0, None, C.c_float(0.5), None, C.byref(n)) == capi.ERR_INVALID_ARG


# ------------------------------------------------------------------ the .npz file
def _records(rng, counts):
    r = np.zeros(len(counts), plugin.STORED_SCAN)
    r["time"] = rng.uniform(0, 100, len(counts))
    r["rot"] = rng.normal(size=(len(counts), 4))
    r["pos"] = rng.normal(size=(len(counts), 3))
    r["temporal_comp"]["t"] = rng.normal(size=(len(counts), 2, 3))
    r["slot_tag"] = rng.normal(size=(len(counts), 3)).astype(F)
    r["n_points"] = counts
    return r


def test_npz_round_trip(tmp_path):
    rng = np.random.default_rng(3)
    counts = [[5, 0, 2], [0, 0, 0], [1, 1, 1]]
    recs = _records(rng, counts)
    xyz = rng.normal(size=(10, 3)).astype(F)
    xyz[3] = (np.nan, -0.0, np.inf)
    p = tmp_path / "store.npz"
    plugin.write_scan_store_npz(str(p), recs, xyz)
    got, pts = plugin.read_scan_store_npz(str(p))
    assert got.tobytes() == recs.tobytes()
    assert [q.shape[0] for q in pts] == [7, 0, 3]
    assert np.concatenate(pts).tobytes() == xyz.tobytes()
    rec = capi.StoredScan.from_buffer_copy(got[2].tobytes())
    assert list(rec.n_points) == [1, 1, 1] and rec.time == recs["time"][2] and list(rec.state.rot) == list(recs["rot"][2])


def test_npz_refuses_counts_that_do_not_add_up(tmp_path):
    rng = np.random.default_rng(4)
    with pytest.raises(ValueError):
        plugin.write_scan_store_npz(str(tmp_path / "a.npz"), _records(rng, [[2, 0, 0]]), np.zeros((3, 3), F))
    p = tmp_path / "b.npz"
    np.savez(p, format=np.int64(plugin.SCAN_STORE_FORMAT), records=_records(rng, [[2, 0, 0]]), xyz=np.zeros((1, 3), F))
    with pytest.raises(ValueError):
        plugin.read_scan_store_npz(str(p))
    plugin.write_scan_store_npz(str(tmp_path / "empty.npz"), np.zeros(0, plugin.STORED_SCAN), np.zeros((0, 3), F))
    recs, pts = plugin.read_scan_store_npz(str(tmp_path / "empty.npz"))
    assert recs.shape == (0,) and pts == []
