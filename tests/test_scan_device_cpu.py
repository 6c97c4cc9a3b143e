"""The measurement path's device-memory entry points without a GPU: their ctypes signatures against the header, NULL handles and
NULL arguments answered with an error code (in a subprocess: a missing check would be a segmentation fault), the torch
wrappers' argument checks, which run before anything reaches the library, and pack_scan_tensor against numpy records."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from malio_b200 import capi, plugin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("malio_upload_scan_from_device", "malio_download_aux_device", "malio_map_incremental_device", "malio_world_register_device")


def _header_args(name):
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    args = [re.sub(r"/\*.*?\*/", "", a).strip() for a in m.group(1).split(",")]
    out = []
    for a in args:
        if "*" in a:
            out.append(C.c_void_p)
        elif a.startswith("uint32_t"):
            out.append(C.c_uint32)
        elif a.startswith("double"):
            out.append(C.c_double)
        elif a.startswith("int "):
            out.append(C.c_int)
        else:
            raise AssertionError(f"{name}: unexpected argument {a!r}")
    return out


@pytest.mark.parametrize("name", NEW)
def test_ctypes_signatures_match_the_header(name):
    lib = capi.load()
    fn = getattr(lib, name)
    assert fn.argtypes == _header_args(name)
    assert fn.restype is C.c_int
    assert name in capi.EXPORTS


def test_header_signatures_carry_their_scalars():
    # the parser above must see the double and the int arguments, not only pointers
    assert _header_args("malio_map_incremental_device")[2:4] == [C.c_double, C.c_int]
    assert _header_args("malio_world_register_device")[2] is C.c_int


def test_null_handle_and_null_arguments_return_an_error():
    code = textwrap.dedent("""
        from malio_b200 import capi
        lib = capi.load()
        for n in (0, 5):
            print("upload", n, lib.malio_upload_scan_from_device(None, None, n, None, None, None, None), flush=True)
            print("aux", n, lib.malio_download_aux_device(None, None, None, None, None, None, None), flush=True)
            print("incr", n, lib.malio_map_incremental_device(None, None, 0.5, 1, None, None, None), flush=True)
            print("world", n, lib.malio_world_register_device(None, None, 0, None, None, n, None, None), flush=True)
        print("DONE")
    """)
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "ma-lio_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "DONE" and len(lines) == 9
    for l in lines[:-1]:
        assert l.split()[2] == str(capi.ERR_INVALID_ARG), l


class _Lib:
    """Stands in for the library: any call reaching it fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _model():
    m = object.__new__(plugin.MeasurementModel)   # no handle (no GPU here): only the Python-side checks can run
    m.lib, m._h, m.device, m.n_lidar, m.n_points = _Lib(), C.c_void_p(), 0, 1, 0
    return m


@pytest.mark.parametrize("bad", ["cpu", "float32", "int64", "shape", "rank", "non_contiguous", "numpy"])
def test_upload_scan_tensor_rejects_before_the_call(bad):
    p = {"cpu": torch.zeros((8, 4), dtype=torch.int32), "float32": torch.zeros((8, 4)),
         "int64": torch.zeros((8, 4), dtype=torch.int64), "shape": torch.zeros((8, 3), dtype=torch.int32),
         "rank": torch.zeros(32, dtype=torch.int32), "non_contiguous": torch.zeros((8, 8), dtype=torch.int32)[:, ::2],
         "numpy": np.zeros((8, 4), np.int32)}[bad]
    table = np.zeros(2, dtype=capi.POSE_ENTRY)
    with pytest.raises(ValueError) as e:
        _model().upload_scan_tensor(p, table, np.array([0, 2], np.uint32), None)
    if bad == "non_contiguous":
        assert "contiguous" in str(e.value)


def _records_numpy(xyz, lidar, table_idx):
    r = np.zeros(xyz.shape[0], dtype=capi.SCAN_PT)
    r["xyz"], r["lidar"], r["table_idx"] = xyz, lidar, table_idx
    return r


def test_pack_scan_tensor_equals_numpy_records():
    rng = np.random.default_rng(3)
    n = 5000
    xyz = rng.normal(0, 30, (n, 3)).astype(np.float32)
    xyz[:4] = [[np.nan, 0, -0.0], [np.inf, -np.inf, 1e-45], [0, 0, 0], [-1, 2, 3]]   # the bits are copied, not the values
    lidar = rng.integers(0, 3, n)
    tidx = rng.integers(0, 65536, n)
    tidx[:3] = [0, 65535, 32768]
    lidar[:3] = [65535, 0, 32768]
    ref = _records_numpy(xyz, lidar, tidx)
    for lt, tt in ((torch.int64, torch.int64), (torch.int32, torch.int32), (torch.int32, torch.int64)):
        out = plugin.pack_scan_tensor(torch.from_numpy(xyz), torch.from_numpy(lidar).to(lt), torch.from_numpy(tidx).to(tt))
        assert out.dtype == torch.int32 and tuple(out.shape) == (n, 4) and out.is_contiguous()
        assert out.numpy().tobytes() == ref.tobytes()
    small = plugin.pack_scan_tensor(torch.from_numpy(xyz[:10]), torch.zeros(10, dtype=torch.uint8), torch.ones(10, dtype=torch.int16))
    assert small.numpy().tobytes() == _records_numpy(xyz[:10], 0, 1).tobytes()
    empty = plugin.pack_scan_tensor(torch.empty((0, 3)), torch.empty(0, dtype=torch.int64), torch.empty(0, dtype=torch.int64))
    assert tuple(empty.shape) == (0, 4)


@pytest.mark.parametrize("which,value", [("lidar", -1), ("lidar", 65536), ("table_idx", -1), ("table_idx", 1 << 20)])
def test_pack_scan_tensor_rejects_out_of_range_ids(which, value):
    n = 100
    ids = {"lidar": torch.zeros(n, dtype=torch.int64), "table_idx": torch.zeros(n, dtype=torch.int64)}
    ids[which][57] = value
    with pytest.raises(ValueError) as e:
        plugin.pack_scan_tensor(torch.zeros((n, 3)), ids["lidar"], ids["table_idx"])
    assert which in str(e.value)


@pytest.mark.parametrize("bad", ["xyz_float64", "xyz_shape", "float_ids", "short_ids", "numpy_ids"])
def test_pack_scan_tensor_rejects_bad_tensors(bad):
    n = 8
    xyz, lid, tid = torch.zeros((n, 3)), torch.zeros(n, dtype=torch.int64), torch.zeros(n, dtype=torch.int64)
    if bad == "xyz_float64":
        xyz = xyz.double()
    elif bad == "xyz_shape":
        xyz = torch.zeros((n, 4))
    elif bad == "float_ids":
        lid = lid.float()
    elif bad == "short_ids":
        tid = tid[:5]
    else:
        lid = lid.numpy()
    with pytest.raises(ValueError):
        plugin.pack_scan_tensor(xyz, lid, tid)
