"""The front half of a scan on device memory (malio_undistort_device, malio_voxel_grid_device, malio_scan_uncertainty_resident,
malio_upload_scan_resident) without a GPU: the ctypes signatures against the header, NULL handles answered with an error code
(in a subprocess: a missing check would be a segmentation fault), and the tensor wrappers' argument checks, which run before
anything reaches the library."""
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
NEW = ("malio_undistort_device", "malio_voxel_grid_device", "malio_scan_uncertainty_resident", "malio_upload_scan_resident")
SCALARS = (("uint32_t", C.c_uint32), ("float", C.c_float), ("double", C.c_double), ("int", C.c_int))


def _header_args(name):
    hdr = open(os.path.join(ROOT, "include", "malio_b200.h")).read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    out = []
    for a in (re.sub(r"/\*.*?\*/", "", a).strip() for a in m.group(1).split(",")):
        if "*" in a:
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


def test_header_signatures_carry_their_scalars():
    # the parser above must see the int, the count and the float, not only pointers
    assert _header_args("malio_undistort_device")[1:4] == [C.c_int, C.c_void_p, C.c_uint32]
    assert _header_args("malio_voxel_grid_device")[3:5] == [C.c_uint32, C.c_float]
    assert len(_header_args("malio_undistort_device")) == 12 and len(_header_args("malio_voxel_grid_device")) == 9


def test_null_handle_returns_an_error():
    code = textwrap.dedent("""
        import ctypes as C
        from malio_b200 import capi
        lib = capi.load()
        a, s, k = capi.UndistortArgs(), capi.ScanUncArgs(), C.c_uint32(0)
        for n in (0, 5):
            print("undistort", n, lib.malio_undistort_device(None, 0, None, n, None, None, None, None, None, None, None, None), flush=True)
            print("undistort-args", n, lib.malio_undistort_device(None, 0, None, n, C.addressof(a), None, None, None, None, None, C.addressof(k), None), flush=True)
            print("voxel", n, lib.malio_voxel_grid_device(None, 0, None, n, 0.5, None, n, None, None), flush=True)
            print("voxel-count", n, lib.malio_voxel_grid_device(None, 0, None, n, 0.5, None, 0, C.addressof(k), None), flush=True)
        print("unc", lib.malio_scan_uncertainty_resident(None, None, None, None), flush=True)
        print("unc-args", lib.malio_scan_uncertainty_resident(None, C.addressof(s), None, None), flush=True)
        print("upload", lib.malio_upload_scan_resident(None, None), flush=True)
        print("upload-count", lib.malio_upload_scan_resident(None, C.addressof(k)), flush=True)
        print("DONE")
    """)
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "ma-lio_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "DONE" and len(lines) == 13
    for l in lines[:-1]:
        assert l.split()[-1] == str(capi.ERR_INVALID_ARG), l


class _Lib:
    """Stands in for the library: any call reaching it fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _model():
    m = object.__new__(plugin.MeasurementModel)   # no handle (no GPU here): only the Python-side checks can run
    m.lib, m._h, m.device, m.n_lidar, m.n_points, m._slot_rows = _Lib(), C.c_void_p(), 0, 1, 0, {}
    return m


def _bad(cols, which):
    return {"cpu": torch.zeros((8, cols)), "float64": torch.zeros((8, cols), dtype=torch.float64),
            "int32": torch.zeros((8, cols), dtype=torch.int32), "shape": torch.zeros((8, cols + 1)),
            "rank": torch.zeros(8 * cols), "non_contiguous": torch.zeros((8, 2 * cols))[:, ::2],
            "numpy": np.zeros((8, cols), np.float32)}[which]


BAD = ["cpu", "float64", "int32", "shape", "rank", "non_contiguous", "numpy"]
Q0 = (np.array([1.0, 0, 0, 0]), np.zeros(3))


@pytest.mark.parametrize("bad", BAD)
def test_undistort_tensor_rejects_before_the_call(bad):
    with pytest.raises(ValueError) as e:
        _model().undistort_tensor(0, _bad(4, bad), 0.0, Q0, Q0, np.arange(4.0), np.tile(np.eye(4).ravel(), (4, 1)), np.zeros(0), -1)
    if bad == "non_contiguous":
        assert "contiguous" in str(e.value)


def test_undistort_tensor_rejects_an_unknown_output(monkeypatch):
    monkeypatch.setattr(plugin, "_check_tensor", lambda *a, **k: None)   # no CUDA tensor can be made here: let a CPU one pass
    with pytest.raises(ValueError) as e:
        _model().undistort_tensor(0, torch.zeros((8, 4)), 0.0, Q0, Q0, np.arange(4.0), np.tile(np.eye(4).ravel(), (4, 1)), np.zeros(0), -1,
                                  want=("cloud", "xyz"))
    assert "xyz" in str(e.value)


@pytest.mark.parametrize("bad", BAD)
def test_voxel_grid_tensor_rejects_before_the_call(bad):
    with pytest.raises(ValueError) as e:
        _model().voxel_grid_tensor(0, _bad(5, bad), 0.5)
    if bad == "non_contiguous":
        assert "contiguous" in str(e.value)
