"""The device-memory entry points without a GPU: their ctypes signatures against the header, NULL handles and NULL arguments
answered with an error code (in a subprocess: a missing check would be a segmentation fault), and the torch wrappers'
argument checks, which run before anything reaches the library."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import pytest
import torch

from malio_b200 import capi, plugin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("malio_knn_device", "malio_map_build_device", "malio_map_add_points_device")


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


def test_null_handle_and_null_arguments_return_an_error():
    code = textwrap.dedent("""
        from malio_b200 import capi
        lib = capi.load()
        for n in (0, 5):
            print("knn", n, lib.malio_knn_device(None, None, n, None, None, None), flush=True)
            print("build", n, lib.malio_map_build_device(None, None, None, None, n, None), flush=True)
            print("add", n, lib.malio_map_add_points_device(None, None, None, None, n, None), flush=True)
        print("DONE")
    """)
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "ma-lio_b200"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout[-400:], r.stderr[-400:])
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "DONE" and len(lines) == 7
    for l in lines[:-1]:
        assert l.split()[2] == str(capi.ERR_INVALID_ARG), l


class _Lib:
    """Stands in for the library: any call reaching it fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called")


def _model():
    m = object.__new__(plugin.MeasurementModel)   # no handle (no GPU here): only the Python-side checks can run
    m.lib, m._h, m.device = _Lib(), C.c_void_p(), 0
    return m


@pytest.mark.parametrize("bad", ["cpu", "float64", "int32", "shape", "rank", "non_contiguous", "numpy"])
def test_torch_wrappers_reject_before_the_call(bad):
    q = {"cpu": torch.zeros((8, 3)), "float64": torch.zeros((8, 3), dtype=torch.float64),
         "int32": torch.zeros((8, 3), dtype=torch.int32), "shape": torch.zeros((8, 4)), "rank": torch.zeros(24),
         "non_contiguous": torch.zeros((8, 6))[:, ::2], "numpy": torch.zeros((8, 3)).numpy()}[bad]
    m = _model()
    with pytest.raises(ValueError) as e:
        m.knn_tensor(q)
    if bad == "non_contiguous":
        assert "contiguous" in str(e.value)
    for fn in (m.map_build_tensor, m.map_add_points_tensor):
        with pytest.raises(ValueError):
            fn(q, torch.zeros(8))
