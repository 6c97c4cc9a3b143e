"""examples/replay_city.cpp — the call sequence INTEGRATION.md describes (readers, undistortion, voxel grid, pose table, merged
scan, iterated update, map deltas) as one C++ program against the header, the library and the REAL reference tree type.
build() compiles and links it into oracle/_ref/ (oracle/Makefile, the reference's ikd_Tree.h/.cpp resolved through the
oracle's PCL shim).  Here its host-only part must run, and without a GPU the full program must fail loudly at malio_create;
tests/test_gpu_more.py runs the full program on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "replay_city")


@pytest.mark.skipif(not os.path.exists(EXE), reason="oracle/_ref/replay_city not built (needs the reference's ikd_Tree.cpp)")
def test_cpp_example_compiles_links_and_its_host_side_runs():
    r = subprocess.run([EXE, "--host-only"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-500:])
    line = [l for l in r.stdout.splitlines() if l.startswith("host-only:")][0]
    assert "table entries 4 (offsets 0 2 4)" in line and "spline ok 1 p.x 0.350000" in line and "outside 0" in line
    import torch
    if not torch.cuda.is_available():
        r = subprocess.run([EXE], capture_output=True, text=True, timeout=120)
        assert r.returncode == 1 and "malio_create:" in r.stderr      # no silent CPU fallback
