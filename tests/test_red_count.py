"""Reduction counts of the hash-grid scatters on the benchmark's rays (host only): scripts/red_count.py counts what the kernels
issue with vertex runs, one update per distinct grid vertex of a warp, beside the per-lane and cell-run counts.
(bench.py::red_counts models the former cell-run path, L4D_STATIC_VERTEX_RUNS=0.)"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_vertex_run_counts_on_the_benchmark_rays():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "red_count.py")], capture_output=True, text=True,
                         timeout=600, check=True).stdout
    totals = [ln.split()[1:] for ln in out.splitlines() if ln.strip().startswith("total")]
    assert [float(t) for t in totals[0]] == [128.0, 112.2, 97.4]          # static: per-lane, cell-run, vertex-run
    assert "former path (cell runs up to res 1200): 113.4" in out
    d = [float(t) for t in totals[1]]
    assert d[0] == 192.0 and d[2] < 131.0                                 # dynamic: 3 planes x 16 levels x 4 corners -> 129.8


def test_vertex_counts_of_a_still_ray():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import red_count
    cell = np.full((2, 64, 3), 5, np.int64)
    assert red_count.warp_counts(cell) == (8.0, 8.0 / 32, 8.0 / 32)
    step = np.zeros((1, 32, 2), np.int64)
    step[0, :, 0] = np.arange(32)                                    # one cell per sample along x: 33 x 2 vertices per warp
    assert red_count.warp_counts(step) == (4.0, 4.0, 66.0 / 32)
