"""bench.py contract pieces that can be checked without a GPU: the reference arm (CPU oracle port) prints the
required JSON line on rank 0 and stays silent on the other ranks; the GPU arm refuses to run without CUDA."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(extra_env, *args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", **extra_env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                          timeout=600, env=env)


def test_reference_arm_prints_the_contract_line_on_rank0_only():
    args = ("--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0", "--cpu-rays", "2", "--levels", "2")
    r0 = _run({"RANK": "0", "WORLD_SIZE": "2"}, *args)
    assert r0.returncode == 0, r0.stderr[-400:]
    line = json.loads([ln for ln in r0.stdout.splitlines() if ln.startswith("{")][-1])
    assert line["impl"] == "reference" and line["unit"] == "rays/s" and line["higher_is_better"] is True
    assert line["n_gpus"] == 2 and line["steps"] == 1 and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["value"] == line["value"]
    assert line["e2e"] == {"value": line["value"], "unit": "rays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert line["metric"].startswith("training rays/sec") and "workload" in line["config"]
    r1 = _run({"RANK": "1", "WORLD_SIZE": "2"}, *args)
    assert r1.returncode == 0 and not [ln for ln in r1.stdout.splitlines() if ln.startswith("{")]


def test_gpu_arm_fails_loudly_without_cuda():
    r = _run({"RANK": "0", "WORLD_SIZE": "1"}, "--steps", "1", "--warmup", "1", "--no-cpu-baseline")
    assert r.returncode != 0
    assert "needs a GPU" in (r.stderr + r.stdout)


def test_executed_red_count_of_the_static_scatter():
    """bench.py's RED-rate binding of k_bwd_scatter_static uses the reductions the kernel EXECUTES: 8 per level, and at the
    warp-aggregated levels 8 per run of consecutive samples that share a cell (host-side run statistics of the rays)."""
    sys.path.insert(0, ROOT)
    import numpy as np
    import bench
    from lidar4d_b200.geometry import FieldConfig
    from lidar4d_b200.rays import synthetic_sweep
    cfg = FieldConfig(**bench.model_kwargs(16))
    assert bench.red_counts(cfg)["k_bwd_scatter_static"] == 128.0
    ro, rd, _ = synthetic_sweep(7)
    r = bench.red_counts(cfg, (ro, rd))
    agg = int((cfg.static_grid().resolution <= bench.STATIC_AGG_RES).sum())
    assert agg == 4 and r["k_bwd_scatter_static_algorithmic"] == 128.0
    assert 128.0 - 8.0 * agg < r["k_bwd_scatter_static"] < 128.0          # runs exist, and no level disappears
    # a ray that stays inside one cell for a whole warp issues 8 reductions per 32 samples at an aggregated level
    still = (np.zeros((4, 3), np.float32), np.zeros((4, 3), np.float32))
    assert abs(bench.red_counts(cfg, still)["k_bwd_scatter_static"] - (128.0 - 8.0 * agg * (1 - 1 / 32))) < 1e-6
    # the macro the count mirrors
    src = open(os.path.join(ROOT, "lidar4d_b200", "csrc", "l4d_split.cuh")).read()
    assert f"#define L4D_STATIC_AGG_RES {bench.STATIC_AGG_RES}" in src
