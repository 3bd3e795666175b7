"""GPU: k_bwd_encoders, the backward's scatter launch whose CTAs share two work queues - the encoder blocks (planes, time
rows, dynamic hash, dL/dflow) and the static-hash (level, block) pairs - and drain the other queue when their own is empty.

Every case runs the same backward twice in a row, and each run is held entry by entry to the float64 scatter of its own
inputs (tests/test_gpu_scatter_exact.py, tests/scatter_ref.py).  The second run starts from work-ticket counters the
first left behind, so it fails unless the last CTA of every launch zeroed them; a launch whose CTAs did not drain both
queues leaves blocks without gradients, which the bound catches.  Sizes:
  - fewer samples than one CTA (one ray of 45 samples), L = 3;
  - few samples at L = 16 (3 rays x 768): the encoder queue empties long before the 16 levels of the static hash;
  - many samples at L = 3 (more rays than the grid has threads): the static queue empties long before the encoder one;
in both MLP modes, and launches of several frames against their rows launched one by one."""
import numpy as np
import pytest
import torch

from parity_util import cuda_model_from_oracle, test_rays as _rays
from test_gpu_scatter_exact import MODES, assert_scatter_exact, full_model, n_wrap, small_oracle
from test_gpu_multiframe import TIMES, check_multi_vs_rows, work_is_zero
from test_gpu_launch_scale import model_for, rays_for
from test_gpu_launch_scale import small_oracle as small_oracle_seeded

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def twice(m, ro, rd, t, S, mode, monkeypatch, what):
    for k in range(2):
        assert_scatter_exact(m, ro, rd, t, S, mode, monkeypatch, f"{what} run {k}")
        assert work_is_zero(m), f"{what} run {k}: work buffer not zero after the backward"


@pytest.mark.parametrize("mode", MODES)
def test_launch_smaller_than_one_cta(dev, monkeypatch, mode):
    m = cuda_model_from_oracle(small_oracle(3, n_levels_hash=3)).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 3
    ro, rd = _rays(1, 1)
    twice(m, torch.from_numpy(ro), torch.from_numpy(rd), 0.4, 45, mode, monkeypatch, f"1 ray S45 L3 {mode}")


@pytest.mark.parametrize("mode", MODES)
def test_encoder_queue_empties_first(dev, monkeypatch, mode):
    from lidar4d_b200.rays import synthetic_sweep
    ro, rd, _ = synthetic_sweep(25)
    sel = np.linspace(0, ro.shape[0] - 1, 3).astype(np.int64)
    m = full_model(mode)
    twice(m, torch.from_numpy(ro[sel]).contiguous(), torch.from_numpy(rd[sel]).contiguous(), 0.5, 768, mode, monkeypatch,
          f"3 rays S768 L16 {mode}")


@pytest.mark.parametrize("mode", MODES)
def test_static_queue_empties_first(dev, monkeypatch, mode):
    m = cuda_model_from_oracle(small_oracle(5, n_levels_hash=3)).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 5
    ro, rd = rays_for(n_wrap())
    twice(m, ro, rd, 0.62, 333, mode, monkeypatch, f"{n_wrap()} rays S333 L3 {mode}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("rays_per_row", [1, 97])
def test_several_frames(dev, mode, rays_per_row):
    """One launch over rows of several frames against the rows launched one by one (their gradients summed), twice."""
    B, S, seed = len(TIMES), 200, 7
    m = model_for(small_oracle_seeded(seed), mode, "split", seed)
    ro, rd = rays_for(B * rays_per_row)
    for k in range(2):
        check_multi_vs_rows(m, ro, rd, TIMES, S, dev, "split", f"{B} frames x {rays_per_row} rays {mode} run {k}", seed=11 + k)
