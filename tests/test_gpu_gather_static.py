"""GPU: the split forward gathers the static hash level-major (k_fwd_gather's second phase): level pairs, plus a
single-level pass when the level count is odd.  Checked against the oracle at even and odd level counts through both
feature sinks (fp16 operand tiles for the tensor-core dense kernels, fp32 SoA planes for the FMA kernels)."""
import pytest
import torch

from oracle import lidar4d_oracle as O
from parity_util import small_config, rel_err, cuda_model_from_oracle, test_rays as _rays

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.mark.parametrize("fp16", [True, False])
@pytest.mark.parametrize("levels", [3, 4, 5])
def test_split_forward_at_odd_and_even_level_counts(dev, levels, fp16):
    orc = O.build_seeded(small_config(n_levels_hash=levels), 7, flow_last_std=0.02)
    if fp16:
        orc.mlp_dtype = "fp16"
    m = cuda_model_from_oracle(orc).set_mlp_fp16(fp16)
    m.pipeline = "split"
    ro, rd = _rays(3, 8)
    S, t = 200, 0.4
    ref = orc.render(torch.from_numpy(ro), torch.from_numpy(rd), t, num_steps=S, perturb=True, seed=0)
    with torch.no_grad():
        out = m.render(torch.from_numpy(ro)[None].to(dev), torch.from_numpy(rd)[None].to(dev), torch.tensor([[t]]),
                       staged=False, num_steps=S, perturb=True)
    for k in ("depth_lidar", "image_lidar", "weights_sum_lidar"):
        assert rel_err(out[k], ref[k]) < TOL, k

