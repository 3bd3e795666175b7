"""GPU: the backward scatter kernels sum hash-grid gradients per distinct grid vertex within a warp (l4d_vertex_sum) before
they reduce to L2.  Warps straddle two rays when S is not a multiple of 32, and the last warp of a launch is partial when the
sample count is not; both must break the vertex runs.  The static and dynamic hash gradients of the split backward are
checked against the oracle at such shapes, in both MLP modes."""
import pytest
import torch

from oracle import lidar4d_oracle as O
from parity_util import small_config, rel_err, relu_margin, cuda_model_from_oracle, test_rays as _rays

pytestmark = pytest.mark.gpu
TOL = 1e-4
MIN_RELU_MARGIN = 1e-8      # as tests/test_gpu_parity.py


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("S,n_rays", [(45, 24), (200, 23), (333, 7)])
def test_split_backward_hash_gradients_at_straddling_and_partial_warps(dev, S, n_rays, fp16):
    assert S % 32 and (S * n_rays) % 32
    orc = O.build_seeded(small_config(), 3, flow_last_std=0.02)
    if fp16:
        orc.mlp_dtype = "fp16"
    m = cuda_model_from_oracle(orc).set_mlp_fp16(fp16)
    m.pipeline = "split"
    m.jitter_seed = 3
    ro, rd = _rays(3, 8)
    ro, rd = ro[:n_rays], rd[:n_rays]
    t = 0.4
    ref = orc.render(torch.from_numpy(ro), torch.from_numpy(rd), t, num_steps=S, perturb=True, seed=3, return_stages=True)
    assert relu_margin(orc, ref) > MIN_RELU_MARGIN
    out = m.render(torch.from_numpy(ro)[None].to(dev), torch.from_numpy(rd)[None].to(dev), torch.tensor([[t]]),
                   staged=False, num_steps=S, perturb=True)
    g = torch.Generator().manual_seed(1)
    gd, gi = torch.randn(n_rays, generator=g), torch.randn(n_rays, 2, generator=g)
    (ref["depth_lidar"] * gd).sum().add((ref["image_lidar"] * gi).sum()).backward()
    ((out["depth_lidar"][0] * gd.to(dev)).sum() + (out["image_lidar"][0] * gi.to(dev)).sum()).backward()
    og = orc.ref_named_grads()
    got = {k: p.grad for k, p in m.named_parameters()}
    keys = [k for k in og if k.startswith("hash_encoder.") and og[k].numel()]
    assert any("hash_static" in k for k in keys) and any("hash_dynamic" in k for k in keys)
    errs = {k: rel_err(got[k], og[k]) for k in keys}
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, f"worst {max(errs.values()):.2e}; failing: {bad}"
