"""GPU: k_bwd_composite, the compositing backward of the tensor-core pipeline, sample by sample against a float64
evaluation of its own inputs (tests/compositing_ref.py).

The kernel leaves {dL/dσ, dL/da0, dL/da1, attribute mask} of every sample in feature columns 0..3 of the saved
dL/dfeature, where k_bwd_dense_tc reads them before it overwrites them.  l4d_composite_backward runs it alone on the
saved buffer of a training forward, and the four columns are held to:

    dL/dσ:       CR.dsigma_bound + 2^-149   (where dL/dσ is subnormal, its last two products round by up to half a
                                            subnormal ulp each, an absolute error the relative bound does not carry)
    dL/da_h:     |got - ŵ g_h m| <= |g_h| weight_bound + 2^-24 |ŵ g_h|      (m = the kernel's mask)
    mask:        equal to ŵ > 1e-4 wherever ŵ is farther than its bound from 1e-4

Cases: one-ray launches, partial last tiles (S = 129, 333) and launches whose persistent grid wraps
(N = 2·16·SMs + 37 rays), in the default and the surface-like density regime (α == 1, T underflowing)."""
import ctypes as C

import numpy as np
import pytest
import torch

import compositing_ref as CR
import scatter_ref as SR
from lidar4d_b200 import _capi
from lidar4d_b200.model import _RenderFn
from oracle import lidar4d_oracle as O
from parity_util import small_config, make_surface_like, cuda_model_from_oracle, test_rays as _rays

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def n_wrap() -> int:
    return 2 * 16 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def model_for(surface: bool):
    orc = O.build_seeded(small_config(), 3, flow_last_std=0.02)
    O.snap_mlp_weights_fp16(orc)
    if surface:
        make_surface_like(orc)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(True)
    m.pipeline = "split"
    m.jitter_seed = 3
    return m


def composite_columns(m, N, S, U, dev, monkeypatch):
    """Training forward + backward; returns (outputs, saved copy taken before the backward, dL/dfeature columns 0..3
    [P, 4] written by k_bwd_composite alone on that copy)."""
    H = 32
    ro, rd = _rays(H, (N + H - 1) // H)
    ro, rd = torch.from_numpy(ro[:N]).contiguous(), torch.from_numpy(rd[:N]).contiguous()
    captured = {}
    orig = _RenderFn.backward

    def keep(ctx, *g):
        captured["saved"] = ctx.saved.clone()
        captured["rays"] = ctx.rays_args
        captured["g"] = g
        captured["want_weights"] = ctx.want_weights
        return orig(ctx, *g)
    monkeypatch.setattr(_RenderFn, "backward", staticmethod(keep))
    m.zero_grad(set_to_none=False)
    m._jitter_calls = 0
    out = m.render(ro[None].to(dev), rd[None].to(dev), torch.tensor([[0.4]]), num_steps=S, perturb=True)
    outs = {"depth_lidar": out["depth_lidar"][0], "image_lidar": out["image_lidar"][0],
            "weights_sum_lidar": out["weights_sum_lidar"], "weights": out["weights"]}
    torch.autograd.backward([outs[k] for k in U], [U[k] for k in U])
    torch.cuda.synchronize()
    monkeypatch.undo()

    saved = captured["saved"]
    n, s, perturb, seed, ray_offset = captured["rays"]
    assert (n, s) == (N, S)
    g_depth, g_image, g_wsum, *rest = captured["g"]
    z = lambda t, shape: torch.zeros(shape, device=dev) if t is None else t.contiguous().float()
    g_depth, g_image = z(g_depth, (N,)), z(g_image, (N, 2))
    g_wsum = None if g_wsum is None else g_wsum.contiguous().float()
    g_weights = rest[0].contiguous().float() if (captured["want_weights"] and rest and rest[0] is not None) else None
    ro_d, rd_d = ro.to(dev), rd.to(dev)
    rays = _capi.L4DRays()
    rays.rays_o, rays.rays_d = ro_d.data_ptr(), rd_d.data_ptr()
    rays.n_rays, rays.n_steps, rays.perturb, rays.seed, rays.ray_offset = N, S, perturb, seed, ray_offset
    eng = m._engine
    lib = eng._lib()
    with torch.cuda.device(dev):
        rc = lib.l4d_composite_backward(C.byref(eng.ccfg), C.byref(rays),
                                        saved.data_ptr(), saved.numel(), g_depth.data_ptr(), g_image.data_ptr(),
                                        g_wsum.data_ptr() if g_wsum is not None else None,
                                        g_weights.data_ptr() if g_weights is not None else None,
                                        torch.cuda.current_stream().cuda_stream)
    _capi.check(lib, rc, "l4d_composite_backward")
    torch.cuda.synchronize()
    cols = SR.decode_saved(m.cfg, saved, N, S)["dfeat"][:, :4]
    return {k: v.detach() for k, v in out.items()}, saved, cols


def upstream(N: int, S: int, dev):
    g = torch.Generator().manual_seed(17)
    U = {"depth_lidar": torch.randn(N, generator=g), "image_lidar": torch.randn(N, 2, generator=g),
         "weights_sum_lidar": torch.randn(N, generator=g), "weights": torch.randn(N, S, generator=g) * 0.01}
    return {k: v.to(dev) for k, v in U.items()}


CASES = [(1, 129, False), (1, 333, True), (8, 129, True), (8, 333, False), ("wrap", 129, False), ("wrap", 333, True)]


@pytest.mark.parametrize("N,S,surface", CASES, ids=[f"N{n}-S{s}-{'surface' if f else 'default'}" for n, s, f in CASES])
def test_composite_against_own_inputs(dev, monkeypatch, N, S, surface):
    N = n_wrap() if N == "wrap" else N
    m = model_for(surface)
    cfg = m.cfg
    U = upstream(N, S, dev)
    out, saved, cols = composite_columns(m, N, S, U, dev, monkeypatch)
    L = SR.saved_layout(cfg, N, S)
    sigma = saved[L["sigma"]:L["sigma"] + 4 * N * S].view(torch.float32).view(N, S)
    attr = saved[L["attr"]:L["attr"] + 8 * N * S].view(torch.float32).view(2, N, S).double()
    sd = float(np.float32((np.float32(cfg.far_lidar) - np.float32(cfg.near_lidar)) / np.float32(S)))
    ref = CR.composite(sigma, attr, out["z_vals"], sd, cfg.density_scale, cfg.active_sensor, U)
    what = f"N={N} S={S} {'surface' if surface else 'default'}"
    got = cols.double().view(N, S, 4)

    err = (got[..., 0] - ref["dsigma"]).abs()
    r = err / (CR.dsigma_bound(ref) + 2.0 ** -149)
    worst = int(torch.argmax(r))
    assert float(r.reshape(-1)[worst]) <= 1.0, (what, "dL/dσ", worst, float(got[..., 0].reshape(-1)[worst]),
                                                float(ref["dsigma"].reshape(-1)[worst]), int((r > 1).sum()))

    wb = CR.weight_bound(ref)
    clear = (ref["weights"] - CR.MASK_THRESHOLD).abs() > wb
    mask = got[..., 3]
    assert bool(((mask == 0) | (mask == 1)).all()), what
    assert int(((mask != 0) != ref["mask"])[clear].sum()) == 0, (what, "mask")
    gi = U["image_lidar"].double().reshape(N, 2)
    for h in range(2):
        exact = ref["weights"] * gi[:, h, None] * (mask != 0)          # the kernel's own mask decides near 1e-4
        bound = gi[:, h, None].abs() * wb + CR.EPS32 * exact.abs()
        assert bool(((got[..., 1 + h] - exact).abs() <= bound).all()), (what, f"dL/da{h}")
        assert bool((got[..., 1 + h][mask == 0] == 0).all()), (what, f"dL/da{h} outside the mask")
    n_masked = int((mask != 0).sum())
    if not surface:
        assert n_masked > 0, (what, "no sample in the attribute mask")
    print(f"[composite] {what}: dL/dσ {float(r.max()):.3f} of its bound, {n_masked} of {N * S} samples in the mask")
