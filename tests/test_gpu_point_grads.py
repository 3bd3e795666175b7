"""GPU: LiDAR4D.density / .attribute are differentiable (csrc/l4d_points.cuh).  Gradients against oracle autograd in both
grad modes, the forward bits of the grad-mode calls, a pure-PyTorch restatement of LiDAR_Renderer.run built on the two
methods against model.render, the full-size configuration, linearity, shapes and the stale-forward error."""
import numpy as np
import pytest
import torch

from oracle import lidar4d_oracle as O
from lidar4d_b200.geometry import make_frame
from parity_util import (small_config, rel_err, relu_margin, cuda_model_from_oracle, grad_errors, full_oracle,
                         test_rays as _rays)
from test_point_grads_hostsim import attr_margin, density_case, MIN_RELU_MARGIN, TIMES

pytestmark = pytest.mark.gpu
TOL = 1e-4
HEADS = ("intensity_net.params", "raydrop_net.params")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _tt(t):
    return torch.tensor([[float(t)]])


def model_grads(m, loss_fn, grad_mode):
    """gradients of loss_fn(m) w.r.t. every parameter: through .grad (arena) or torch.autograd.grad (autograd)"""
    m.grad_mode = grad_mode
    m.zero_grad(set_to_none=True)
    loss = loss_fn(m)
    names, params = zip(*m.named_parameters())
    if grad_mode == "arena":
        loss.backward()
        return {k: (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)) for k, p in zip(names, params)}
    gs = torch.autograd.grad(loss, params, allow_unused=True)
    return {k: (g.detach().clone() if g is not None else torch.zeros_like(p)) for k, p, g in zip(names, params, gs)}


def assert_grads(got, og, tol=TOL):
    errs = {k: rel_err(got[k], og[k]) for k in og if og[k].numel()}
    bad = {k: v for k, v in errs.items() if not v < tol}
    assert not bad, f"worst {max(errs.values()):.2e}; failing: {bad}"


# ---- 1. against the oracle -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("grad_mode", ["arena", "autograd"])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("t", TIMES)
def test_density_grads_against_oracle(dev, t, fp16, grad_mode):
    orc = density_case(21, fp16)
    m = cuda_model_from_oracle(orc)
    g = torch.Generator().manual_seed(4)
    n = 300
    x = torch.rand(n, 3, generator=g) * 2 - 1
    g_s, g_g = torch.randn(n, generator=g), torch.randn(n, 15, generator=g)
    ref = orc.density(x, make_frame(t, orc.cfg.num_frames, orc.cfg.time_resolution), return_features=True)
    assert relu_margin(orc, ref) > MIN_RELU_MARGIN
    ((ref["sigma"] * g_s).sum() + (ref["geo_feat"] * g_g).sum()).backward()
    og = orc.ref_named_grads()
    xd, gsd, ggd = x.to(dev), g_s.to(dev), g_g.to(dev)

    def loss(mm):
        out = mm.density(xd, _tt(t))
        assert out["sigma"].requires_grad and out["geo_feat"].requires_grad
        assert rel_err(out["sigma"], ref["sigma"]) < TOL and rel_err(out["geo_feat"], ref["geo_feat"]) < TOL
        return (out["sigma"] * gsd).sum() + (out["geo_feat"] * ggd).sum()
    got = model_grads(m, loss, grad_mode)
    assert_grads(got, og)


@pytest.mark.parametrize("grad_mode", ["arena", "autograd"])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("mask_kind", ["none", "partial", "empty"])
def test_attribute_grads_against_oracle(dev, mask_kind, fp16, grad_mode):
    orc = O.build_seeded(small_config(), 14)
    if fp16:
        orc.mlp_dtype = "fp16"
    m = cuda_model_from_oracle(orc)
    g = torch.Generator().manual_seed(2)
    n = 301
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    geo = torch.randn(n, 15, generator=g)
    mask = {"none": None, "partial": torch.rand(n, generator=g) > 0.4, "empty": torch.zeros(n, dtype=torch.bool)}[mask_kind]
    g_out = torch.randn(n, 2, generator=g)
    assert attr_margin(orc, d, geo, mask) > MIN_RELU_MARGIN
    geo_t = geo.clone().requires_grad_(True)
    ref = orc.attribute(d, geo_t, mask)
    if mask_kind != "empty":
        (ref * g_out.to(ref.dtype)).sum().backward()
    og = {k: v for k, v in orc.ref_named_grads().items() if k in HEADS}
    ref_geo = geo_t.grad if geo_t.grad is not None else torch.zeros(n, 15)
    dd, md, god = d.to(dev), (None if mask is None else mask.to(dev)), g_out.to(dev)
    geo_d = geo.to(dev).requires_grad_(True)
    m.grad_mode = grad_mode
    m.zero_grad(set_to_none=True)
    m._engine.ensure_staged()                      # stage now: the launch count below covers the attribute call alone
    l0 = m.gpu_launches
    out = m.attribute(None, dd, md, geo_d)
    assert out.shape == (n, 2) and out.requires_grad
    assert float((out.detach().cpu() - ref.detach()).abs().max()) < 1e-5
    l = (out * god).sum()
    heads = [dict(m.named_parameters())[k] for k in HEADS]
    if grad_mode == "arena":
        l.backward()
        got = {k: p.grad for k, p in zip(HEADS, heads)}
        got_geo = geo_d.grad
    else:
        gs = torch.autograd.grad(l, heads + [geo_d], allow_unused=True)
        got = dict(zip(HEADS, gs[:2]))
        got_geo = gs[2]
    if mask_kind == "empty":
        assert m.gpu_launches == l0                 # neither the forward nor the backward launched a kernel
        assert got_geo is not None and float(got_geo.abs().max()) == 0.0
        assert all(v is None or float(v.abs().max()) == 0.0 for v in got.values())
        return
    assert rel_err(got_geo, ref_geo) < TOL
    if mask is not None:
        assert float(got_geo.cpu()[~mask].abs().max()) == 0.0
    for k in HEADS:
        assert rel_err(got[k], og[k]) < TOL, k


def test_attribute_one_input_requiring_grad(dev):
    """geo_feat alone (heads frozen) and the heads alone (geo_feat a plain tensor)."""
    orc = O.build_seeded(small_config(), 14)
    m = cuda_model_from_oracle(orc)
    g = torch.Generator().manual_seed(3)
    n = 200
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(dev)
    geo = torch.randn(n, 15, generator=g).to(dev)
    both_geo = geo.clone().requires_grad_(True)
    m.attribute(None, d, None, both_geo).sum().backward()
    ref_heads = {k: dict(m.named_parameters())[k].grad.clone() for k in HEADS}
    for p in m.parameters():
        p.requires_grad_(False)
    only_geo = geo.clone().requires_grad_(True)
    m.attribute(None, d, None, only_geo).sum().backward()
    assert torch.allclose(only_geo.grad, both_geo.grad, rtol=0, atol=1e-6 * float(both_geo.grad.abs().max()))
    for k in HEADS:
        dict(m.named_parameters())[k].requires_grad_(True)
        dict(m.named_parameters())[k].grad = None
    m.attribute(None, d, None, geo).sum().backward()
    for k in HEADS:
        assert rel_err(dict(m.named_parameters())[k].grad, ref_heads[k]) < 1e-5, k


# ---- 2. the grad-mode forward is the no-grad forward, bit for bit -----------------------------------------------------
@pytest.mark.parametrize("fp16", [False, True])
def test_forward_bits_match_inference(dev, fp16):
    orc = density_case(21, fp16)
    m = cuda_model_from_oracle(orc)
    x = (torch.rand(1000, 3, generator=torch.Generator().manual_seed(0)) * 2 - 1).to(dev)
    for t in TIMES:
        a = m.density(x, _tt(t), return_features=True)
        assert a["sigma"].requires_grad and not a["features"].requires_grad and not a["flow"].requires_grad
        with torch.no_grad():
            b = m.density(x, _tt(t), return_features=True)
        for k in ("sigma", "geo_feat", "features", "flow"):
            assert torch.equal(a[k].detach(), b[k]), (t, k)
    d = torch.nn.functional.normalize(torch.randn(1000, 3, generator=torch.Generator().manual_seed(1)), dim=-1).to(dev)
    mask = (torch.rand(1000, generator=torch.Generator().manual_seed(2)) > 0.3).to(dev)
    ga = m.attribute(None, d, mask, a["geo_feat"])
    with torch.no_grad():
        gb = m.attribute(None, d, mask, a["geo_feat"])
    assert ga.requires_grad and torch.equal(ga.detach(), gb)


# ---- 3. LiDAR_Renderer.run restated on density + attribute reproduces render ------------------------------------------
def restated_run(m, ro, rd, t, z):
    """renderer.py:44-140 in PyTorch on model.density / model.attribute, given the z grid (perturb=False)"""
    N, S = z.shape
    c = m.cfg
    xyz = ro.unsqueeze(-2) + rd.unsqueeze(-2) * z.unsqueeze(-1)
    xyz = torch.min(torch.max(xyz, m.aabb[:3]), m.aabb[3:])
    dens = m.density(xyz.reshape(-1, 3), _tt(t))
    sigma = dens["sigma"].view(N, S)
    near, far = np.float32(c.near_lidar), np.float32(c.far_lidar)
    sample_dist = float(np.float32(np.float32(far - near) / np.float32(S)))
    deltas = torch.cat([z[:, 1:] - z[:, :-1], sample_dist * torch.ones_like(z[:, :1])], -1)
    k = 2.0 if c.active_sensor else 1.0
    alphas = 1 - torch.exp(-k * deltas * c.density_scale * sigma)
    shifted = torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-15], -1)
    weights = alphas * torch.cumprod(shifted, -1)[:, :-1]
    mask = weights > 1e-4
    dirs = rd.view(-1, 1, 3).expand(N, S, 3).reshape(-1, 3)
    attr = m.attribute(None, dirs, mask.reshape(-1), dens["geo_feat"]).view(N, S, -1)
    depth = (weights * z).sum(-1)
    image = (weights.unsqueeze(-1) * attr).sum(-2)
    return depth, image, weights, mask


@pytest.mark.parametrize("t,S,seed", [(0.4, 200, 3), (0.0, 150, 4), (1.0, 130, 5)])
def test_restated_renderer_matches_render(dev, t, S, seed):
    ro_np, rd_np = _rays(3, 8)
    ro, rd = torch.from_numpy(ro_np).to(dev), torch.from_numpy(rd_np).to(dev)
    N = ro.shape[0]
    for s in range(seed, seed + 40):          # a seed whose weights stay clear of the 1e-4 attribute threshold
        orc = O.build_seeded(small_config(), s, flow_last_std=0.02)
        m = cuda_model_from_oracle(orc)
        with torch.no_grad():
            w = m.render(ro[None], rd[None], _tt(t), num_steps=S, perturb=False)["weights"]
        if float((w - 1e-4).abs().min()) >= 5e-7:
            break
    g = torch.Generator().manual_seed(1)
    gd, gi = torch.randn(N, generator=g).to(dev), torch.randn(N, 2, generator=g).to(dev)
    m.zero_grad(set_to_none=True)
    out = m.render(ro[None], rd[None], _tt(t), num_steps=S, perturb=False)
    ((out["depth_lidar"][0] * gd).sum() + (out["image_lidar"][0] * gi).sum()).backward()
    ref = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    m.zero_grad(set_to_none=True)
    depth, image, weights, mask = restated_run(m, ro, rd, t, out["z_vals"].detach())
    ((depth * gd).sum() + (image * gi).sum()).backward()
    got = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert torch.equal(mask, out["weights"].detach() > 1e-4)
    assert rel_err(depth, out["depth_lidar"][0]) < TOL
    assert rel_err(image, out["image_lidar"][0]) < TOL
    assert rel_err(weights, out["weights"]) < TOL
    assert set(got) == set(ref)
    assert_grads(got, ref)


# ---- 4. full size: L = 16 default tables, band-limited -----------------------------------------------------------------
def test_density_grads_full_size(dev):
    orc = full_oracle(16, 31, smooth=True)
    m = cuda_model_from_oracle(orc)
    g = torch.Generator().manual_seed(6)
    n, t = 2048, 0.5
    x = torch.rand(n, 3, generator=g) * 1.8 - 0.9
    g_s, g_g = torch.randn(n, generator=g), torch.randn(n, 15, generator=g)
    ref = orc.density(x, make_frame(t, orc.cfg.num_frames, orc.cfg.time_resolution))
    ((ref["sigma"] * g_s).sum() + (ref["geo_feat"] * g_g).sum()).backward()
    og = orc.ref_named_grads()
    out = m.density(x.to(dev), _tt(t))
    ((out["sigma"] * g_s.to(dev)).sum() + (out["geo_feat"] * g_g.to(dev)).sum()).backward()
    fails = {}
    for k, p in m.named_parameters():
        r = og[k]
        if not r.numel() or k in HEADS:
            continue
        a = p.grad.detach().cpu().double()
        _, norm, frac = grad_errors(a, r)
        if frac > 1e-3 or norm > (5e-3 if k.startswith("flow_net") else 1e-3):
            fails[k] = (norm, frac)
        if "hash" in k or "grid_enc" in k:
            if not torch.equal(a.reshape(-1) != 0, r.reshape(-1) != 0):
                fails[k + " touched"] = int(((a.reshape(-1) != 0) != (r.reshape(-1) != 0)).sum())
    assert not fails, fails


# ---- 5. linearity in the upstream gradient ---------------------------------------------------------------------------
def _density_grads(m, x, t, gs, gg):
    m.zero_grad(set_to_none=True)
    out = m.density(x, _tt(t))
    ((out["sigma"] * gs).sum() + (out["geo_feat"] * gg).sum()).backward()
    return {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}


def _attr_grads(m, d, mask, geo, go):
    m.zero_grad(set_to_none=True)
    geo = geo.clone().requires_grad_(True)
    (m.attribute(None, d, mask, geo) * go).sum().backward()
    out = {k: dict(m.named_parameters())[k].grad.clone() for k in HEADS}
    out["geo"] = geo.grad
    return out


@pytest.mark.parametrize("scale", [65536.0, 2.0 ** -20])
def test_linearity(dev, scale):
    orc = density_case(21, False)
    m = cuda_model_from_oracle(orc)
    g = torch.Generator().manual_seed(8)
    n = 1000
    x = (torch.rand(n, 3, generator=g) * 2 - 1).to(dev)
    gs, gg = torch.randn(n, generator=g).to(dev), torch.randn(n, 15, generator=g).to(dev)
    a = _density_grads(m, x, 0.4, gs, gg)
    b = _density_grads(m, x, 0.4, gs * scale, gg * scale)
    for k in a:
        assert rel_err(b[k] / scale, a[k]) < 2e-5, k
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(dev)
    mask = (torch.rand(n, generator=g) > 0.3).to(dev)
    geo, go = torch.randn(n, 15, generator=g).to(dev), torch.randn(n, 2, generator=g).to(dev)
    a = _attr_grads(m, d, mask, geo, go)
    b = _attr_grads(m, d, mask, geo, go * scale)
    for k in a:
        assert rel_err(b[k] / scale, a[k]) < 2e-5, k


# ---- 6. shapes -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 333])
def test_small_shapes(dev, n):
    orc = density_case(21, False)
    m = cuda_model_from_oracle(orc)
    g = torch.Generator().manual_seed(9)
    x = torch.rand(n, 3, generator=g) * 2 - 1
    gs, gg = torch.randn(n, generator=g), torch.randn(n, 15, generator=g)
    out = m.density(x.to(dev), _tt(0.4), return_features=True)
    assert out["sigma"].shape == (n,) and out["geo_feat"].shape == (n, 15) and out["features"].shape[0] == n
    ((out["sigma"] * gs.to(dev)).sum() + (out["geo_feat"] * gg.to(dev)).sum()).backward()
    got = {k: p.grad for k, p in m.named_parameters()}
    if n == 0:
        assert all(v is None or not v.numel() or float(v.abs().max()) == 0.0 for v in got.values())
    else:
        ref = orc.density(x, make_frame(0.4, orc.cfg.num_frames, orc.cfg.time_resolution))
        ((ref["sigma"] * gs).sum() + (ref["geo_feat"] * gg).sum()).backward()
        og = orc.ref_named_grads()
        assert_grads({k: (v if v is not None else torch.zeros_like(og[k])) for k, v in got.items()}, og)
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(dev)
    geo = torch.randn(n, 15, generator=g).to(dev).requires_grad_(True)
    a = m.attribute(None, d, None, geo)
    assert a.shape == (n, 2)
    a.sum().backward()
    assert geo.grad.shape == (n, 15)


def test_large_batch_grid_stride_and_repeatability(dev):
    """> 300k points: the backward kernels walk their tiles with a grid-stride loop, and the density backward's grid is
    capped to its scratch blocks.  The batch's gradients equal the sum of its chunks' and two identical backwards agree,
    both up to the order of the float atomics."""
    orc = density_case(21, False)
    m = cuda_model_from_oracle(orc)
    g = torch.Generator().manual_seed(10)
    n = 300_001
    x = (torch.rand(n, 3, generator=g) * 2 - 1).to(dev)
    gs, gg = torch.randn(n, generator=g).to(dev), torch.randn(n, 15, generator=g).to(dev)
    # a texel of a coarse plane sums ~1e4..1e5 contributions of either sign: fp32 reordering moves it by ~sqrt(N) ulp of
    # the running sum (measured up to 1.1e-5 of max), so the parity tolerance is the bound here
    tol = 1e-4
    full1 = _density_grads(m, x, 0.4, gs, gg)
    full2 = _density_grads(m, x, 0.4, gs, gg)
    parts = [_density_grads(m, x[i:i + 100_000], 0.4, gs[i:i + 100_000], gg[i:i + 100_000]) for i in range(0, n, 100_000)]
    for k in full1:
        assert rel_err(full2[k], full1[k]) < tol, k
        assert rel_err(sum(p[k] for p in parts if k in p), full1[k]) < tol, k
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(dev)
    mask = (torch.rand(n, generator=g) > 0.3).to(dev)
    geo, go = torch.randn(n, 15, generator=g).to(dev), torch.randn(n, 2, generator=g).to(dev)
    a1, a2 = _attr_grads(m, d, mask, geo, go), _attr_grads(m, d, mask, geo, go)
    ap = [_attr_grads(m, d[i:i + 100_000], mask[i:i + 100_000], geo[i:i + 100_000], go[i:i + 100_000])
          for i in range(0, n, 100_000)]
    for k in HEADS:
        assert rel_err(a2[k], a1[k]) < tol, k
        assert rel_err(sum(p[k] for p in ap), a1[k]) < tol, k
    assert torch.equal(a1["geo"], a2["geo"])            # per point, no atomics
    assert torch.equal(torch.cat([p["geo"] for p in ap]), a1["geo"])


# ---- 7. stale forward ------------------------------------------------------------------------------------------------
def test_backward_after_parameter_change_raises(dev):
    orc = density_case(21, False)
    m = cuda_model_from_oracle(orc)
    opt = torch.optim.Adam(m.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15)
    x = (torch.rand(500, 3, generator=torch.Generator().manual_seed(11)) * 2 - 1).to(dev)
    d = torch.nn.functional.normalize(x, dim=-1)
    la = m.density(x, _tt(0.4))["sigma"].sum()
    geo = torch.randn(500, 15, device=dev)
    lat = m.attribute(None, d, None, geo).sum()
    lb = m.density(x, _tt(0.4))["sigma"].sum()
    lb.backward()
    opt.step()
    m.density(x, _tt(0.4))                          # re-stages the working set for the new parameters
    with pytest.raises(RuntimeError, match="changed between this forward and its backward"):
        la.backward()
    with pytest.raises(RuntimeError, match="changed between this forward and its backward"):
        lat.backward()
