"""GPU (H100) parity tests proper: the product path - LiDAR4D module -> ctypes ->
liblidar4d_b200.so kernels - against the oracle and the committed golden vectors.
Tolerance 1e-4 rel-to-max fp32 (BASELINE.json north_star); hash indices bit-exact."""
import os

import numpy as np
import pytest
import torch

from oracle import lidar4d_oracle as O
from lidar4d_b200.geometry import FieldConfig, make_frame
from parity_util import small_config, rel_err, make_surface_like, relu_margin, cuda_model_from_oracle, test_rays as _rays

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def test_native_library_is_loaded(dev):
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    assert lib.l4d_abi_version() == 1
    maps = open("/proc/self/maps").read()
    assert "liblidar4d_b200.so" in maps


def test_hash_indices_bit_exact(dev):
    from lidar4d_b200 import LiDAR4D
    fx = np.load(os.path.join(GOLD, "hash_indices.npz"))
    m = LiDAR4D().to(dev)
    for gid, name in [(0, "static3d"), (1, "dyn2d_xy"), (2, "dyn2d_xz"), (4, "flow3d")]:
        x = torch.from_numpy(fx[name + ":x"]).to(dev)
        for l in range(int(fx[name + ":scale"].shape[0])):
            idx, w = m.hash_indices(gid, l, x)
            assert np.array_equal(idx.cpu().numpy().view(np.uint32), fx[f"{name}:idx{l}"]), (name, l)
            assert np.array_equal(w.cpu().numpy(), fx[f"{name}:w{l}"]), (name, l)


@pytest.mark.parametrize("t", [0.4, 0.0, 1.0])
def test_density_stages(dev, t):
    orc = O.build_seeded(small_config(), 3, flow_last_std=0.02)
    m = cuda_model_from_oracle(orc)
    x = torch.rand(1000, 3, generator=torch.Generator().manual_seed(0)) * 2 - 1
    ref = orc.density(x, make_frame(t, orc.cfg.num_frames, orc.cfg.time_resolution), return_features=True)
    got = m.density(x.to(dev), torch.tensor([[t]]), return_features=True)
    for k in ("flow", "features", "sigma", "geo_feat"):
        assert rel_err(got[k], ref[k]) < TOL, k


CASES = [(0.4, 200, False, 3, False), (0.0, 150, True, 4, False), (1.0, 130, True, 5, False),
         (0.6, 260, True, 6, True), (0.4, 768, True, 27, False)]
MIN_RELU_MARGIN = 1e-8      # see tests/test_hostsim_parity.py


@pytest.mark.parametrize("pipeline", ["split", "fused"])
@pytest.mark.parametrize("t,S,perturb,seed,surface", CASES)
def test_render_forward_backward(dev, t, S, perturb, seed, surface, pipeline):
    orc = O.build_seeded(small_config(), seed, flow_last_std=0.02)
    if surface:
        make_surface_like(orc)
    m = cuda_model_from_oracle(orc)
    m.pipeline = pipeline
    m.jitter_seed = seed
    ro, rd = _rays(3, 8) if S < 700 else _rays(2, 5)
    N = ro.shape[0]
    ref = orc.render(torch.from_numpy(ro), torch.from_numpy(rd), t, num_steps=S, perturb=perturb, seed=seed,
                     return_stages=True)
    assert relu_margin(orc, ref) > MIN_RELU_MARGIN
    out = m.render(torch.from_numpy(ro)[None].to(dev), torch.from_numpy(rd)[None].to(dev), torch.tensor([[t]]),
                   staged=False, num_steps=S, perturb=perturb)
    assert out["depth_lidar"].shape == (1, N) and out["image_lidar"].shape == (1, N, 2)
    assert np.array_equal(out["z_vals"].cpu().numpy(), ref["z_vals"].numpy())
    for k in ("depth_lidar", "image_lidar", "weights_sum_lidar", "weights"):
        assert rel_err(out[k], ref[k]) < TOL, k
    g = torch.Generator().manual_seed(1)
    gd, gi = torch.randn(N, generator=g), torch.randn(N, 2, generator=g)
    gw, gww = torch.randn(N, generator=g) * 0.1, torch.randn(N, S, generator=g) * 0.01
    (ref["depth_lidar"] * gd).sum().add((ref["image_lidar"] * gi).sum()).add(
        (ref["weights_sum_lidar"] * gw).sum()).add((ref["weights"] * gww).sum()).backward()
    loss = (out["depth_lidar"][0] * gd.to(dev)).sum() + (out["image_lidar"][0] * gi.to(dev)).sum() + \
           (out["weights_sum_lidar"] * gw.to(dev)).sum() + (out["weights"] * gww.to(dev)).sum()
    loss.backward()
    og = orc.ref_named_grads()
    got = {k: p.grad for k, p in m.named_parameters()}
    errs = {k: rel_err(got[k], g_ref) for k, g_ref in og.items() if g_ref.numel()}
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, f"worst {max(errs.values()):.2e}; failing: {bad}"


@pytest.mark.parametrize("name", ["ref_small_interior", "ref_small_first", "ref_small_last", "ref_small_active"])
def test_against_reference_golden(dev, name):
    import ast
    fx = np.load(os.path.join(GOLD, name + ".npz"))
    extra = ast.literal_eval(str(fx["extra"])) if "extra" in fx.files else {}    # active_sensor / density_scale / bound of the case
    orc = O.build_seeded(small_config(**extra), int(fx["seed"]), flow_last_std=0.02)
    m = cuda_model_from_oracle(orc)
    m.jitter_seed = int(fx["seed"])
    S = int(fx["num_steps"])
    out = m.render(torch.from_numpy(fx["rays_o"])[None].to(dev), torch.from_numpy(fx["rays_d"])[None].to(dev),
                   torch.tensor([[float(fx["time"])]]), num_steps=S, perturb=bool(fx["perturb"]))
    assert rel_err(out["depth_lidar"], fx["ref_depth_lidar"]) < TOL
    assert rel_err(out["image_lidar"], fx["ref_image_lidar"]) < TOL
    assert rel_err(out["weights"], fx["ref_weights"]) < TOL
    loss = (out["depth_lidar"][0] * torch.from_numpy(fx["g_depth"]).to(dev)).sum() + \
           (out["image_lidar"][0] * torch.from_numpy(fx["g_image"]).to(dev)).sum()
    loss.backward()
    got = {k: p.grad for k, p in m.named_parameters()}
    for k in [k[5:] for k in fx.files if k.startswith("grad:")]:
        if fx["grad:" + k].size:
            assert rel_err(got[k], fx["grad:" + k]) < TOL, k
    for k in [k[9:] for k in fx.files if k.startswith("gradnorm:")]:
        n_ref = float(fx["gradnorm:" + k])
        if got.get(k) is None:                     # view_encoder.params: empty tensor, never receives a gradient
            assert n_ref == 0.0, k
            continue
        assert abs(float(got[k].double().norm()) - n_ref) <= 1e-4 * n_ref + 1e-12, k


@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_renderer_options_against_oracle(dev, mode):
    """active_sensor (exponent x2, renderer.py:100-102), density_scale and a non-unit bound, both kernel families."""
    from parity_util import relu_margin_all
    ro, rd = _rays(3, 8)
    N, S = ro.shape[0], 150
    for seed in range(12, 60):          # first seed with every ReLU (attribute heads included) clear of its kink
        orc = O.build_seeded(small_config(active_sensor=True, density_scale=0.7, bound=1.5), seed, flow_last_std=0.02)
        if mode == "tc":
            orc.mlp_dtype = "fp16"
        ref = orc.render(torch.from_numpy(ro), torch.from_numpy(rd), 0.4, num_steps=S, perturb=True, seed=seed, return_stages=True)
        if relu_margin_all(orc, ref, rd) > 3e-7:
            break
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = seed
    out = m.render(torch.from_numpy(ro)[None].to(dev), torch.from_numpy(rd)[None].to(dev), torch.tensor([[0.4]]), num_steps=S, perturb=True)
    for k in ("depth_lidar", "image_lidar", "weights"):
        assert rel_err(out[k], ref[k]) < TOL, k
    (ref["depth_lidar"].sum() + ref["image_lidar"].sum()).backward()
    (out["depth_lidar"].sum() + out["image_lidar"].sum()).backward()
    og = orc.ref_named_grads()
    errs = {k: rel_err(p.grad, og[k]) for k, p in m.named_parameters() if p.grad is not None and og[k].numel()}
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad


def test_flow_forward_backward(dev):
    orc = O.build_seeded(small_config(), 8, flow_last_std=0.05)
    m = cuda_model_from_oracle(orc)
    x = torch.rand(1333, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1
    g = torch.randn(1333, 6, generator=torch.Generator().manual_seed(3))
    ref = orc.flow(x, 0.35)
    fl = torch.cat([ref["forward"], ref["backward"]], -1)
    (fl * g).sum().backward()
    out = m.flow(x.to(dev), torch.tensor([[0.35]]))
    got = torch.cat([out["forward"], out["backward"]], -1)
    assert rel_err(got, fl) < TOL
    (got * g.to(dev)).sum().backward()
    og = orc.ref_named_grads()
    for k in ("flow_net.grid_enc.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight"):
        assert rel_err(dict(m.named_parameters())[k].grad, og[k]) < TOL, k


@pytest.mark.parametrize("fp16", [False, True])
def test_attribute_heads_standalone(dev, fp16):
    """LiDAR4D.attribute (lidar4d.py:191-223) on explicit directions / geo features, with and without a mask."""
    orc = O.build_seeded(small_config(), 14)
    if fp16:
        orc.mlp_dtype = "fp16"
    m = cuda_model_from_oracle(orc).set_mlp_fp16(fp16)
    g = torch.Generator().manual_seed(2)
    n = 301
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    geo = torch.randn(n, 15, generator=g)
    mask = torch.rand(n, generator=g) > 0.4
    for mk in (None, mask, torch.zeros(n, dtype=torch.bool)):
        ref = orc.attribute(d, geo, mk)
        got = m.attribute(None, d.to(dev), None if mk is None else mk.to(dev), geo.to(dev))
        assert got.shape == (n, 2)
        assert float((got.cpu() - ref).abs().max()) < 1e-5
        if mk is not None:
            assert float(got.cpu()[~mk].abs().max() if (~mk).any() else 0.0) == 0.0


def test_staged_render_and_empty_mask(dev):
    orc = O.build_seeded(small_config(), 9)
    c = orc.cfg
    with torch.no_grad():
        orc.p("sigma_net.params")[64 * c.sigma_in_pad:64 * c.sigma_in_pad + 64] = -3.0
    m = cuda_model_from_oracle(orc)
    ro, rd = _rays(2, 7)
    with torch.no_grad():
        out = m.render(torch.from_numpy(ro)[None].to(dev), torch.from_numpy(rd)[None].to(dev), torch.tensor([[0.4]]),
                       staged=True, max_ray_batch=5, num_steps=129)
    assert set(out.keys()) == {"depth_lidar", "image_lidar"}
    assert float(out["image_lidar"].abs().max()) == 0.0
    ref = orc.render(torch.from_numpy(ro), torch.from_numpy(rd), 0.4, num_steps=129)
    assert float((out["depth_lidar"].cpu()[0] - ref["depth_lidar"]).abs().max()) < 1e-6


# ---- full-size configuration: size-independent properties -------------------------------------
@pytest.fixture(scope="module")
def full_model(dev):
    from lidar4d_b200 import LiDAR4D
    torch.manual_seed(0)
    m = LiDAR4D(num_frames=51, near_lidar=0.0105, far_lidar=0.851).to(dev)
    g = torch.Generator(device="cpu").manual_seed(0)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if "hash" in k or "grid_enc" in k:
                p.copy_(((torch.rand(p.shape, generator=g) - 0.5)).to(dev))
            elif k.endswith("mlp.4.weight"):
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(dev))
            elif "planes" in k:      # constant time planes have zero spatial derivative: no gradient would reach the flow net
                p.add_((torch.randn(p.shape, generator=g) * 0.1).to(dev))
    return m


def test_full_size_properties(dev, full_model):
    from lidar4d_b200.rays import synthetic_sweep
    m = full_model
    ro, rd, t = synthetic_sweep(7)
    sel = np.arange(0, 65536, 257)[:200]
    ro_t, rd_t = torch.from_numpy(ro[sel])[None].to(dev), torch.from_numpy(rd[sel])[None].to(dev)
    tt = torch.tensor([[float(t)]])
    with torch.no_grad():
        a = m.render(ro_t, rd_t, tt, num_steps=768, perturb=False)
        b = m.render(ro_t, rd_t, tt, num_steps=768, perturb=False)
        # determinism, chunk invariance (renderer.py:165-177) and the ray_offset contract
        for k in ("depth_lidar", "image_lidar", "weights"):
            assert torch.equal(a[k], b[k]), k
        c = m.render(ro_t, rd_t, tt, staged=True, max_ray_batch=64, num_steps=768, perturb=False)
        assert torch.equal(c["depth_lidar"], a["depth_lidar"]) and torch.equal(c["image_lidar"], a["image_lidar"])
        # the single-kernel and the split pipeline run the same per-sample code: results agree to fp32 rounding
        m.pipeline = "fused"
        f = m.render(ro_t, rd_t, tt, num_steps=768, perturb=False)
        m.pipeline = "split"
        assert rel_err(f["depth_lidar"], a["depth_lidar"]) < 1e-5 and rel_err(f["image_lidar"], a["image_lidar"]) < 1e-5
    w = a["weights"]
    assert torch.isfinite(w).all() and float(w.min()) >= 0.0
    assert float(a["weights_sum_lidar"].max()) <= 1.0 + 1e-4
    assert torch.allclose(a["weights_sum_lidar"], w.sum(-1), rtol=1e-4, atol=1e-5)
    assert torch.allclose(a["depth_lidar"][0], (w * a["z_vals"]).sum(-1), rtol=1e-4, atol=1e-5)
    assert float(a["image_lidar"].min()) >= 0.0 and float(a["image_lidar"].max()) <= 1.0 + 1e-4
    z = a["z_vals"]
    assert bool((z[:, 1:] > z[:, :-1]).all())                       # sortedness of the samples

    # linearity of the backward in the upstream gradient: grad(2g1 + g2) == 2 grad(g1) + grad(g2)
    def grads(gd, gi):
        m.zero_grad(set_to_none=True)
        out = m.render(ro_t[:, :32], rd_t[:, :32], tt, num_steps=768, perturb=True)
        m._jitter_calls = 0
        ((out["depth_lidar"][0] * gd).sum() + (out["image_lidar"][0] * gi).sum()).backward()
        return {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    g = torch.Generator().manual_seed(5)
    gd1, gi1 = torch.randn(32, generator=g).to(dev), torch.randn(32, 2, generator=g).to(dev)
    gd2, gi2 = torch.randn(32, generator=g).to(dev), torch.randn(32, 2, generator=g).to(dev)
    m._jitter_calls = 0
    G1, G2, G3 = grads(gd1, gi1), grads(gd2, gi2), grads(2 * gd1 + gd2, 2 * gi1 + gi2)
    for k in G3:
        lin = 2 * G1[k] + G2[k]
        assert rel_err(G3[k], lin) < 2e-4, k          # fp32 atomics: summation order differs run to run
    # every parameter family receives gradient
    for k in ("planes_encoder.planes.0.0", "planes_encoder.planes.3.5", "hash_encoder.hash_static.params",
              "flow_net.grid_enc.params", "flow_net.mlp.0.weight", "sigma_net.params", "raydrop_net.params"):
        assert float(G3[k].abs().max()) > 0, k
    # the warped hash queries are no_grad: only the slices of the (x,t) query receive gradient
    fr = make_frame(t, 51, 8)
    live = {fr.cur.slice_lo, fr.cur.slice_hi}
    for s in range(8):
        gmax = float(G3[f"hash_encoder.hash_dynamic.0.hash_t.{s}.params"].abs().max())
        assert (gmax > 0) == (s in live), (s, live)


def test_training_step_changes_loss(dev, full_model):
    """A few Adam steps through the reference's optimiser recipe (main_lidar4d.py:298-300) reduce an L1 depth loss;
    the staged working set is refreshed after each optimizer.step()."""
    from lidar4d_b200.rays import synthetic_sweep
    m = full_model
    opt = torch.optim.Adam(m.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15)
    ro, rd, t = synthetic_sweep(3)
    sel = np.arange(0, 65536, 64)[:1024]
    ro_t, rd_t = torch.from_numpy(ro[sel])[None].to(dev), torch.from_numpy(rd[sel])[None].to(dev)
    target = torch.full((1, 1024), 0.3, device=dev)
    losses = []
    for it in range(4):
        opt.zero_grad()
        out = m.render(ro_t, rd_t, torch.tensor([[float(t)]]), num_steps=768, perturb=True)
        loss = (out["depth_lidar"] - target).abs().mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


@pytest.mark.parametrize("N,K", [(64, 128), (16, 64), (128, 16), (64, 384), (8 * 2, 16)])
def test_tcgen05_selftest_gemm(dev, N, K):
    """The tensor-core building blocks (smem descriptors, wgmma issue/wait, accumulator fragment layout) in isolation."""
    import ctypes as C
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    g = torch.Generator().manual_seed(N * 1000 + K)
    A = (torch.randn(128, K, generator=g)).half().to(dev)
    B = (torch.randn(N, K, generator=g)).half().to(dev)
    Cc = torch.zeros(128, N, device=dev)
    rc = lib.l4d_tc_selftest(A.data_ptr(), B.data_ptr(), Cc.data_ptr(), N, K, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.l4d_last_error()
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    assert rel_err(Cc, ref) < 1e-5


TC_CASES = [(0.4, 200, False, 3, False), (0.0, 150, True, 4, False), (0.6, 260, True, 6, True), (0.4, 768, True, 27, False)]


# odd level counts: sigma_in_dim = 85 / 99 is not a multiple of 4 or 8, so the feature-tile writer takes its scalar path,
# the last stored 16-byte chunk is partly ones-padding and the last dfeat float4 is partly unused
TC_CASES += [(0.4, 140, True, 11, False, 3), (0.4, 140, True, 11, False, 5)]


@pytest.mark.parametrize("case", TC_CASES)
def test_tensor_core_path(dev, case):
    """mlp_fp16 mode: the dense kernels run on wgmma tensor cores (fp16 hi/lo-split activations, fp16 weights,
    fp32 accumulation).  The oracle emulates the fp16 weight rounding exactly; tolerance stays 1e-4."""
    t, S, perturb, seed, surface = case[:5]
    orc = O.build_seeded(small_config(**({"n_levels_hash": case[5]} if len(case) > 5 else {})), seed, flow_last_std=0.02)
    if surface:
        make_surface_like(orc)
    orc.mlp_dtype = "fp16"
    m = cuda_model_from_oracle(orc).set_mlp_fp16(True)
    m.jitter_seed = seed
    ro, rd = _rays(3, 8) if S < 700 else _rays(2, 5)
    N = ro.shape[0]
    ref = orc.render(torch.from_numpy(ro), torch.from_numpy(rd), t, num_steps=S, perturb=perturb, seed=seed,
                     return_stages=True)
    assert relu_margin(orc, ref) > MIN_RELU_MARGIN
    out = m.render(torch.from_numpy(ro)[None].to(dev), torch.from_numpy(rd)[None].to(dev), torch.tensor([[t]]),
                   staged=False, num_steps=S, perturb=perturb)
    for k in ("depth_lidar", "image_lidar", "weights_sum_lidar", "weights"):
        assert rel_err(out[k], ref[k]) < TOL, k
    g = torch.Generator().manual_seed(1)
    gd, gi = torch.randn(N, generator=g), torch.randn(N, 2, generator=g)
    ((ref["depth_lidar"] * gd).sum() + (ref["image_lidar"] * gi).sum()).backward()
    ((out["depth_lidar"][0] * gd.to(dev)).sum() + (out["image_lidar"][0] * gi.to(dev)).sum()).backward()
    og = orc.ref_named_grads()
    got = {k: p.grad for k, p in m.named_parameters()}
    errs = {k: rel_err(got[k], g_ref) for k, g_ref in og.items() if g_ref.numel()}
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, f"worst {max(errs.values()):.2e}; failing: {bad}"


def _tile_kmajor(X):       # X [rows][K] fp16 -> [K/8][rows][8]
    rows, K = X.shape
    return X.view(rows, K // 8, 8).permute(1, 0, 2).contiguous()


def _tile_mnmajor(X):      # X [rows=mn][K] fp16 -> [mn/8][K][8]
    rows, K = X.shape
    return X.view(rows // 8, 8, K).permute(0, 2, 1).contiguous()


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(128, 64, 128, 0, 0), (128, 64, 128, 1, 0), (128, 64, 64, 0, 1), (128, 176, 64, 0, 1),
                                             (128, 64, 128, 1, 1), (64, 64, 128, 1, 1), (64, 16, 128, 1, 1), (64, 8, 128, 1, 1),
                                             (64, 64, 64, 0, 0), (128, 16, 16, 0, 1)])
def test_tcgen05_selftest_layouts(dev, M, N, K, a_mn, b_mn):
    """MN-major operands (sample-major tiles read transposed) and M=64 accumulators, as the tensor-core backward uses them."""
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    g = torch.Generator().manual_seed(M + 7 * N + 13 * K + a_mn + 2 * b_mn)
    A = torch.randn(M, K, generator=g).half()
    B = torch.randn(N, K, generator=g).half()
    At = (_tile_mnmajor(A) if a_mn else _tile_kmajor(A)).to(dev)
    Bt = (_tile_mnmajor(B) if b_mn else _tile_kmajor(B)).to(dev)
    Cc = torch.zeros(M, N, device=dev)
    rc = lib.l4d_tc_selftest2(At.data_ptr(), Bt.data_ptr(), Cc.data_ptr(), M, N, K, a_mn, b_mn, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.l4d_last_error()
    torch.cuda.synchronize()
    assert rel_err(Cc, A.float() @ B.float().t()) < 1e-5
