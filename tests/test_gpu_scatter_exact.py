"""GPU: the backward's scatter stage, entry by entry, against a float64 scatter of its own inputs.

The gradient sinks of the split pipeline (k_bwd_scatter with its segmented and per-vertex warp sums, k_bwd_scatter_static,
k_fold_planes, k_fold_dynamic, k_bwd_flowgrid + k_fold_flow) make no decisions: given what they consumed - dL/dfeature
(SavedView::dfeat), the forward's flow and, in tensor-core mode, dL/d(flow-MLP input) written over flow_in - the table
gradients are a linear function that tests/scatter_ref.py evaluates in float64.  Every entry of every table gradient (static
hash, every dynamic slice, all planes, the flow grid in tensor-core mode) and the saved dL/dflow of every sample is held to

    |got - ref| <= (n + 16) * 2^-24 * A,   got == 0 where no contribution reaches the entry,

with A the sum of the contributions' magnitudes and n their count: a bound that holds whatever order the sums take, so a run
merged over the wrong lanes, a tail lane counted twice or a fold with the wrong weight shows up even where it is far below
1e-4 of the largest entry.  (The end-to-end oracle tests cannot be this strict: the kernels and the oracle make different
ReLU decisions upstream.)

Cases, in both MLP modes of the split pipeline:
  a. the benchmark configuration (L = 16, S = 768, jitter) at N = 2 * 16 * SMs + 37 rays, every scatter CTA wraps; rays of
     synthetic_sweep frames 0, 25, 49 (origins at x = -0.25, 0, +0.25: samples clamp to the box) at the first, an interior
     and the last frame time (both no-neighbour branches);
  b. L = 3 and 5 (odd level counts), S = 45 and 333 (warps straddle rays, a partial last warp);
  c. rays leaving the box through a face, an edge and a corner (clamped samples, bit-identical positions in a row), and
     one batch at bound = 0.5;
  d. a flow large enough that many warped positions leave [0, 1], and a zero flow (warped positions on the faces).
Cases c and d are also rendered end to end through tc-split, fp32-split and fused against the float64 oracle at 1e-4."""
import ctypes
import time

import numpy as np
import pytest
import torch

import scatter_ref as SR
from lidar4d_b200.geometry import make_frame
from lidar4d_b200.model import _RenderFn
from oracle import lidar4d_oracle as O
from parity_util import small_config, cuda_model_from_oracle, rel_err, relu_margin_all, test_rays as _rays

pytestmark = pytest.mark.gpu
MODES = ("tc", "fp32")
MAX_CTAS_128 = 16


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def n_wrap() -> int:
    return 2 * MAX_CTAS_128 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def upstream(N: int, S: int, seed: int, dev):
    g = torch.Generator().manual_seed(seed)
    return {"depth_lidar": torch.randn(N, generator=g).to(dev), "image_lidar": torch.randn(N, 2, generator=g).to(dev),
            "weights_sum_lidar": (torch.randn(N, generator=g) * 0.1).to(dev),
            "weights": (torch.randn(N, S, generator=g) * 0.01).to(dev)}


def train_step(m, ro, rd, t, S, U, monkeypatch=None):
    """One render + backward with a cleared gradient arena; returns (outputs, saved buffer or None)."""
    captured = {}
    if monkeypatch is not None:
        orig = _RenderFn.backward

        def keep_saved(ctx, *g):
            captured["saved"] = ctx.saved             # the backward drops it when it is done
            return orig(ctx, *g)
        monkeypatch.setattr(_RenderFn, "backward", staticmethod(keep_saved))
    m.zero_grad(set_to_none=False)
    m._jitter_calls = 0
    dev = U["depth_lidar"].device
    out = m.render(ro[None].to(dev), rd[None].to(dev), torch.tensor([[t]]), num_steps=S, perturb=True)
    outs = {"depth_lidar": out["depth_lidar"][0], "image_lidar": out["image_lidar"][0],
            "weights_sum_lidar": out["weights_sum_lidar"], "weights": out["weights"]}
    torch.autograd.backward([outs[k] for k in U], [U[k] for k in U])
    torch.cuda.synchronize()
    if monkeypatch is not None:
        monkeypatch.undo()
    return {k: v.detach() for k, v in out.items()}, captured.get("saved")


def assert_scatter_exact(m, ro, rd, t, S, mode, monkeypatch, what, seed=21):
    """Render + backward, then every table-gradient entry and the saved dL/dflow against the float64 scatter."""
    dev = torch.device("cuda:0")
    cfg = m.cfg
    N = ro.shape[0]
    t0 = time.perf_counter()
    out, saved = train_step(m, ro, rd, t, S, upstream(N, S, seed, dev), monkeypatch)
    eng = m._engine
    assert SR.saved_layout(cfg, N, S)["total"] == eng._lib().l4d_saved_bytes(ctypes.byref(eng.ccfg), N, S)
    sv = SR.decode_saved(cfg, saved, N, S)
    x01 = SR.sample_x01(ro.to(dev), rd.to(dev), out["z_vals"], cfg.bound)
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    params = {k: p.detach() for k, p in m.named_parameters()}
    ref = SR.scatter_reference(cfg, params, fr, x01, sv["dfeat"], sv["flow"], sv["flow_in"] if mode == "tc" else None)
    grads = {k: p.grad for k, p in m.named_parameters()}
    bad, worst, touched = {}, 0.0, 0
    for k, r in ref.items():
        got = sv["dflow"].t() if k == "dflow" else grads[k]
        nbad, ratio, at = SR.check_entries(got, r)
        worst = max(worst, ratio)
        touched += int((r[..., 2] > 0).sum())
        if nbad:
            g = got.reshape(-1)[at].item()
            rr = r.reshape(-1, 3)[at]
            bad[k] = (f"{nbad} entries; worst at {at}: got {g:.9e} ref {rr[0].item():.9e} A {rr[1].item():.3e} "
                      f"n {int(rr[2].item())} ({ratio:.2f} x bound)")
    assert not bad, f"{what}: {bad}"
    dflow_live = float(sv["dflow"].abs().max())
    print(f"[scatter-exact] {what}: {touched} touched entries + samples, worst {worst:.3f} of the bound, "
          f"max |dflow| {dflow_live:.2e}, {time.perf_counter() - t0:.1f} s")
    return out, sv, x01


def full_model(mode, seed=0):
    from lidar4d_b200 import LiDAR4D
    torch.manual_seed(seed)
    m = LiDAR4D(num_frames=51, near_lidar=0.0105, far_lidar=0.851, n_levels_hash=16).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if "hash" in k or "grid_enc" in k:
                p.copy_((torch.rand(p.shape, generator=g) - 0.5).cuda())
            elif k.endswith("mlp.4.weight"):
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).cuda())
            elif "planes" in k:
                p.add_((torch.randn(p.shape, generator=g) * 0.1).cuda())
    m.set_mlp_fp16(mode == "tc")
    m.jitter_seed = 5
    return m


# ---- a. the benchmark configuration ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("frame,t", [(0, 0.0), (25, 0.5), (49, 1.0)], ids=["first", "interior", "last"])
def test_benchmark_config(dev, monkeypatch, mode, frame, t):
    """synthetic_sweep frame 49 sits at origin x = +0.25; its rays are rendered at t = 1 so that the launch has no forward
    neighbour (frame 0: no backward neighbour)."""
    from lidar4d_b200.rays import synthetic_sweep
    N, S = n_wrap(), 768
    ro, rd, _ = synthetic_sweep(frame)
    sel = np.linspace(0, ro.shape[0] - 1, N).astype(np.int64)
    ro, rd = torch.from_numpy(ro[sel]).contiguous(), torch.from_numpy(rd[sel]).contiguous()
    m = full_model(mode)
    _, _, x01 = assert_scatter_exact(m, ro, rd, t, S, mode, monkeypatch, f"L16 {mode} frame {frame} t={t}")
    if frame != 25:
        assert bool(((x01 == 0) | (x01 == 1)).any()), "no sample clamps to the box"


# ---- b. odd level counts, warps straddling rays ----------------------------------------------------------------------------
def small_oracle(seed, **over):
    rand = {k: over.pop(k) for k in ("flow_last_std",) if k in over}
    orc = O.build_seeded(small_config(**over), seed, **{"flow_last_std": 0.02, **rand})
    return O.snap_mlp_weights_fp16(orc)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("L,S", [(3, 45), (3, 333), (5, 45), (5, 333)])
def test_small_config_levels(dev, monkeypatch, mode, L, S):
    orc = small_oracle(3, n_levels_hash=L)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 3
    ro, rd = _rays(8, 37)
    assert_scatter_exact(m, torch.from_numpy(ro), torch.from_numpy(rd), 0.4, S, mode, monkeypatch,
                         f"L{L} S{S} {mode}")


# ---- c. rays that leave the box ---------------------------------------------------------------------------------------------
def exit_rays(k: int, n: int, bound: float, seed: int):
    """n rays whose samples clamp on k coordinates: exits through a face (k = 1), an edge (2) or a corner (3) of the box,
    on random sides; far = 0.851 carries them past the box."""
    g = np.random.default_rng(seed)
    ro = np.zeros((n, 3), np.float32)
    rd = np.zeros((n, 3), np.float32)
    for i in range(n):
        axes = g.permutation(3)[:k]
        sign = g.choice([-1.0, 1.0], 3)
        d = g.normal(0, 0.08, 3)
        d[axes] = sign[axes]
        o = g.uniform(-0.1, 0.1, 3) * bound
        o[axes] = sign[axes] * 0.7 * bound
        ro[i], rd[i] = o, d / np.linalg.norm(d)
    return ro, rd


def clamp_batch(bound: float = 1.0, n: int = 32):
    parts = [exit_rays(k, n, bound, 10 + k) for k in (1, 2, 3)]
    return (torch.from_numpy(np.concatenate([p[0] for p in parts])).contiguous(),
            torch.from_numpy(np.concatenate([p[1] for p in parts])).contiguous())


CLAMP_CASES = {"exits": dict(), "bound0.5": dict(bound=0.5)}
FLOW_CASES = {"large-flow": dict(flow_last_std=1.0), "zero-flow": dict()}


def case_setup(name: str, seed: int):
    over = dict(CLAMP_CASES.get(name, {}), **FLOW_CASES.get(name, {}))
    orc = small_oracle(seed, **over)
    if name == "zero-flow":
        with torch.no_grad():
            orc.P["flow_net/mlp/4/weight"].zero_()
    ro, rd = clamp_batch(orc.cfg.bound)
    return orc, ro, rd


def clamp_counts(x01: torch.Tensor, S: int):
    """Samples clamped on 1, 2 and 3 coordinates, and the longest run of bit-identical consecutive positions."""
    on = ((x01 == 0) | (x01 == 1)).sum(1)
    same = (x01[1:] == x01[:-1]).all(1).view(-1)
    run, best = 0, 0
    for v in same.cpu().tolist():
        run = run + 1 if v else 0
        best = max(best, run)
    return [int((on == k).sum()) for k in (1, 2, 3)], best + 1


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["exits", "bound0.5", "large-flow", "zero-flow"])
def test_clamped_and_warped_samples(dev, monkeypatch, mode, name):
    S, t = 256, 0.4
    orc, ro, rd = case_setup(name, 3)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 3
    out, sv, x01 = assert_scatter_exact(m, ro, rd, t, S, mode, monkeypatch, f"{name} {mode}")
    counts, run = clamp_counts(x01, S)
    assert min(counts) > 0 and run >= 32, (counts, run)           # face, edge and corner samples; corner runs span warps
    fl = sv["flow"].t()
    warped = torch.cat([x01 + fl[:, :3], x01 + fl[:, 3:]], 0)
    outside = float(((warped < 0) | (warped > 1)).any(1).double().mean())
    if name == "large-flow":
        assert outside > 0.2, outside
    if name == "zero-flow":
        assert float(fl.abs().max()) == 0.0
        assert bool(((warped == 0) | (warped == 1)).any())
    print(f"[scatter-exact] {name} {mode}: clamped on 1/2/3 coordinates {counts}, longest identical run {run}, "
          f"warped outside the box {outside:.2f}")


# ---- end-to-end parity of cases c and d -----------------------------------------------------------------------------------
MIN_RELU_MARGIN = 5e-8
_e2e = {}


def e2e_case(name: str, S: int):
    """First seed from 3 whose every ReLU keeps > MIN_RELU_MARGIN from its kink and whose weights keep > 1e-6 from the
    1e-4 attribute-mask threshold, then the float64 oracle's outputs and gradients."""
    if name not in _e2e:
        for seed in range(3, 60):
            orc, ro, rd = case_setup(name, seed)
            with torch.no_grad():
                st = orc.render(ro, rd, 0.4, num_steps=S, perturb=True, seed=seed, return_stages=True)
            if relu_margin_all(orc, st, rd.numpy()) > MIN_RELU_MARGIN and bool(((st["weights"] - 1e-4).abs() > 1e-6).all()):
                break
        else:
            pytest.fail(f"{name}: no seed with a ReLU margin > {MIN_RELU_MARGIN}")
        exact = case_setup(name, seed)[0].to_float64()
        ref = exact.render(ro, rd, 0.4, num_steps=S, perturb=True, seed=seed)
        U = upstream(ro.shape[0], S, 16, "cpu")
        torch.autograd.backward([ref[k] for k in U], [U[k].to(ref[k].dtype) for k in U])
        _e2e.clear()
        _e2e[name] = (seed, orc, ro, rd, U, {k: v.detach() for k, v in ref.items()}, exact.ref_named_grads())
    return _e2e[name]


@pytest.mark.parametrize("mode,pipeline", [("tc", "split"), ("fp32", "split"), ("tc", "fused")],
                         ids=["tc-split", "fp32-split", "fused"])
@pytest.mark.parametrize("name", ["exits", "bound0.5", "zero-flow"])
def test_clamped_and_warped_render_parity(dev, name, mode, pipeline):
    """The large-flow case is left out here: its warped positions spread over thousands of texel edges, d(plane)/d(x)
    jumps at every edge, and a sample whose warped position lies within the kernels' flow difference (~1e-6) of an edge
    moves the flow-net gradients by more than 1e-4 of their max in every pipeline.  Measured on an H100: 2.6e-3 on the
    flow grid with the fp32-FMA and fused kernels; with the tensor-core split kernels, whose flow differs more from the
    oracle's, 7e-2 on the flow grid and up to 2e-3 on the other tables.  The exact scatter check above covers that case."""
    S = 128
    seed, orc, ro, rd, U, ref, og = e2e_case(name, S)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.pipeline = pipeline
    m.jitter_seed = seed
    out, _ = train_step(m, ro, rd, 0.4, S, {k: v.to(dev) for k, v in U.items()})
    assert np.array_equal(out["z_vals"].cpu().numpy(), ref["z_vals"].float().numpy())
    for k in ("depth_lidar", "image_lidar", "weights_sum_lidar", "weights"):
        assert rel_err(out[k].reshape(ref[k].shape), ref[k]) < 1e-4, (k, rel_err(out[k].reshape(ref[k].shape), ref[k]))
    G = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    errs = {k: rel_err(G[k], g) for k, g in og.items() if g.numel() and k in G}
    bad = {k: v for k, v in errs.items() if not v < 1e-4}
    assert not bad, f"{name} {mode}/{pipeline} seed {seed}: failing {bad}"
    print(f"[scatter-exact] parity {name} {mode}/{pipeline} seed {seed}: worst gradient {max(errs.values()):.2e}")
