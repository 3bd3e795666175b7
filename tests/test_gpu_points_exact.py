"""GPU: the explicit-point kernels, output by output and entry by entry, against a float64 evaluation of their own inputs.

LiDAR4D.flow (k_flow_fwd / k_flow_bwd), LiDAR4D.density (k_density_train / k_density_bwd) and LiDAR4D.attribute
(k_attribute / k_attribute_bwd) gather from the uncontracted working layouts, scatter straight into the master gradients,
reduce their weight gradients with tile_outer_accum and, in the attribute backward, keep the ones rows' sums per thread
over a CTA's whole grid-stride loop.  tests/points_check.py holds every output to tests/gather_ref.py,
tests/dense_ref.py and tests/scatter_ref.py:

    flow       flow [n, 6], the saved flow-MLP input [16, n], flow_net.mlp.{0,2,4} and every flow-grid entry (exactly 0
               where nothing reaches it, and in a basis slot whose Lagrange weight is 0);
    density    the returned and the saved features and flow-MLP input, σ, geo_feat and flow; every entry of the gradients
               of sigma_net.params (ones columns included), the static hash, all slices of each dynamic plane (exactly 0
               outside the live pair), all planes, the flow MLP and the flow grid;
    attribute  the output [n, 2] and dL/dgeo (exactly 0 outside the mask), every entry of both heads' gradients (the 9 ones
               rows included; rows 1..15 of W3 exactly 0).

Cases: both MLP modes (fp16-rounded working weights, fp32; both run the FMA kernels); L = 3, 8, 9 on small_config with a
bound of 0.75 (2 bound is not a power of two, so (x + b) / (2b) rounds) and the full-size L = 16 configuration; launch sizes
1, 127, 128, 129 and N = 2 * 16 * SMs * 128 + 37, where every CTA of every point kernel gets at least two tiles and the
density backward's 1,024-CTA grid wraps; the first, an interior and the last frame and gather_ref.special_times; points
uniform in the box, out to 1.5 bound, and on hash-cell and plane-texel edges; upstream gradients on σ, on geo or on both
(the kernel then gets a null pointer for the other), scaled by 65536, 2^-20 and 2^-120; attribute masks none, partial, empty
and all but one, directions on the axes; both grad modes, and gradients that hold values before the backward.
Each case prints the worst fraction of the bound per output and the number of ambiguous points."""
import time

import numpy as np
import pytest
import torch

import gather_ref as GR
import points_check as PC
from lidar4d_b200.model import _DensityFn, _FlowFn
from oracle import lidar4d_oracle as O
from parity_util import small_config, cuda_model_from_oracle
from test_gpu_dense_exact import full_model

pytestmark = pytest.mark.gpu
MODES = {"fp16": True, "fp32": False}
SMALL_N = (1, 127, 128, 129)
SCALES = {"x1": 1.0, "x65536": 65536.0, "x2^-20": 2.0 ** -20, "x2^-120": 2.0 ** -120}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


_AMB = [0, 0]                   # points with an ambiguous sigma- or flow-MLP unit, points held (flow and density runs)


@pytest.fixture(autouse=True)
def ambiguity_cap():
    """Over each test's launches, at most MAX_AMBIGUOUS of the points have a sigma- or flow-MLP unit within its bound of
    the kink, so that the bounds stay meaningful without searching for seeds."""
    _AMB[:] = [0, 0]
    yield
    assert _AMB[0] <= PC.MAX_AMBIGUOUS * _AMB[1], f"{_AMB[0]} of {_AMB[1]} points with an ambiguous sigma- or flow-MLP unit"


def n_wrap() -> int:
    """Every point kernel launches at most (resident 128-thread CTAs per SM) x SMs CTAs; N gives each of them >= 2 tiles
    and passes 2 x 1,024 tiles, so the density backward's capped grid wraps too."""
    p = torch.cuda.get_device_properties(0)
    n = 2 * 16 * p.multi_processor_count * 128 + 37
    tiles = (n + 127) // 128
    assert tiles >= 2 * (p.max_threads_per_multi_processor // 128) * p.multi_processor_count and tiles > 2 * 1024
    return n


def small_model(L: int, fp16: bool, seed: int = 3):
    orc = O.build_seeded(small_config(n_levels_hash=L, bound=0.75), seed, flow_last_std=0.02)
    return cuda_model_from_oracle(orc).set_mlp_fp16(fp16)


def points(kind: str, n: int, cfg, seed: int) -> torch.Tensor:
    b = cfg.bound
    g = torch.Generator().manual_seed(seed)
    if kind == "uniform":
        return (torch.rand(n, 3, generator=g) * 2 - 1) * b
    if kind == "outside":
        return (torch.rand(n, 3, generator=g) * 3 - 1.5) * b
    assert kind == "edges"
    # x01 on a plane texel edge i / (R - 1) or a static-hash cell boundary (k - 0.5) / scale, each coordinate on its own;
    # x is nudged by up to 2 ulp so that the kernels' (x + b) / (2b) lands on the target where it can
    tg = [np.arange(cfg.min_resolution * s) / (cfg.min_resolution * s - 1) for s in cfg.plane_scales]
    gs = cfg.static_grid()
    tg += [(np.arange(1, int(gs.scale[l]) + 1) - 0.5) / float(gs.scale[l]) for l in range(cfg.n_levels_hash)]
    rng = np.random.default_rng(seed)
    c = rng.choice(np.concatenate(tg), (n, 3)).astype(np.float32)
    bf = np.float32(b)
    x = (c.astype(np.float64) * 2 * b - b).astype(np.float32)
    best = x.copy()
    for k in (1, 2):
        for sgn in (-1, 1):
            y = x.copy()
            for _ in range(k):
                y = np.nextafter(y, np.float32(sgn * np.inf))
            hit = ((y + bf) / (bf * np.float32(2))) == c
            best = np.where(hit & ~(((best + bf) / (bf * np.float32(2))) == c), y, best)
    return torch.from_numpy(best)


def capture(monkeypatch, cls):
    """The autograd context of the next cls.apply (its saved buffer)."""
    box = {}
    orig = cls.forward

    def fwd(ctx, *a):
        out = orig(ctx, *a)
        box["ctx"] = ctx
        return out
    monkeypatch.setattr(cls, "forward", staticmethod(fwd))
    return box


def params_of(m):
    return {k: p.detach() for k, p in m.named_parameters()}


def grads_of(m, loss, grad_mode, prefill):
    names, ps = zip(*m.named_parameters())
    m.grad_mode = grad_mode
    if grad_mode == "arena":
        for k, p in zip(names, ps):
            p.grad = None if prefill is None else prefill[k].clone()
        if prefill is None:
            m.zero_grad(set_to_none=False)
        loss.backward()
        return {k: (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)) for k, p in zip(names, ps)}
    gs = torch.autograd.grad(loss, ps, allow_unused=True)
    return {k: (g.detach().clone() if g is not None else torch.zeros_like(p)) for k, p, g in zip(names, ps, gs)}


def make_prefill(m, seed=9):
    g = torch.Generator().manual_seed(seed)
    return {k: (torch.randn(p.shape, generator=g) * 1e-3).float().to(p.device) for k, p in m.named_parameters()}


# ---- runners ---------------------------------------------------------------------------------------------------------
def run_flow(m, x, t, scale, monkeypatch, grad_mode="arena", prefill=None, backward=True, what=""):
    dev = torch.device("cuda:0")
    t0 = time.perf_counter()
    n = x.shape[0]
    g_flow = (torch.randn(n, 6, generator=torch.Generator().manual_seed(5)) * scale).to(dev) if backward else None
    box = capture(monkeypatch, _FlowFn)
    out = m.flow(x.to(dev), torch.tensor([[t]]))
    fl = torch.cat([out["forward"], out["backward"]], 1)
    fin = box["ctx"].saved.clone()
    grads = grads_of(m, (fl * g_flow).sum(), grad_mode, prefill) if backward else None
    monkeypatch.undo()
    torch.cuda.synchronize()
    st = PC.hold_flow(m.cfg, params_of(m), m._engine.mlp_fp16, t, x.to(dev), fl.detach(), fin, g_flow, grads, prefill,
                      what=what)
    _AMB[0] += st["ambiguous"]
    _AMB[1] += n
    print(f"[points-exact] flow {what}: {st['holder'].line()}; ambiguous {st['ambiguous']} of {n}; "
          f"{time.perf_counter() - t0:.1f} s")
    return st


def run_density(m, x, t, scale, which, monkeypatch, grad_mode="arena", prefill=None, what=""):
    dev = torch.device("cuda:0")
    t0 = time.perf_counter()
    n = x.shape[0]
    g = torch.Generator().manual_seed(6)
    gs = (torch.randn(n, generator=g) * scale).to(dev) if which in ("sigma", "both") else None
    gg = (torch.randn(n, 15, generator=g) * scale).to(dev) if which in ("geo", "both") else None
    box = capture(monkeypatch, _DensityFn)
    out = m.density(x.to(dev), torch.tensor([[t]]), return_features=True)
    fin, feat = PC.density_saved_views(m.cfg, box["ctx"].saved, n)
    fin, feat = fin.clone(), feat.clone()
    loss = sum(((out[k] * u).sum() for k, u in (("sigma", gs), ("geo_feat", gg)) if u is not None))
    grads = grads_of(m, loss, grad_mode, prefill)
    monkeypatch.undo()
    torch.cuda.synchronize()
    o = {k: v.detach() for k, v in out.items()}
    st = PC.hold_density(m.cfg, params_of(m), m._engine.mlp_fp16, t, x.to(dev), o, fin, feat, gs, gg, grads, prefill,
                         what=what)
    _AMB[0] += st["ambiguous"]
    _AMB[1] += n
    print(f"[points-exact] density {what}: {st['holder'].line()}; ambiguous {st['ambiguous']} of {n}; "
          f"{time.perf_counter() - t0:.1f} s")
    return st


def run_attribute(m, n, mask_kind, scale, grad_mode="arena", prefill=None, what="", seed=2):
    dev = torch.device("cuda:0")
    t0 = time.perf_counter()
    g = torch.Generator().manual_seed(seed)
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    ax = torch.tensor([[1.0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0], [0, -1.0, 0], [0, 0, 1.0], [0, 0, -1.0]])
    k = min(n, 6)
    d[:k] = ax[:k]
    geo = torch.randn(n, 15, generator=g)
    mask = {"none": None, "partial": torch.rand(n, generator=g) > 0.4, "empty": torch.zeros(n, dtype=torch.bool),
            "all-but-one": torch.arange(n) != n // 2}[mask_kind]
    g_out = (torch.randn(n, 2, generator=g) * scale).to(dev)
    d, geo_d = d.to(dev), geo.to(dev).requires_grad_(True)
    md = None if mask is None else mask.to(dev)
    m.grad_mode = grad_mode
    out = m.attribute(None, d, md, geo_d)
    heads = [dict(m.named_parameters())[k] for k in PC.HEADS]
    if grad_mode == "arena":
        for k, p in zip(PC.HEADS, heads):
            p.grad = None if prefill is None else prefill[k].clone()
        (out * g_out).sum().backward()
        grads = {k: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for k, p in zip(PC.HEADS, heads)}
        g_geo = geo_d.grad
    else:
        gs = torch.autograd.grad((out * g_out).sum(), heads + [geo_d], allow_unused=True)
        grads = {k: (v if v is not None else torch.zeros_like(p)) for k, p, v in zip(PC.HEADS, heads, gs[:2])}
        g_geo = gs[2]
    torch.cuda.synchronize()
    st = PC.hold_attribute(m.cfg, params_of(m), m._engine.mlp_fp16, d, geo_d.detach(), md, out.detach(), g_out, g_geo,
                           grads, prefill, what=what)
    print(f"[points-exact] attribute {what}: {st['holder'].line()}; ambiguous (attribute nets) {st['ambiguous']} of {n}; "
          f"{time.perf_counter() - t0:.1f} s")
    return st


# ---- small configurations: launch sizes, frames, points, upstream gradients ----------------------------------------
def frames(cfg):
    single, row = GR.special_times(cfg)
    return {"first": 0.0, "interior": 0.4, "last": 1.0, "single": single, "row": row}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("L", [3, 8, 9])
def test_small_launches(dev, monkeypatch, mode, L):
    """Every frame x point kind at n = 129 and the interior frame at n = 1, 127, 128: flow and density (σ and geo
    upstream), and the attribute nets at each n."""
    m = small_model(L, MODES[mode])
    cfg = m.cfg
    cases = [(f, k, 129) for f in frames(cfg) for k in ("uniform", "outside", "edges")]
    cases += [("interior", "uniform", n) for n in SMALL_N if n != 129]
    for ci, (fname, kind, n) in enumerate(cases):
        x = points(kind, n, cfg, 100 * L + ci)
        w = f"L{L} {mode} {fname} {kind} n={n}"
        run_flow(m, x, frames(cfg)[fname], 1.0, monkeypatch, what=w)
        run_density(m, x, frames(cfg)[fname], 1.0, "both", monkeypatch, what=w)
    for n in SMALL_N:
        run_attribute(m, n, "partial" if n > 1 else "none", 1.0, what=f"L{L} {mode} n={n}")


@pytest.mark.parametrize("mode", list(MODES))
def test_edges_are_hit(dev, monkeypatch, mode):
    """The edge points do sit on hash-cell and plane-texel edges in the kernels' own float32 arithmetic."""
    m = small_model(8, MODES[mode])
    cfg = m.cfg
    x = points("edges", 4096, cfg, 1)
    import scatter_ref as SR
    x01 = SR.point_x01(x, cfg.bound)
    on_texel = on_cell = 0
    for s in cfg.plane_scales:
        R = cfg.min_resolution * s
        on_texel += int((SR.axis(x01.reshape(-1), R)[3] == 0).sum())
    gs = cfg.static_grid()
    for l in range(cfg.n_levels_hash):
        on_cell += int((O.hash_indices(x01, gs, l)[1] == 0).any(1).sum())
    assert on_texel > 1000 and on_cell > 100, (on_texel, on_cell)
    run_density(m, x, 0.4, 1.0, "both", monkeypatch, what=f"edges n=4096 {mode}")


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("scale", list(SCALES))
@pytest.mark.parametrize("which", ["sigma", "geo", "both"])
def test_upstream_gradients(dev, monkeypatch, mode, scale, which):
    m = small_model(8, MODES[mode])
    x = points("outside", 3000, m.cfg, 7)
    run_density(m, x, 0.4, SCALES[scale], which, monkeypatch, what=f"{which} {scale} {mode}")
    if which == "both":
        run_flow(m, x, 0.4, SCALES[scale], monkeypatch, what=f"{scale} {mode}")
        for mk in ("none", "partial", "empty", "all-but-one"):
            run_attribute(m, 3000, mk, SCALES[scale], what=f"mask {mk} {scale} {mode}")


@pytest.mark.parametrize("mode", list(MODES))
def test_flow_forward_only(dev, monkeypatch, mode):
    m = small_model(8, MODES[mode])
    for fname, t in frames(m.cfg).items():
        run_flow(m, points("outside", 2000, m.cfg, 8), t, 1.0, monkeypatch, backward=False, what=f"forward only {fname} {mode}")


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("grad_mode,prefilled", [("autograd", False), ("arena", True)], ids=["autograd", "prefilled"])
def test_grad_modes(dev, monkeypatch, mode, grad_mode, prefilled):
    m = small_model(9, MODES[mode])
    pf = make_prefill(m) if prefilled else None
    x = points("uniform", 3000, m.cfg, 9)
    w = f"{grad_mode}{' prefilled' if prefilled else ''} {mode}"
    run_flow(m, x, 0.4, 1.0, monkeypatch, grad_mode, pf, what=w)
    run_density(m, x, 0.4, 1.0, "both", monkeypatch, grad_mode, pf, what=w)
    run_attribute(m, 3000, "partial", 1.0, grad_mode, pf, what=w)


# ---- full size and the wrap size ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
def test_full_size_wrap(dev, monkeypatch, mode):
    """The benchmark configuration (L = 16, default tables) at N: first, interior and last frame for flow and density,
    points out to 1.5 bound; the attribute nets with a partial mask."""
    m = full_model("tc" if MODES[mode] else "fp32")
    assert m.cfg.sigma_in_dim == 176
    N = n_wrap()
    for fname, t in (("first", 0.0), ("interior", 0.5), ("last", 1.0)):
        x = points("outside", N, m.cfg, 11)
        run_flow(m, x, t, 1.0, monkeypatch, what=f"L16 N={N} {fname} {mode}")
        run_density(m, x, t, 1.0, "both", monkeypatch, what=f"L16 N={N} {fname} {mode}")
    run_attribute(m, N, "partial", 1.0, what=f"L16 N={N} {mode}")
    run_attribute(m, 129, "all-but-one", 1.0, what=f"L16 n=129 {mode}")
