"""GPU: the MLP stages of the split pipeline, output by output and entry by entry, against a float64 evaluation of their
own inputs.

k_fwd_dense{,_tc}, k_bwd_dense{,_tc}, k_fwd_flow_tc / the flow MLP of k_fwd_gather, and k_bwd_flow{,_tc} are held to
tests/dense_ref.py: given the features X the training forward saved (fp16 hi + lo operand tiles in tensor-core mode), the
attribute mask it decided, the working weights, dL/dσ and dL/dattr of the compositing evaluated exactly on the saved σ and
attributes (tests/compositing_ref.py, with its bounds carried in), the flow-MLP input (copied before the backward, which
overwrites it in tensor-core mode) and the saved dL/dflow, every output must lie within the reference's bound:

    forward    σ, both attribute heads (exactly 0 outside the mask), the 6 flow outputs, per sample;
    backward   dL/dfeature [P, K] per sample, dL/d(flow-MLP input) [P, 16] in tensor-core mode; every entry of the
               gradients of sigma_net.params (W1 with its ones columns, W2), intensity_net.params and raydrop_net.params
               (W1 with its direction and 9 ones rows, W2, W3; rows 1..15 of W3 exactly 0) and flow_net.mlp.{0,2,4}.

Cases, in tensor-core and fp32 split modes:
  a. the benchmark configuration (L = 16: in_pad 176, the third 64-column block, no ones column; S = 768) at
     N = 2 * 16 * SMs + 37 rays, so every per-ray CTA of the dense kernels gets >= 2 rays (the per-ray s_csum reset and
     flush of the attribute nets); an interior and the first frame;
  b. L = 3, 8, 9, 10 (K = 85, 120, 127, 134: 11, 8, 1 and 10 ones columns; at L = 10 the third block is partial) with
     S = 2, 129, 333 (partial last tiles, flow tiles straddling rays), MLP masters not rounded to fp16 beforehand; and
     one-ray launches, where an entry has so few contributions that a hi|lo product missing one of its terms shows;
  c. transparent, opaque (tiles behind the surface carry deltas of ~1e-35 next to ~1) and active_sensor, with upstream
     gradients on every term (image included), on the image only (the sigma MLP then reached through geo alone), times
     65536 and times 2^-20; and upstream gradients of 2^-110 and 2^-120, whose whole tiles carry deltas so small that the
     tile scale sc sits at its 2^126 cap and sc r passes 2^128 (asserted from the reference's tile maxima), where
     1 / (sc r) would be 0 and (1/sc)/r is a subnormal;
  d. a launch with every sample outside the attribute mask, and rays partly inside it;
  e. gradients that hold values when the backward starts: `got - prefill` against the bound plus one rounding (the
     kernels accumulate into the gradient arena's work slices, which k_unstage_jobs folds into .grad).
Each case prints the worst fraction of the bound per output and the number of samples with an ambiguous ReLU unit."""
import time

import numpy as np
import pytest
import torch

import compositing_ref as CR
import dense_ref as DR
import scatter_ref as SR
from oracle import lidar4d_oracle as O
from parity_util import small_config, make_surface_like, cuda_model_from_oracle, test_rays as _rays
from saved_util import train_step, saved_features

pytestmark = pytest.mark.gpu
MODES = ("tc", "fp32")
GRADS = ("sigma_net.params", "intensity_net.params", "raydrop_net.params", "flow_net.mlp.0.weight",
         "flow_net.mlp.2.weight", "flow_net.mlp.4.weight")
MAX_AMBIGUOUS = 1e-2            # fraction of samples with a sigma- or flow-MLP unit within its bound of the kink
MAX_AMBIGUOUS_ATTR = 0.3        # fraction of live samples with an attribute-net unit within its bound (measured: <= 23 %)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def upstream(pattern: str, N: int, S: int, dev, seed: int = 23, quiet: int = 0):
    """Upstream gradients; the first `quiet` rays get none on any term (their tiles carry no gradient at all)."""
    g = torch.Generator().manual_seed(seed)
    U = {"depth_lidar": torch.randn(N, generator=g), "image_lidar": torch.randn(N, 2, generator=g),
         "weights_sum_lidar": torch.randn(N, generator=g) * 0.1, "weights": torch.randn(N, S, generator=g) * 0.01}
    if pattern == "image":
        U = {"image_lidar": U["image_lidar"]}
    elif pattern == "x65536":
        U = {k: v * 65536.0 for k, v in U.items()}
    elif pattern.startswith("x2^-"):
        U = {k: v * 2.0 ** -int(pattern[4:]) for k, v in U.items()}
    for v in U.values():
        v[:quiet] = 0.0
    return {k: v.to(dev) for k, v in U.items()}


def assert_dense_exact(m, ro, rd, S, U, mode, monkeypatch, what, t=0.4, prefill=None):
    """Render + backward, then every output of the MLP stages against tests/dense_ref.py.  Returns the live mask [N, S],
    the largest log2(sc r) of the tensor-core sigma backward's delta tiles and the number of flat 128-sample flow tiles
    without dL/dflow."""
    dev = torch.device("cuda:0")
    cfg = m.cfg
    N = ro.shape[0]
    tc = mode == "tc"
    t0 = time.perf_counter()
    out, saved = train_step(m, ro, rd, S, U, monkeypatch, t=t, keep_flow_in=True, prefill=prefill)
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if k in GRADS}
    L = SR.saved_layout(cfg, N, S)
    sigma = saved[L["sigma"]:L["sigma"] + 4 * N * S].view(torch.float32).view(N, S)
    attr = saved[L["attr"]:L["attr"] + 8 * N * S].view(torch.float32).view(2, N, S)
    sd = float(np.float32((np.float32(cfg.far_lidar) - np.float32(cfg.near_lidar)) / np.float32(S)))
    cref = CR.composite(sigma, attr, out["z_vals"], sd, cfg.density_scale, cfg.active_sensor, U)
    live = (attr != 0).any(0)
    up = DR.compositing_inputs(cref, U, live, CR.weight_bound(cref), CR.dsigma_bound(cref))
    W = DR.working_weights(cfg, {k: p.detach() for k, p in m.named_parameters()}, tc)
    enc, enc_e = DR.direction_encoding(rd.to(dev))
    sv = SR.decode_saved(cfg, saved, N, S)
    worst, at = {}, {}

    def hold(name, got, v, b, p0=0):
        r = DR.ratio(got, v, b)
        i = int(torch.argmax(r))
        if float(r.reshape(-1)[i]) >= worst.get(name, -1.0):
            worst[name] = float(r.reshape(-1)[i])
            at[name] = (p0, i, float(got.double().reshape(-1)[i]), float(v.reshape(-1)[i]), float(b.reshape(-1)[i]))

    def on_dense(p0, p1, o):
        hold("sigma", sigma.reshape(-1)[p0:p1], *o["sigma"], p0)
        hold("attr", attr.reshape(2, -1)[:, p0:p1], *o["attr"], p0)
        hold("dfeat", sv["dfeat"][p0:p1], *o["dfeat"], p0)

    def on_flow(p0, p1, o):
        hold("flow", sv["flow"][:, p0:p1].t(), *o["flow"], p0)
        if tc:                                   # the backward wrote dL/d(flow-MLP input) over flow_in
            hold("dfin", sv["flow_in"][:, p0:p1].t(), *o["dfin"], p0)
    ref = DR.dense_reference(cfg, W, saved_features(cfg, saved, N, S, mode), N, S, enc, enc_e, live.reshape(-1), up, tc,
                             on_dense)
    fref = DR.flow_reference(W, out["flow_in"], sv["dflow"], tc, on_flow)
    for k in GRADS:
        v, b = (ref if k in ref else fref)[k]
        got = grads[k].double().reshape(-1)
        if prefill is not None:
            got = got - prefill[k].double().reshape(-1)
            b = b.reshape(-1) + DR.EPS32 * grads[k].double().abs().reshape(-1)      # the one rounding of the fold into .grad
        hold(k, got, v.reshape(-1), b.reshape(-1))
    amb, n_live = ref["ambiguous"] + fref["ambiguous"], int(live.sum())
    bad = {k: f"{v:.3g} x bound at {at[k]}" for k, v in worst.items() if not v <= 1.0}
    assert not bad, f"{what}: {bad}"
    assert amb <= MAX_AMBIGUOUS * N * S, f"{what}: {amb} of {N * S} samples with an ambiguous sigma- or flow-MLP unit"
    assert ref["ambiguous_attr"] <= MAX_AMBIGUOUS_ATTR * n_live, \
        f"{what}: {ref['ambiguous_attr']} of {n_live} live samples with an ambiguous attribute-net unit"
    P = N * S
    quiet_tiles = int((sv["dflow"][:, :P // 128 * 128].reshape(6, -1, 128) == 0).all(2).all(0).sum())
    print(f"[dense-exact] {what}: " + " ".join(f"{k.replace('.params', '').replace('_net', '')} {v:.2e}"
                                               for k, v in worst.items())
          + f"; ambiguous: {amb} of {N * S} samples, attribute nets {ref['ambiguous_attr']} of {n_live} live; "
            + (f"max log2(sc r) {ref['max_log2_scale']:.0f}; " if tc else "")
            + f"{quiet_tiles} flow tiles without dL/dflow; {time.perf_counter() - t0:.1f} s")
    return dict(live=live, max_log2_scale=ref["max_log2_scale"], quiet_flow_tiles=quiet_tiles)


# ---- a. the benchmark configuration ---------------------------------------------------------------------------------------
def n_wrap() -> int:
    return 2 * 16 * torch.cuda.get_device_properties(0).multi_processor_count + 37


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


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("frame,t", [(25, 0.5), (0, 0.0)], ids=["interior", "first"])
def test_benchmark_config(dev, monkeypatch, mode, frame, t):
    from lidar4d_b200.rays import synthetic_sweep
    N, S = n_wrap(), 768
    ro, rd, _ = synthetic_sweep(frame)
    sel = np.linspace(0, ro.shape[0] - 1, N).astype(np.int64)
    ro, rd = torch.from_numpy(ro[sel]).contiguous(), torch.from_numpy(rd[sel]).contiguous()
    m = full_model(mode)
    assert m.cfg.sigma_in_pad == 176 and m.cfg.sigma_in_dim == 176
    assert_dense_exact(m, ro, rd, S, upstream("all", N, S, dev), mode, monkeypatch, f"L16 S768 {mode} frame {frame}", t=t)


# ---- b. ones columns, partial tiles, masters off the fp16 grid --------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("S", [2, 129, 333])
@pytest.mark.parametrize("L", [3, 8, 9, 10])
def test_small_configs(dev, monkeypatch, mode, L, S):
    """296 rays: the tensor-core dense kernels (one CTA per SM) wrap their persistent grid here too.  The first two rays
    get no upstream gradient, so at S >= 129 whole flat 128-sample flow tiles carry no dL/dflow: the flow backward skips
    them and must write exact zeros to dL/d(flow-MLP input)."""
    orc = O.build_seeded(small_config(n_levels_hash=L), 3, flow_last_std=0.02)      # masters not snapped to fp16
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 3
    K, ip = m.cfg.sigma_in_dim, m.cfg.sigma_in_pad
    assert K == 64 + 7 * L and ip == (K + 15) // 16 * 16
    p = m.sigma_net.params.detach().float()
    assert not bool((p.half().float() == p).all()), "masters already on the fp16 grid"
    ro, rd = _rays(8, 37)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    st = assert_dense_exact(m, ro, rd, S, upstream("all", ro.shape[0], S, dev, quiet=2), mode, monkeypatch,
                            f"L{L} (K {K}, in_pad {ip}) S{S} {mode}")
    assert S < 128 or st["quiet_flow_tiles"] > 0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("S", [2, 129])
def test_one_ray(dev, monkeypatch, mode, S):
    orc = O.build_seeded(small_config(n_levels_hash=8), 7, flow_last_std=0.02)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 7
    ro, rd = _rays(3, 8)
    ro, rd = torch.from_numpy(ro[5:6]).contiguous(), torch.from_numpy(rd[5:6]).contiguous()
    assert_dense_exact(m, ro, rd, S, upstream("all", 1, S, dev), mode, monkeypatch, f"one ray S{S} {mode}")


# ---- c. density regimes and upstream gradients ---------------------------------------------------------------------------
REGIMES = {"transparent": dict(density_scale=0.02), "opaque": dict(density_scale=200.0), "active": dict(active_sensor=True)}
PATTERNS = ("all", "image", "x65536", "x2^-20")


def regime_model(regime: str, mode: str, seed: int = 3):
    orc = O.build_seeded(small_config(**REGIMES.get(regime, {})), seed, flow_last_std=0.02)
    O.snap_mlp_weights_fp16(orc)
    if regime == "opaque":
        make_surface_like(orc)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = seed
    return m


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("regime", list(REGIMES))
def test_regimes_and_upstream(dev, monkeypatch, mode, regime):
    S = 256
    m = regime_model(regime, mode)
    ro, rd = _rays(8, 37)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    N = ro.shape[0]
    st = {p: assert_dense_exact(m, ro, rd, S, upstream(p, N, S, dev), mode, monkeypatch, f"{regime} {p} {mode}")
          for p in PATTERNS}
    if regime == "opaque":           # rays partly inside the attribute mask: the surface inside, the samples behind it out
        n_in = st["all"]["live"].sum(1)
        assert bool(((n_in > 0) & (n_in < S)).any()), "no ray partly inside the attribute mask"



@pytest.mark.parametrize("mode", MODES)
def test_delta_scales_past_2_128(dev, monkeypatch, mode):
    """The opaque regime's tiles behind the surface carry dL/dσ of exactly 0 (the transmittance underflows), so their
    scales stay small; here every tile of the launch is tiny, and the sigma backward undoes scales beyond 2^128."""
    S = 256
    m = regime_model("transparent", mode)
    ro, rd = _rays(8, 37)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    top = max(assert_dense_exact(m, ro, rd, S, upstream(p, ro.shape[0], S, dev), mode, monkeypatch,
                                 f"transparent {p} {mode}")["max_log2_scale"] for p in ("x2^-110", "x2^-120"))
    assert mode != "tc" or top >= 130, f"largest sc r of the sigma backward 2^{top:.0f}"


# ---- d. the attribute mask -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_outside_attribute_mask(dev, monkeypatch, mode):
    """density_scale 1e-7: every weight lies below 1e-4, the attribute heads never run, and their gradients must be
    exactly 0 (the reference's bound is 0 there)."""
    orc = O.build_seeded(small_config(density_scale=1e-7), 3, flow_last_std=0.02)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 3
    ro, rd = _rays(3, 8)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    S = 129
    st = assert_dense_exact(m, ro, rd, S, upstream("all", ro.shape[0], S, dev), mode, monkeypatch,
                            f"outside the mask {mode}")
    assert not bool(st["live"].any())
    for k in ("intensity_net.params", "raydrop_net.params"):
        assert float(dict(m.named_parameters())[k].grad.abs().max()) == 0.0, k


# ---- e. accumulation into gradients that hold values -------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_accumulates_into_existing_gradients(dev, monkeypatch, mode):
    orc = O.build_seeded(small_config(n_levels_hash=8), 5, flow_last_std=0.02)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.jitter_seed = 5
    ro, rd = _rays(8, 37)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    S = 129
    U = upstream("all", ro.shape[0], S, dev)
    train_step(m, ro, rd, S, U, monkeypatch)
    g = torch.Generator().manual_seed(9)
    prefill = {k: (torch.randn(p.shape, generator=g) * float(p.grad.abs().max())).float().to(dev)
               for k, p in m.named_parameters() if k in GRADS}
    assert_dense_exact(m, ro, rd, S, U, mode, monkeypatch, f"prefilled gradients {mode}", prefill=prefill)
