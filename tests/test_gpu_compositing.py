"""GPU: the compositing of every render pipeline, sample by sample, against a float64 evaluation of its own inputs.

The compositing (σ -> α, T, weights -> depth, image, Σw; backward: dL/dσ) makes no decision other than the attribute mask,
so given what it consumed - the σ and the attributes a training forward saves, z (bit-exact against the reference, see
test_gpu_launch_scale.py) - tests/compositing_ref.py evaluates it exactly, and every output is held to a bound derived
there from the operations the kernels perform, valid for any association order of their scans:

    weights:             |w_j - ŵ_j| <= RHO_W_j 2^-24 ŵ_j (+ a subnormal floor),  RHO_W_j <= 9 j + 7 while α <= 1/2
    depth, image, Σw:    |got - ref| <= Σ_j (RHO_W_j + S + 2) 2^-24 |t_j|          t_j = ŵ_j z_j, ŵ_j attr_j, ŵ_j
    attributes:          exactly 0 where ŵ_j <= 1e-4 and > 0 above it (samples within the weight bound of 1e-4 skipped)
    dL/dσ (split):       |got - ref| <= (RHO_END + S + 16) 2^-24 A_j + the projection's own rounding (below)

A float32 α formed as 1 - expf(e) misses the first bound by orders of magnitude wherever α is small (at α = 5e-6 one ulp
of expf near 1 is 1.2e-2 of α), however short the ray.

dL/dσ is not stored: the split pipelines' backward writes dL/dfeature, which with g_image = 0 (no gradient reaches the
attribute heads, so none reaches the geo features) is dL/dσ_j exp(clamp(h0_j, -15, 15)) J_j, J_j the sigma MLP's input
Jacobian of its σ output, J_k = Σ_h W2[0, h] [hidden_h > 0] W1[h, k].  J is evaluated in float64 on the kernel's own saved
features (fp16 hi + lo in tensor-core mode) and fp16-exact weights, dL/dσ recovered by projecting dL/dfeature on J, and
samples with a hidden unit within 2^-12 of its pre-activation's magnitude of the ReLU kink are skipped.  The projection
adds 128 2^-24 |dL/dσ| <Ĵ, |J|> / <J, J> (Ĵ_k = Σ_h |W2[0, h] W1[h, k]| over the live units): the fp16 hi|lo splits and
the 64-term sums of the two matrix products.  In tensor-core mode the delta tiles are fp16 hi|lo scaled by a power of
two per tile (amax to [32, 64)), which resolves a tile to ~2^-30 of its largest entry: there the bound adds
2^-20 <Ĵ, |J|> / <J, J> max_tile |dL/dσ exp(h0)| / exp(h0_j) (2^10 for the second scaled tile and the 64-term sums).
The fused pipeline writes no dL/dfeature; its backward stays covered end
to end (test_gpu_launch_scale.py, test_gpu_parity.py).

Cases: tc-split, fp32-split, fused; S at tile edges from 2 to 8192; density regimes transparent (density_scale 0.02),
default, opaque (surface-like σ at density_scale 200: α == 1 in float32, T underflowing to 0, the + 1e-15 and suf / v
paths) and active_sensor; upstream gradients with every term, Σw only, depth only, per-sample weights only, and all
terms times 65536.  In tensor-core mode, tiles behind an opaque surface carry dL/dσ of 0 or of ~1e-35 next to entries of
~1, through the per-tile power-of-two scales of the delta tiles."""
import numpy as np
import pytest
import torch

import compositing_ref as CR
import scatter_ref as SR
from oracle import lidar4d_oracle as O
from parity_util import small_config, make_surface_like, cuda_model_from_oracle, test_rays as _rays
from saved_util import train_step, saved_features

pytestmark = pytest.mark.gpu
MODES = [("tc", "split"), ("fp32", "split"), ("tc", "fused")]
MODE_IDS = ["tc-split", "fp32-split", "fused"]
S_LIST = [2, 127, 128, 129, 255, 256, 257, 1024, 8191, 8192]
REGIMES = {"transparent": dict(density_scale=0.02), "default": dict(), "opaque": dict(density_scale=200.0),
           "active": dict(active_sensor=True)}
PATTERNS = ("all", "wsum", "depth", "weights", "x65536")
RELU_MARGIN = 2.0 ** -12
PROJ_SLACK = 128.0
TC_RES = 2.0 ** -20


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def upstream(pattern: str, N: int, S: int, dev):
    """Upstream gradients without an image term (see the module docstring), except in `all`."""
    g = torch.Generator().manual_seed(17)
    U = {"depth_lidar": torch.randn(N, generator=g), "image_lidar": torch.randn(N, 2, generator=g),
         "weights_sum_lidar": torch.randn(N, generator=g), "weights": torch.randn(N, S, generator=g) * 0.01}
    if pattern == "wsum":
        U = {"weights_sum_lidar": U["weights_sum_lidar"]}
    elif pattern == "depth":
        U = {"depth_lidar": U["depth_lidar"]}
    elif pattern == "weights":
        U = {"weights": U["weights"]}
    elif pattern == "x65536":
        U = {k: v * 65536.0 for k, v in U.items() if k != "image_lidar"}
    return {k: v.to(dev) for k, v in U.items()}


def model_for(regime: str, mode: str, pipeline: str):
    orc = O.build_seeded(small_config(**REGIMES[regime]), 3, flow_last_std=0.02)
    O.snap_mlp_weights_fp16(orc)
    if regime == "opaque":
        make_surface_like(orc)
    m = cuda_model_from_oracle(orc).set_mlp_fp16(mode == "tc")
    m.pipeline = pipeline
    m.jitter_seed = 3
    return m


def sigma_jacobian(m, feat: torch.Tensor):
    """J [P, K], Ĵ [P, K] and the usable-sample mask (every hidden unit clear of its ReLU kink), float64."""
    cfg = m.cfg
    K, ip = cfg.sigma_in_dim, cfg.sigma_in_pad
    p = m.sigma_net.params.detach().double()
    W1 = p[:64 * ip].view(64, ip)
    w2 = p[64 * ip:64 * ip + 64]                                     # output row 0 (σ) of W2 [16, 64]
    x = feat.double()
    hid = x @ W1[:, :K].t() + W1[:, K:].sum(1)[None]
    mag = x.abs() @ W1[:, :K].abs().t() + W1[:, K:].abs().sum(1)[None]
    live = (hid > 0).double() * w2[None]
    J = live @ W1[:, :K]
    Jh = live.abs() @ W1[:, :K].abs()
    ok = ((hid.abs() > RELU_MARGIN * mag) | (w2 == 0)[None]).all(1)
    return J, Jh, ok


def check_forward(out, ref, attr, what):
    N, S = ref["weights"].shape
    w = out["weights"].double()
    wb = CR.weight_bound(ref)
    ratio = float(((w - ref["weights"]).abs() / wb).max())
    z = out["z_vals"].double()
    sums = {"depth": (out["depth_lidar"].double().reshape(N), ref["depth"], ref["weights"] * z),
            "image0": (out["image_lidar"].double().reshape(N, 2)[:, 0], ref["image"][:, 0], ref["weights"] * attr[0]),
            "image1": (out["image_lidar"].double().reshape(N, 2)[:, 1], ref["image"][:, 1], ref["weights"] * attr[1]),
            "wsum": (out["weights_sum_lidar"].double().reshape(N), ref["wsum"], ref["weights"])}
    sratio = {k: float(((g - r).abs() / CR.sum_bound(ref, t)).max()) for k, (g, r, t) in sums.items()}
    clear = (ref["weights"] - CR.MASK_THRESHOLD).abs() > wb
    live = attr != 0
    bad_mask = int(((live[0] != ref["mask"]) & clear).sum() + ((live[1] != ref["mask"]) & clear).sum())
    wmax = float(ref["weights"].abs().max())
    rel = {"weights": float((w - ref["weights"]).abs().max()) / wmax,
           "depth": float((sums["depth"][0] - sums["depth"][1]).abs().max()) / float(sums["depth"][1].abs().max())}
    assert ratio <= 1.0 and max(sratio.values()) <= 1.0 and bad_mask == 0, \
        (what, f"weights {ratio:.3g} x bound", {k: f"{v:.3g}" for k, v in sratio.items()}, f"{bad_mask} mask decisions",
         f"rel. to max: weights {rel['weights']:.2e} depth {rel['depth']:.2e}")
    return ratio, max(sratio.values()), rel


def check_backward(m, sv_dfeat, J, Jh, ok, ref, sigma, mode, what):
    """Projected dL/dσ of the split pipelines against the reference; returns (worst fraction of the bound, samples)."""
    N, S = ref["weights"].shape
    JJ = (J * J).sum(1)
    use = ok & (JJ > 0)
    d = sv_dfeat.double()
    sp = sigma.double().reshape(-1).clamp(float(np.exp(-15.0)), float(np.exp(15.0)))
    got = (d * J).sum(1) / JJ.clamp_min(1e-300) / sp
    exact = ref["dsigma"].reshape(-1)
    kappa = (Jh * J.abs()).sum(1) / JJ.clamp_min(1e-300)
    bound = CR.dsigma_bound(ref).reshape(-1) + (PROJ_SLACK * kappa + 4.0) * CR.EPS32 * exact.abs()
    if mode == "tc":                # fp16 hi|lo resolves a tile to ~2^-30 of its largest dL/dσ exp(h0)
        ds = (exact * sp).abs().view(N, S)
        nt = (S + 127) // 128
        amax = torch.nn.functional.pad(ds, (0, nt * 128 - S)).view(N, nt, 128).amax(-1)
        amax = amax.repeat_interleave(128, -1)[:, :S].reshape(-1)
        bound = bound + TC_RES * kappa * amax / sp
    err = (got - exact).abs()
    r = torch.where(use, err / bound, torch.zeros_like(err))
    worst = int(torch.argmax(r))
    assert float(r[worst]) <= 1.0, (what, f"sample {worst} (j = {worst % S}): got {float(got[worst]):.6e} "
                                          f"ref {float(exact[worst]):.6e} bound {float(bound[worst]):.3e} "
                                          f"A {float(ref['A'].reshape(-1)[worst]):.3e}", f"{int((r > 1).sum())} samples over")
    return float(r[worst]), int(use.sum())


@pytest.mark.parametrize("mode,pipeline", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("S", S_LIST)
def test_compositing_against_own_inputs(dev, monkeypatch, S, regime, mode, pipeline):
    m = model_for(regime, mode, pipeline)
    cfg = m.cfg
    ro, rd = _rays(3, 8)
    ro, rd = torch.from_numpy(ro), torch.from_numpy(rd)
    N = ro.shape[0]
    sd = float(np.float32((np.float32(cfg.far_lidar) - np.float32(cfg.near_lidar)) / np.float32(S)))
    worst_b, n_b, stats = 0.0, 0, None
    for pattern in PATTERNS:
        U = upstream(pattern, N, S, dev)
        out, saved = train_step(m, ro, rd, S, U, monkeypatch)
        L = SR.saved_layout(cfg, N, S)
        sigma = saved[L["sigma"]:L["sigma"] + 4 * N * S].view(torch.float32).view(N, S)
        attr = saved[L["attr"]:L["attr"] + 8 * N * S].view(torch.float32).view(2, N, S).double()
        ref = CR.composite(sigma, attr, out["z_vals"], sd, cfg.density_scale, cfg.active_sensor, U)
        what = f"{mode}/{pipeline} S={S} {regime} {pattern}"
        if stats is None:                            # the forward does not depend on the upstream gradients
            stats = check_forward(out, ref, attr, what)
            if regime == "opaque":                   # α == 1 in float32 up to S = 1024, T below float32's range from S = 127
                assert S > 1024 or bool((ref["alpha"].float() == 1.0).any()), "no sample with α == 1"
                assert S < 127 or bool((ref["T"] < 2.0 ** -149).any()), "no transmittance underflow"
            if regime == "transparent":
                assert float(ref["T"][:, -1].min()) > 0.1, "not transparent"
        if pipeline == "split" and "image_lidar" not in U:
            sv = SR.decode_saved(cfg, saved, N, S)
            if pattern == "wsum":                    # the Jacobian depends on the forward only
                J, Jh, ok = sigma_jacobian(m, saved_features(cfg, saved, N, S, mode))
            r, n = check_backward(m, sv["dfeat"], J, Jh, ok, ref, sigma, mode, what)
            assert n >= 0.8 * N * S, (what, f"dL/dσ checked on {n} of {N * S} samples")
            worst_b, n_b = max(worst_b, r), max(n_b, n)
    print(f"[compositing] {mode}/{pipeline} S={S} {regime}: weights {stats[0]:.3f} and sums {stats[1]:.3f} of their "
          f"bounds, rel. to max weights {stats[2]['weights']:.1e} depth {stats[2]['depth']:.1e}"
          + (f"; dL/dσ {worst_b:.3f} of its bound on {n_b} of {N * S} samples" if pipeline == "split" else ""))
