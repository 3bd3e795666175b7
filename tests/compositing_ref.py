"""Float64 reference of the render path's compositing stage (test infrastructure).

Given what the compositing consumed - σ [N, S], the attribute heads' outputs [2, N, S] (0 outside the attribute mask, as
the kernels save them), z [N, S] and the launch constants - the compositing (renderer.py:98-129) is a smooth function:

    δ_j = z_{j+1} - z_j (float32, as the kernels and the reference; the last δ is sample_dist)
    e_j = -k δ_j density_scale σ_j          k = 2 with active_sensor, else 1
    α_j = 1 - exp(e_j),  v_j = (1 - α_j) + 1e-15,  T_j = prod_{i<j} v_i,  w_j = α_j T_j
    depth = Σ w z,  image = Σ w attr,  Σw,  mask = w > 1e-4

and its backward, with upstream gradients g_depth [N], g_image [N, 2], g_wsum [N], g_weights [N, S]:

    g_j = g_depth z_j + g_image · attr_j + g_wsum + g_weights_j                     dL/dw_j
    dL/dσ_j = k δ_j density_scale (1 - α_j) (g_j T_j - Σ_{i>j} g_i w_i / v_j)
    dL/dattr_{c,j} = g_image_c w_j where the sample is inside the mask, else 0.

Everything after δ is float64 here, with α = -expm1(e) and 1 - α = exp(e): no cancellation anywhere, so these are the
exact values of the function of the given inputs to ~1e-15.

Error bounds (u = 2^-24).  A float32 evaluation in any association order of the scans, whose per-sample arithmetic is

    e:  two roundings (the factor 2 of active_sensor is exact)            relative error <= 2u
    α = -expm1f(e): <= 2 ulp (CUDA's documented bound is 1), <= 4u, plus the e error carried through
        (|dα/de| |e| / α = |e| e^e / (1 - e^e) <= 1)                        relative error <= C_ALPHA u = 6u
    v = (1 - α) + 1e-15: two roundings plus the α error seen relative to v      <= (2 + C_ALPHA α/v) u
    T_j: a product of j factors v_i and the carry 1 in any association order   <= j roundings
    w_j = α_j T_j: one rounding

satisfies, to first order in u,

    |w_j - ŵ_j| <= RHO_W_j u ŵ_j + TINY_j,  RHO_W_j = Σ_{i<j} (3 + C_ALPHA α_i / v_i) + C_ALPHA + 1,

with TINY_j = (j + 2) 2^-149 for products that pass through float32's subnormal range (each rounding there is absolute,
<= 2^-150).  Where every α_i <= 1/2 (α/v <= 1) RHO_W_j <= a j + b with a = 3 + C_ALPHA = 9, b = C_ALPHA + 1 = 7; behind
a sample with α near 1 the factor α/v grows as the float32 1 - α loses its bits, and the bound grows with it: there the
float32 function itself (the reference's `1 - alphas + 1e-15` included) is ill-conditioned.  A sum Σ_j t_j of n terms
(depth, image, Σw) whose terms carry relative errors RHO_W_j u is off by at most Σ_j (RHO_W_j + n + C_SUM) u |t_j| + Σ_j TINY_j
|t_j / w_j|, C_SUM = 2 (the product w z and the float32 rounding of z - attributes are taken as given).

The backward: dL/dσ_j is a difference of two terms, each within (RHO_END + n + C_BWD) u of its magnitude, where RHO_END
is the largest RHO_W of the ray (the suffix sum runs over every later weight) and C_BWD = 16 covers g_j (five terms),
the division by v, (1 - α) and the three-factor scale.  Its magnitude scale is

    A_j = k density_scale δ_j (|g|_j T_{j+1} + Σ_{i>j} |g|_i w_i),   |g|_j = Σ of the magnitudes of g_j's terms,

not |dL/dσ_j|: with only a Σw gradient the exact value is k ds δ_j g (T_end - T_{j+1}) - tiny behind an opaque surface -
and any float32 evaluation forms it as a difference of two O(1) numbers."""
from __future__ import annotations

import torch

EPS32 = 2.0 ** -24
C_ALPHA = 6.0
C_SUM = 2.0
C_BWD = 16.0
MASK_THRESHOLD = 1e-4


def deltas32(z: torch.Tensor, sample_dist: float) -> torch.Tensor:
    """δ in float32 exactly as the kernels and the reference form it: z_{j+1} - z_j, then sample_dist."""
    z = z.float()
    last = torch.full_like(z[:, :1], float(torch.tensor(sample_dist, dtype=torch.float32)))
    return torch.cat([z[:, 1:] - z[:, :-1], last], -1)


def composite(sigma, attr, z, sample_dist: float, density_scale: float, active_sensor: bool, U: dict = None) -> dict:
    """Float64 compositing of the given inputs.

    sigma [N, S], attr [2, N, S], z [N, S] (float32 values); U: the upstream gradients (keys depth_lidar [N],
    image_lidar [N, 2], weights_sum_lidar [N], weights [N, S]; missing keys are zero) or None.
    Returns float64 tensors: alpha, T, weights [N, S], depth [N], image [N, 2], wsum [N], mask [N, S] (bool), and the
    bound magnitudes rho_w [N, S] (RHO_W above), tiny [N, S]; with U also g [N, S] (dL/dw), dsigma [N, S],
    dattr [2, N, S], A [N, S], A_tiny [N, S] (A's subnormal floor) and rho_end [N]."""
    dev = sigma.device
    N, S = sigma.shape
    k = 2.0 if active_sensor else 1.0
    d32 = deltas32(z, sample_dist)
    d = d32.double()
    zz = z.double()
    s = sigma.double()
    at = attr.double()
    e = -k * d * float(density_scale) * s
    alpha = -torch.expm1(e)
    keep = torch.exp(e)                                        # 1 - α without cancellation
    v = keep + 1e-15
    T = torch.cat([torch.ones_like(v[:, :1]), torch.cumprod(v, -1)[:, :-1]], -1)
    w = alpha * T
    out = dict(alpha=alpha, T=T, weights=w, depth=(w * zz).sum(-1), image=(w[None] * at).sum(-1).t(),
               wsum=w.sum(-1), mask=w > MASK_THRESHOLD)
    per = 3.0 + C_ALPHA * alpha / v
    rho_T = torch.cat([torch.zeros_like(per[:, :1]), torch.cumsum(per, -1)[:, :-1]], -1)
    out["rho_w"] = rho_T + C_ALPHA + 1.0
    out["tiny"] = (torch.arange(S, device=dev, dtype=torch.float64)[None] + 2.0).expand(N, S) * 2.0 ** -149
    if U is None:
        return out
    z0 = torch.zeros(N, dtype=torch.float64, device=dev)
    gd = U["depth_lidar"].double().reshape(N) if "depth_lidar" in U else z0
    gi = U["image_lidar"].double().reshape(N, 2) if "image_lidar" in U else torch.zeros(N, 2, dtype=torch.float64, device=dev)
    gs = U["weights_sum_lidar"].double().reshape(N) if "weights_sum_lidar" in U else z0
    gW = U["weights"].double().reshape(N, S) if "weights" in U else torch.zeros_like(w)
    g = gd[:, None] * zz + gi[:, 0, None] * at[0] + gi[:, 1, None] * at[1] + gs[:, None] + gW
    ga = (gd[:, None] * zz).abs() + (gi[:, 0, None] * at[0]).abs() + (gi[:, 1, None] * at[1]).abs() + gs.abs()[:, None] + gW.abs()

    def excl_suffix(x):
        c = torch.flip(torch.cumsum(torch.flip(x, [-1]), -1), [-1])
        return torch.cat([c[:, 1:], torch.zeros_like(c[:, :1])], -1)

    suf = excl_suffix(g * w)
    sufa = excl_suffix(ga * w)
    scale = k * float(density_scale) * d
    out["g"] = g
    out["dsigma"] = scale * (g * T * keep - suf * (keep / v))
    out["A"] = scale * (ga * T * keep + sufa)
    out["A_tiny"] = scale * (ga + excl_suffix(ga)) * out["tiny"]
    out["dattr"] = torch.stack([gi[:, 0, None] * w, gi[:, 1, None] * w]) * out["mask"][None]
    out["rho_end"] = out["rho_w"].max(-1).values
    return out


def weight_bound(ref: dict) -> torch.Tensor:
    """Per-sample bound on |w - ŵ|."""
    return ref["rho_w"] * EPS32 * ref["weights"] + ref["tiny"]


def sum_bound(ref: dict, terms: torch.Tensor) -> torch.Tensor:
    """Bound on |Σ_j t_j - Σ_j t̂_j| over the last axis, t̂_j = ŵ_j x_j given as `terms` [..., S]."""
    S = terms.shape[-1]
    w = ref["weights"]
    ratio = torch.where(w > 0, terms.abs() / w.clamp_min(1e-300), torch.zeros_like(w))
    return ((ref["rho_w"] + S + C_SUM) * EPS32 * terms.abs() + ref["tiny"] * ratio).sum(-1)


def dsigma_bound(ref: dict) -> torch.Tensor:
    """Per-sample bound on |dL/dσ - its reference|."""
    S = ref["weights"].shape[-1]
    return (ref["rho_end"][:, None] + S + C_BWD) * EPS32 * ref["A"] + 4 * ref["A_tiny"]
