"""Float64 reference of the split pipeline's MLP stages, with a per-entry error bound (test infrastructure).

Given what the dense kernels consumed - the sigma MLP's input X [P, K] as the training forward saved it (fp32 SoA, or the
fp16 hi + lo operand tiles the tensor cores read), the direction of every ray, the attribute mask the forward decided
(saved attr != 0), the MLP weights as the kernels hold them (fp16(master) in tensor-core mode, the fp32 masters in fp32
mode), dL/dσ and dL/dattr of the compositing, the flow MLP's input and the upstream dL/dflow - the MLPs are a
piecewise-linear function of those inputs, apart from exp and sigmoid.  This module evaluates it in float64:

    sigma MLP      h = relu(W1 [x, 1..1]),  o = W2 h,  σ = exp(o_0),  geo = o_1..15
    attribute nets a_in = [enc(d), geo, 1 x 9],  h1 = relu(Wa1 a_in),  h2 = relu(Wa2 h1),  attr = sigmoid(Wa3_0 · h2)
                   (samples inside the attribute mask only; attr is 0 elsewhere)
    flow MLP       flow = F2 relu(F1 relu(F0 fin))

and their backward: dL/dlogit = dL/dattr a (1 - a), dL/do_0 = dL/dσ exp(clamp(o_0, -15, 15)), dL/dgeo from both attribute
nets, dL/dX = W1^T dh (the kernels' dL/dfeature), dL/dfin = F0^T dh1 (written over flow_in in tensor-core mode), and every
weight gradient as the sum over the launch's samples of an outer product.

Error bound.  Every value v comes with an absolute error bound E that holds, to first order in u = 2^-24, for any float32
evaluation in any association order that makes the same ReLU decisions.  It is a running error bound: each operation
adds the rounding of its own operands, whose magnitudes are at most |v| + E, and carries the errors of its inputs:

    layer y = W a (n inputs)  E_y = |W| E_a + (n + C_LAYER) u |W| (|a| + E_a)     the n roundings of the inner product;
                                                                                   C_LAYER = 8 for the epilogue and, in
                                                                                   tensor-core mode, the hi|lo split of
                                                                                   the activation operand (2^-22 = 4u)
    relu                      E_h = E_y where the unit is on or ambiguous, else 0 (relu is 1-Lipschitz; a unit decided
                              off is exactly 0)
    delta g = W^T d, masked   E_g = |W|^T E_d + (n + C_LAYER) u |W|^T (|d| + E_d) on live units; on an ambiguous unit the
                              kernel may pass g or 0, so E_g = |g| + E_g there
    σ = exp(o_0)              σ expm1(E_o) + 3u σ e^E_o            (expf: 2 ulp)
    attr = sigmoid(l)         a (1 - a) E_l e^E_l + 8u a             (1 / (1 + expf(-l)))
    direction encoding        sinf of the float32 argument (formed op by op as l4d_freq): 2 ulp, 4u |enc|
    weight gradient Σ_p d_p x_p
                              Σ_p (E_d m_x + m_d E_x) + (2 T_e + min(128, N_e) + C_SUM) u Σ_p m_d m_x,   m = |v| + E

where T_e and N_e are the numbers of 128-sample tiles and of samples with a contribution to the entry: the kernels sum a
tile's products in some order (wgmma over K = 128, or tile_outer_accum) and reduce the tiles' sums with atomics in any
order (the attribute nets' direction and ones rows per ray first, then over the rays); a tile without a contribution adds
an exact 0.  A dropped or doubled tile moves an entry by that tile's share, which the bound sees wherever a few tiles
dominate the entry (small launches, the attribute nets, the ones columns and rows); it does not see it in an entry
spread evenly over 25 k tiles.  A rounding in float32's subnormal range is absolute (<= 2^-150): every bound adds its
rounding count times 2^-149 where an operand is non-zero.  Float atomics on global memory flush subnormal operands and
results to zero, so each atomic of a weight gradient may move it by up to 2^-126: up to four per entry and tile
(tile_outer_accum splits a tile's samples over up to four warps) and one for the per-ray sums.

The point kernels (csrc/l4d_points.cuh, density_point_reference / attribute_point_reference / flow_reference(points=True))
reduce differently, and their rounding depth per entry is 4 T_e + min(128, N_e) + C_SUM (POINT_TILE_ROUNDINGS = 4):
  * tile_outer_accum over NT = 128 points and 4 warps: a product of K <= 16 rows gives each warp 32 points (an fma chain
    of <= 32) and issues 4 atomics per entry and tile, so depth <= 32 + 4 T_e; K = 24: <= 64 + 2 T_e; K = 64: <= 128 + T_e.
    With 2 T_e the first case is not covered once T_e > 56, hence 4 T_e here.
  * dW3 of the attribute nets: tile_colsum (a chain of <= 128) and one atomicAdd per tile: <= min(128, N_e) + T_e.
  * the 9 ones rows of the attribute nets: tile_colsum (<= 128), one add per tile into the thread's csum over the CTA's
    grid-stride loop, one atomicAdd per CTA: <= min(128, N_e) + 2 T_e.
The flush of subnormals stays ATOMICS_PER_TILE per tile (4 warp atomics + 1 per-CTA or per-tile colsum atomic).

Tensor-core mode adds, for every delta tile the kernels scale by a power of two and split into fp16 hi + lo, the
resolution of that tile: an entry is held to ~2^-30 of the tile's largest entry; the bound takes TC_RES = 2^-20 of it (the
same slack as tests/test_gpu_compositing.py).  The tiles are the dense kernels' 128-sample tiles of a ray and the flow
kernel's 128 flat samples (which straddle rays).

Ambiguous ReLUs.  A unit whose float64 pre-activation lies within its own bound E of 0 may be decided either way by a
correct float32 evaluation.  Its forward value is covered by the Lipschitz rule; in the backward the whole delta of the
unit is added to its bound, so the bound covers every output it reaches.  `ambiguous` counts the samples with such a unit;
the tests assert they are rare in the sigma and flow MLPs, so the bound stays meaningful without searching for seeds.  The
attribute nets are four and five layers deep behind the sigma MLP, and their second layer sums 64 inputs with heavy
cancellation (|y| ~ 1e-2 of Σ|W||a|), so there a worst-case bound leaves many units ambiguous (measured on the oracle's
small fixtures: ~20 % of live samples); their count is reported, and their gradients are held with those units' whole
deltas in the bound.

Inputs that are themselves results of float32 arithmetic carry their own bounds: dL/dσ (compositing_ref.dsigma_bound:
the dense backward runs the compositing backward in the same kernel) and dL/dattr = g_image w (the weight bound of
compositing_ref).  dL/dflow is taken as the kernels saved it (tests/test_gpu_scatter_exact.py holds it entry by entry)."""
from __future__ import annotations

import numpy as np
import torch

EPS32 = 2.0 ** -24
TINY = 2.0 ** -149
FTZ = 2.0 ** -126                # a float atomic on global memory flushes subnormals
ATOMICS_PER_TILE = 5.0           # tile_outer_accum splits a tile over up to 4 warps; + 1 for the per-ray row sums
C_LAYER = 8.0
C_SUM = 16.0
TC_RES = 2.0 ** -20
POINT_TILE_ROUNDINGS = 4.0      # the point kernels' rounding depth per contributing tile (module docstring)
CHUNK = 1 << 17                  # samples per pass (whole rays; keeps the float64 temporaries at a few hundred MB)
TILE = 128
ENC = 72                         # 3 dims x 12 frequencies x (sin, cos)
GEO = 15
HEADS = ("raydrop_net.params", "intensity_net.params")     # attribute channels 0 and 1 (the reference concatenates [drop, intensity])
PI32 = float(np.float32(np.pi))
HALF_PI32 = float(np.float32(np.pi / 2))


class V:
    """A float64 value and its absolute error bound E (tensors of one shape)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e):
        self.v, self.e = v, e

    def mag(self):
        """A bound on the magnitude of the float32 value."""
        return self.v.abs() + self.e


def exact(x: torch.Tensor) -> V:
    x = x.double()
    return V(x, torch.zeros_like(x))


def _round(m: torch.Tensor, n: float) -> torch.Tensor:
    """n roundings of a result whose operands' magnitudes sum to m: relative u, absolute 2^-149 in the subnormal range."""
    return n * (EPS32 * m + TINY * (m > 0))


# ---- weights ------------------------------------------------------------------------------------------------------------
def working_weights(cfg, params: dict, tc: bool) -> dict:
    """The MLP weights as the kernels compute with them, float64: fp16(master) in tensor-core mode (round to nearest, as
    the staging does), the fp32 masters otherwise.  params: reference state_dict name -> master tensor."""
    def w(name):
        p = params[name].detach().float()
        return (p.half() if tc else p).double()
    ip, ap = cfg.sigma_in_pad, cfg.attr_in_pad
    s = w("sigma_net.params")
    W = {"s1": s[:64 * ip].view(64, ip), "s2": s[64 * ip:].view(16, 64)}
    for net, name in enumerate(HEADS):
        a = w(name)
        W[f"a1_{net}"] = a[:64 * ap].view(64, ap)
        W[f"a2_{net}"] = a[64 * ap:64 * ap + 4096].view(64, 64)
        W[f"a3_{net}"] = a[64 * ap + 4096:].view(16, 64)
    for i, k in enumerate((0, 2, 4)):
        W[f"f{i}"] = w(f"flow_net.mlp.{k}.weight")
    return W


def direction_encoding(rays_d: torch.Tensor):
    """enc [N, 72] float64 of l4d_freq: the float32 argument ((d + 1) / 2 * 2^k * π_f + phase, op by op), its float64
    sine, and the bound of CUDA's sinf on it (2 ulp)."""
    d = rays_d.float()
    v = (d + 1.0) / 2.0
    cols = []
    for dim in range(3):
        for k in range(12):
            xs = v[:, dim] * float(1 << k)
            base = xs * PI32
            for ph in range(2):
                arg = base + (HALF_PI32 if ph else 0.0)
                cols.append(torch.sin(arg.double()))
    enc = torch.stack(cols, -1)
    return enc, 4.0 * EPS32 * enc.abs() + TINY


# ---- layers ---------------------------------------------------------------------------------------------------------------
def _lin(x: V, W: torch.Tensor, n: int) -> V:
    Wa = W.abs()
    return V(x.v @ W.t(), x.e @ Wa.t() + _round(x.mag() @ Wa.t(), n + C_LAYER))


def _relu(z: V):
    on = z.v > 0
    amb = (z.v.abs() <= z.e) & (z.e > 0)
    return V(z.v.clamp_min(0.0), torch.where(on | amb, z.e, torch.zeros_like(z.e))), on, amb


def _mask(g: V, on, amb) -> V:
    """The ReLU mask of a delta: an ambiguous unit passes g or 0."""
    return V(g.v * on, torch.where(amb, g.v.abs() + g.e, torch.where(on, g.e, torch.zeros_like(g.e))))


def _back(d: V, W: torch.Tensor, n: int, on=None, amb=None) -> V:
    """Delta through y = W a: W^T d, then the ReLU mask of a (if given)."""
    Wa = W.abs()
    g = V(d.v @ W, d.e @ Wa + _round(d.mag() @ Wa, n + C_LAYER))
    return g if on is None else _mask(g, on, amb)


def _tiles_dense(x: torch.Tensor, S: int) -> torch.Tensor:
    """Per sample [c] (c = whole rays of S samples): the largest x of its ray's 128-sample tile."""
    nr = x.shape[0] // S
    nt = (S + TILE - 1) // TILE
    t = torch.nn.functional.pad(x.view(nr, S), (0, nt * TILE - S)).view(nr, nt, TILE).amax(-1)
    return t.repeat_interleave(TILE, -1)[:, :S].reshape(-1)


def _tiles_flat(x: torch.Tensor) -> torch.Tensor:
    """Per sample [c] (c starting at a multiple of 128): the largest x of its flat 128-sample tile."""
    c = x.shape[0]
    nt = (c + TILE - 1) // TILE
    t = torch.nn.functional.pad(x, (0, nt * TILE - c)).view(nt, TILE).amax(-1)
    return t.repeat_interleave(TILE)[:c]


def pow2_log2(amax: torch.Tensor) -> torch.Tensor:
    """log2 of pow2_factor(amax) (l4d_dense_tc.cuh): the power of two that maps amax into [2^5, 2^6), capped at 2^126;
    0 where amax is 0 (the kernels leave such a tile unscaled)."""
    _, e = torch.frexp(amax)
    return torch.where(amax > 0, (6 - e).clamp(max=126).double(), torch.zeros_like(amax))


def _rescale(d: V, amax: torch.Tensor) -> V:
    """A delta tile stored as fp16 hi + lo after a power-of-two scale: + TC_RES of the tile's largest entry."""
    return V(d.v, d.e + TC_RES * amax[:, None])


def _row_amax(d: V) -> torch.Tensor:
    return d.mag().amax(1)


class _Grad:
    """One weight gradient Σ_p d_p ⊗ x_p: value, Σ of the products' magnitudes, propagated input error, and per entry the number of tiles
    and of samples that contribute to it (a tile without a contribution adds an exact 0)."""

    def __init__(self, shape, dev, per_tile: float = 2.0):
        self.per_tile = per_tile
        self.v = torch.zeros(shape, dtype=torch.float64, device=dev)
        self.a = torch.zeros_like(self.v)
        self.e = torch.zeros_like(self.v)
        self.n_tiles = torch.zeros_like(self.v)
        self.n_samples = torch.zeros_like(self.v)

    def add(self, d: V, x: V, tid: torch.Tensor):
        md, mx = d.mag(), x.mag()
        self.v += d.v.t() @ x.v
        self.a += md.t() @ mx
        self.e += d.e.t() @ mx + md.t() @ x.e
        nd, nx = (md > 0).double(), (mx > 0).double()
        self.n_samples += nd.t() @ nx
        nt = int(tid.max()) + 1
        td = torch.zeros(nt, nd.shape[1], dtype=torch.float64, device=nd.device).index_add_(0, tid, nd).clamp_(max=1.0)
        tx = torch.zeros(nt, nx.shape[1], dtype=torch.float64, device=nx.device).index_add_(0, tid, nx).clamp_(max=1.0)
        self.n_tiles += td.t() @ tx

    def result(self):
        """(value, bound): the per-entry rounding depth is at most 128 within a tile, one per contributing tile, and as
        many again for the per-ray sums of the attribute nets' direction and ones rows (per_tile = 2); the point kernels'
        depth is derived in the module docstring (per_tile = POINT_TILE_ROUNDINGS)."""
        n = self.per_tile * self.n_tiles + self.n_samples.clamp(max=TILE) + C_SUM
        return self.v, self.e + _round(self.a, n) + ATOMICS_PER_TILE * FTZ * self.n_tiles


# ---- the dense stage: sigma MLP and attribute heads -------------------------------------------------------------------
def compositing_inputs(ref: dict, U: dict, live: torch.Tensor, weight_bound: torch.Tensor, dsigma_bound: torch.Tensor):
    """dL/dσ and dL/dattr as the dense backward forms them, from compositing_ref.composite's result on the kernel's
    saved σ and attributes.  live [N, S] bool: the forward's attribute mask.  Returns float64 [P] / [2, P] tensors:
    dsig, dsig_e, dattr, dattr_e (dattr = g_image w inside the mask: w within its weight bound, one rounding)."""
    N, S = ref["weights"].shape
    gi = U["image_lidar"].double().reshape(N, 2) if "image_lidar" in U else \
        torch.zeros(N, 2, dtype=torch.float64, device=live.device)
    w = ref["weights"]
    m = live.double()
    dattr = torch.stack([gi[:, 0, None] * w * m, gi[:, 1, None] * w * m]).reshape(2, -1)
    dattr_e = torch.stack([gi[:, 0, None].abs() * weight_bound * m, gi[:, 1, None].abs() * weight_bound * m]).reshape(2, -1)
    dattr_e = dattr_e + EPS32 * dattr.abs()
    return dict(dsig=ref["dsigma"].reshape(-1), dsig_e=dsigma_bound.reshape(-1),
                dattr=dattr, dattr_e=dattr_e)


def _sigma_forward(W: dict, x: torch.Tensor, ip: int) -> dict:
    """Forward of the sigma MLP from exact inputs x [c, K]: the padded input, the hidden layer with its ReLU decisions,
    the output o, σ with its bound and geo."""
    c, K = x.shape
    xt = exact(torch.cat([x.double(), torch.ones(c, ip - K, dtype=torch.float64, device=x.device)], 1))
    h, on1, amb1 = _relu(_lin(xt, W["s1"], ip))
    o = _lin(h, W["s2"], 64)
    sig = o.v[:, 0].exp()
    sig_b = sig * torch.expm1(o.e[:, 0]) + 3.0 * EPS32 * sig * o.e[:, 0].exp() + TINY
    return dict(xt=xt, h=h, on1=on1, amb1=amb1, o=o, sig=sig, sig_b=sig_b, geo=V(o.v[:, 1:], o.e[:, 1:]))


def _sigma_backward(W: dict, K: int, f: dict, ds: torch.Tensor, dse: torch.Tensor, dgeo: V, tid: torch.Tensor, tc: bool,
                    tiles, gS1: _Grad, gS2: _Grad):
    """Backward of the sigma MLP from dL/dσ (ds, its bound dse) and dL/dgeo; adds the weight gradients and returns
    (dL/dX, largest log2(sc r) of the launch's tensor-core delta tiles).  tiles(x): per sample, the largest x of its tile."""
    eo = f["o"].v[:, 0].clamp(-15.0, 15.0).exp()
    d0 = V((ds * eo)[:, None],
           (dse * eo + ds.abs() * eo * torch.expm1(f["o"].e[:, 0]) + _round((ds * eo).abs(), 3.0))[:, None])
    do = V(torch.cat([d0.v, dgeo.v], 1), torch.cat([d0.e, dgeo.e], 1))
    max_log2_scale = 0.0
    if tc:
        do = _rescale(do, tiles(_row_amax(do)))
        lsc = pow2_log2(tiles(do.v.abs().amax(1)))
    gS2.add(do, f["h"], tid)
    dh = _back(do, W["s2"], 16, f["on1"], f["amb1"])
    if tc:              # sc r of the sigma backward's two delta tiles, from the reference's tile maxima
        lr = pow2_log2(tiles(dh.v.abs().amax(1)) * torch.exp2(lsc))
        live_t = (lsc > 0) & (lr > 0)
        if bool(live_t.any()):
            max_log2_scale = float((lsc + lr)[live_t].max())
        dh = _rescale(dh, tiles(_row_amax(dh)))
    gS1.add(dh, f["xt"], tid)
    return _back(dh, W["s1"][:, :K], 64), max_log2_scale


def _attr_stage(W: dict, enc: torch.Tensor, enc_e: torch.Tensor, geo: V, lv: torch.Tensor, dattr: torch.Tensor,
                dattr_e: torch.Tensor, tid: torch.Tensor, tc: bool, tiles, gA1: list, gA2: list, gA3: list):
    """Both attribute nets, forward and backward, on c samples: enc, enc_e [c, 72] (direction encoding per sample), geo,
    lv [c] bool (the mask), dattr, dattr_e [2, c] (dL/dattr, zero outside the mask, and its bound).  Adds the weight
    gradients; returns (attr [2, c], its bound, dL/dgeo, samples with an ambiguous unit)."""
    c = enc.shape[0]
    dev = enc.device
    m = lv.double()[:, None]
    ones9 = torch.ones(c, W["a1_0"].shape[1] - ENC - GEO, dtype=torch.float64, device=dev)
    a_in = V(torch.cat([enc, geo.v, ones9], 1) * m, torch.cat([enc_e, geo.e, torch.zeros_like(ones9)], 1) * m)
    amb_attr = torch.zeros_like(lv)
    attr_v, attr_b, dgeo = [], [], None
    for net in range(2):
        h1, on_a1, amb_a1 = _relu(_lin(a_in, W[f"a1_{net}"], a_in.v.shape[1]))
        h2, on_a2, amb_a2 = _relu(_lin(h1, W[f"a2_{net}"], 64))
        lg = _lin(h2, W[f"a3_{net}"][:1], 64)
        s = torch.sigmoid(lg.v[:, 0])
        sb = s * (1 - s) * lg.e[:, 0] * lg.e[:, 0].exp() + 8.0 * EPS32 * s
        attr_v.append(s * m[:, 0])
        attr_b.append(sb * m[:, 0])
        amb_attr = amb_attr | (lv & (amb_a1.any(1) | amb_a2.any(1)))
        # backward
        da, dae = dattr[net], dattr_e[net]
        q = s * (1 - s)
        dl = V((da * q)[:, None],
               (q * dae + da.abs() * ((1 - 2 * s).abs() * sb + sb * sb) + _round((da * q).abs(), 4.0))[:, None])
        w3 = W[f"a3_{net}"][0]
        if tc:          # dO8 and T3 tiles: scaled by cs from amax(|dl|) max(1, max|w3|)
            am = tiles(_row_amax(dl)) * max(1.0, float(w3.abs().max()))
            dl = _rescale(dl, am)
        gA3[net].add(dl, h2, tid)
        d2 = V(dl.v * w3, dl.e * w3.abs() + _round(dl.mag() * w3.abs(), 1.0))
        if tc:
            d2 = _rescale(d2, am)
        d2 = _mask(d2, on_a2, amb_a2)
        gA2[net].add(d2, h1, tid)
        d1 = _back(d2, W[f"a2_{net}"], 64, on_a1, amb_a1)
        if tc:
            d1 = _rescale(d1, tiles(_row_amax(d1)))
        gA1[net].add(d1, a_in, tid)
        g = _back(d1, W[f"a1_{net}"][:, ENC:ENC + GEO], 64)
        dgeo = g if dgeo is None else V(dgeo.v + g.v, dgeo.e + g.e + _round(dgeo.mag() + g.mag(), 1.0))
    return torch.stack(attr_v), torch.stack(attr_b), dgeo, amb_attr


def _head_results(gA1: list, gA2: list, gA3: list, out: dict, dev):
    for net, name in enumerate(HEADS):
        parts = [gA1[net].result(), gA2[net].result(), gA3[net].result()]
        z = torch.zeros(15 * 64, dtype=torch.float64, device=dev)         # W3 rows 1..15: no contribution
        out[name] = (torch.cat([p[0].reshape(-1) for p in parts] + [z]), torch.cat([p[1].reshape(-1) for p in parts] + [z]))


def dense_reference(cfg, W: dict, X: torch.Tensor, n_rays: int, S: int, enc: torch.Tensor, enc_e: torch.Tensor,
                    live: torch.Tensor, up: dict, tc: bool, on_chunk=None, chunk: int = CHUNK) -> dict:
    """Float64 sigma MLP and attribute heads of a launch of n_rays x S samples, forward and backward.

    W: working_weights; X [P, K] (any float dtype, exact values); enc, enc_e [n_rays, 72]: direction_encoding; live [P]
    bool; up: compositing_inputs (dsig*, dattr* as float64 on X's device).  on_chunk(p0, p1, outs) is called per chunk of
    whole rays with the per-sample outputs name -> (value, bound): sigma [c], attr [2, c] (0 outside the mask),
    geo [c, 15], dfeat [c, K].
    Returns weight gradients name -> (value, bound) in the parameter's flat order - sigma_net.params, intensity_net.params,
    raydrop_net.params - and "ambiguous" / "ambiguous_attr" (samples with an ambiguous ReLU unit in the sigma MLP / in an
    attribute net), "tiles", and in tensor-core mode "max_log2_scale": the largest log2(sc r) of the sigma backward's
    delta tiles (sc for dO, r for dHs), where 1 / (sc r) would overflow to 0 above 128."""
    dev = X.device
    K, ip, ap = cfg.sigma_in_dim, cfg.sigma_in_pad, cfg.attr_in_pad
    P = n_rays * S
    assert X.shape == (P, K) and ap == ENC + GEO + 9
    gS1, gS2 = _Grad((64, ip), dev), _Grad((16, 64), dev)
    gA1 = [_Grad((64, ap), dev) for _ in range(2)]
    gA2 = [_Grad((64, 64), dev) for _ in range(2)]
    gA3 = [_Grad((1, 64), dev) for _ in range(2)]
    rays_per = max(1, chunk // S)
    n_amb = n_amb_attr = 0
    max_log2_scale = 0.0
    tiles = lambda v: _tiles_dense(v, S)
    for r0 in range(0, n_rays, rays_per):
        r1 = min(n_rays, r0 + rays_per)
        p0, p1 = r0 * S, r1 * S
        c = p1 - p0
        j = torch.arange(c, device=dev)
        tid = (j // S) * ((S + TILE - 1) // TILE) + (j % S) // TILE
        f = _sigma_forward(W, X[p0:p1], ip)
        lv = live[p0:p1].to(dev)
        attr_v, attr_b, dgeo, amb_attr = _attr_stage(
            W, enc[r0:r1].repeat_interleave(S, 0), enc_e[r0:r1].repeat_interleave(S, 0), f["geo"], lv,
            up["dattr"][:, p0:p1], up["dattr_e"][:, p0:p1], tid, tc, tiles, gA1, gA2, gA3)
        n_amb += int(f["amb1"].any(1).sum())
        n_amb_attr += int(amb_attr.sum())
        dx, lsc = _sigma_backward(W, K, f, up["dsig"][p0:p1], up["dsig_e"][p0:p1], dgeo, tid, tc, tiles, gS1, gS2)
        max_log2_scale = max(max_log2_scale, lsc)
        if on_chunk is not None:
            on_chunk(p0, p1, {"sigma": (f["sig"], f["sig_b"]), "attr": (attr_v, attr_b),
                              "geo": (f["geo"].v, f["geo"].e), "dfeat": (dx.v, dx.e)})
    T = n_rays * ((S + TILE - 1) // TILE)
    out = {"ambiguous": n_amb, "ambiguous_attr": n_amb_attr, "tiles": T, "max_log2_scale": max_log2_scale}
    v1, b1 = gS1.result()
    v2, b2 = gS2.result()
    out["sigma_net.params"] = (torch.cat([v1.reshape(-1), v2.reshape(-1)]), torch.cat([b1.reshape(-1), b2.reshape(-1)]))
    _head_results(gA1, gA2, gA3, out, dev)
    return out


# ---- the point queries: LiDAR4D.density and LiDAR4D.attribute (csrc/l4d_points.cuh) ------------------------------------
def _point_chunk(chunk: int) -> int:
    return max(TILE, chunk // TILE * TILE)             # the point kernels' flat tiles start at multiples of 128


def density_point_reference(cfg, W: dict, X: torch.Tensor, dsig=None, dgeo=None, on_chunk=None, chunk: int = CHUNK) -> dict:
    """Float64 sigma MLP of n explicit points, forward and backward (k_density_train's σ / geo from its saved features,
    k_density_bwd's B1 and B3).  X [n, K] the saved features (exact); dsig [n] and dgeo [n, 15]: the exact upstream
    gradients, None for a missing one (the kernel then reads a null pointer as 0).  on_chunk(p0, p1, outs) gets sigma [c],
    geo [c, 15] and dfeat [c, K] (dL/dfeature, which the kernel forms from dh without storing it) as (value, bound).
    Returns sigma_net.params -> (value, bound) with the point path's rounding depth, "ambiguous" and "tiles"."""
    dev = X.device
    n, K = X.shape
    ip = cfg.sigma_in_pad
    gS1, gS2 = _Grad((64, ip), dev, POINT_TILE_ROUNDINGS), _Grad((16, 64), dev, POINT_TILE_ROUNDINGS)
    chunk = _point_chunk(chunk)
    n_amb = 0
    for p0 in range(0, n, chunk):
        p1 = min(n, p0 + chunk)
        c = p1 - p0
        tid = torch.arange(c, device=dev) // TILE
        f = _sigma_forward(W, X[p0:p1], ip)
        n_amb += int(f["amb1"].any(1).sum())
        z = torch.zeros(c, dtype=torch.float64, device=dev)
        ds = z if dsig is None else dsig[p0:p1].double().to(dev)
        dg = exact(torch.zeros(c, GEO, dtype=torch.float64, device=dev) if dgeo is None else dgeo[p0:p1].to(dev))
        dx, _ = _sigma_backward(W, K, f, ds, z, dg, tid, False, None, gS1, gS2)
        if on_chunk is not None:
            on_chunk(p0, p1, {"sigma": (f["sig"], f["sig_b"]), "geo": (f["geo"].v, f["geo"].e), "dfeat": (dx.v, dx.e)})
    v1, b1 = gS1.result()
    v2, b2 = gS2.result()
    return {"ambiguous": n_amb, "tiles": (n + TILE - 1) // TILE,
            "sigma_net.params": (torch.cat([v1.reshape(-1), v2.reshape(-1)]), torch.cat([b1.reshape(-1), b2.reshape(-1)]))}


def attribute_point_reference(cfg, W: dict, d: torch.Tensor, geo: torch.Tensor, mask, dattr: torch.Tensor, on_chunk=None,
                              chunk: int = CHUNK) -> dict:
    """Float64 attribute nets of n explicit points, forward and backward (k_attribute, k_attribute_bwd).  d [n, 3] the
    directions (encoded per point, direction_encoding), geo [n, 15] exact, mask [n] bool or None (all points), dattr [n, 2]
    the exact dL/d(raydrop, intensity).  on_chunk(p0, p1, outs) gets attr [2, c] (0 outside the mask) and dgeo [c, 15]
    (0 outside the mask) as (value, bound).  Returns intensity_net.params and raydrop_net.params -> (value, bound) with
    the point path's rounding depth, and "ambiguous_attr"."""
    dev = d.device
    n = d.shape[0]
    assert cfg.attr_in_pad == ENC + GEO + 9
    ap = cfg.attr_in_pad
    gA1 = [_Grad((64, ap), dev, POINT_TILE_ROUNDINGS) for _ in range(2)]
    gA2 = [_Grad((64, 64), dev, POINT_TILE_ROUNDINGS) for _ in range(2)]
    gA3 = [_Grad((1, 64), dev, POINT_TILE_ROUNDINGS) for _ in range(2)]
    chunk = _point_chunk(chunk)
    n_amb = 0
    for p0 in range(0, n, chunk):
        p1 = min(n, p0 + chunk)
        c = p1 - p0
        tid = torch.arange(c, device=dev) // TILE
        lv = torch.ones(c, dtype=torch.bool, device=dev) if mask is None else mask[p0:p1].to(dev).bool()
        enc, enc_e = direction_encoding(d[p0:p1])
        da = dattr[p0:p1].double().t() * lv.double()
        attr_v, attr_b, dgeo, amb = _attr_stage(W, enc, enc_e, exact(geo[p0:p1]), lv, da, torch.zeros_like(da), tid,
                                                False, None, gA1, gA2, gA3)
        n_amb += int(amb.sum())
        if on_chunk is not None:
            on_chunk(p0, p1, {"attr": (attr_v, attr_b), "dgeo": (dgeo.v, dgeo.e)})
    out = {"ambiguous_attr": n_amb, "tiles": (n + TILE - 1) // TILE}
    _head_results(gA1, gA2, gA3, out, dev)
    return out


# ---- the flow MLP ---------------------------------------------------------------------------------------------------------
def flow_reference(W: dict, fin: torch.Tensor, dflow: torch.Tensor, tc: bool, on_chunk=None, chunk: int = CHUNK,
                   dflow_err: torch.Tensor = None, points: bool = False) -> dict:
    """Float64 flow MLP of P samples, forward and backward.

    fin [16, P] (the forward's flow-MLP input, float32 values), dflow [6, P] (the upstream gradient: exact as the kernels
    saved or received it, or a float64 reference with its bound dflow_err [6, P] - the density backward forms dL/dflow
    from its own dL/dfeature and never stores it).  points: the weight gradients take the point kernels' rounding depth.
    on_chunk(p0, p1, outs) gets flow [c, 6] and dfin [c, 16] as (value, bound).  Returns flow_net.mlp.{0,2,4}.weight
    -> (value, bound), "ambiguous" and "tiles"."""
    dev = fin.device
    P = fin.shape[1]
    per_tile = POINT_TILE_ROUNDINGS if points else 2.0
    g0, g1, g2 = _Grad((64, 16), dev, per_tile), _Grad((64, 64), dev, per_tile), _Grad((6, 64), dev, per_tile)
    chunk = max(TILE, chunk // TILE * TILE)           # the kernels' flat tiles start at multiples of 128
    n_amb = 0
    for p0 in range(0, P, chunk):
        p1 = min(P, p0 + chunk)
        f = exact(fin[:, p0:p1].t())
        tid = torch.arange(p1 - p0, device=dev) // TILE
        h1, on1, amb1 = _relu(_lin(f, W["f0"], 16))
        h2, on2, amb2 = _relu(_lin(h1, W["f1"], 64))
        fl = _lin(h2, W["f2"], 64)
        n_amb += int((amb1.any(1) | amb2.any(1)).sum())
        g = exact(dflow[:, p0:p1].t())
        if dflow_err is not None:
            g = V(g.v, dflow_err[:, p0:p1].t().double())
        if tc:
            g = _rescale(g, _tiles_flat(_row_amax(g)))
        g2.add(g, h2, tid)
        d2 = _back(g, W["f2"], 6, on2, amb2)
        if tc:
            d2 = _rescale(d2, _tiles_flat(_row_amax(d2)))
        g1.add(d2, h1, tid)
        d1 = _back(d2, W["f1"], 64, on1, amb1)
        if tc:
            d1 = _rescale(d1, _tiles_flat(_row_amax(d1)))
        g0.add(d1, f, tid)
        dfin = _back(d1, W["f0"], 64)
        if on_chunk is not None:
            on_chunk(p0, p1, {"flow": (fl.v, fl.e), "dfin": (dfin.v, dfin.e)})
    T = (P + TILE - 1) // TILE
    out = {"ambiguous": n_amb, "tiles": T}
    for i, g in enumerate((g0, g1, g2)):
        out[f"flow_net.mlp.{2 * i}.weight"] = g.result()
    return out


def ratio(got: torch.Tensor, value: torch.Tensor, bound: torch.Tensor):
    """|got - value| / bound per entry (inf where the bound is 0 and got differs, 0 where both agree exactly)."""
    err = (got.double().reshape(value.shape) - value).abs()
    return torch.where(bound > 0, err / bound.clamp_min(1e-300),
                       torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
