"""CPU: the float64 reference of the MLP stages (tests/dense_ref.py) against autograd, and its bound from both sides.

The values must match torch autograd through the oracle's fused_mlp in float64 to 1e-12.  The bound must hold for a
torch emulation of each kernel family - a float32 evaluation (the FMA kernels), and the tensor-core arithmetic (fp16
weights, activations and delta tiles as fp16 hi + lo, per-tile power-of-two delta scales capped at 2^126 and undone as
(1/sc)/r, three-term weight-gradient products Ah·δh + Al·δh + Ah·δl summed per 128-sample tile) - and must be left by
each of these mutations of the tensor-core emulation: two-term products, 1/(sc·r) where sc·r passes 2^128, sigma W1's
ones columns without gradient, and one tile's weight gradients counted twice."""
import pytest
import torch

import dense_ref as DR
from oracle import lidar4d_oracle as O
from parity_util import small_config

TINY_RAY = 2.0 ** -124          # dL/dσ scale of ray 0 in the mutation cases: its tiles scale by the 2^126 cap


def fixture(L: int, S: int, tc: bool, seed: int = 5, n_rays: int = 6, tiny_ray: bool = False):
    cfg = small_config(n_levels_hash=L)
    orc = O.build_seeded(cfg, seed, flow_last_std=0.5)
    params = {k: v.detach() for k, v in orc.ref_state_dict().items()}
    W = DR.working_weights(cfg, params, tc)
    g = torch.Generator().manual_seed(seed)
    P, K = n_rays * S, cfg.sigma_in_dim
    X = torch.randn(P, K, generator=g) * 0.5
    if tc:                                  # what the tensor cores read: fp16 hi + lo, exact in float32
        hi = X.half().float()
        X = hi + (X - hi).half().float()
    d = torch.randn(n_rays, 3, generator=g)
    d = (d / d.norm(dim=1, keepdim=True)).float()
    live = torch.rand(P, generator=g) < 0.6
    live[:S] = False                        # ray 0 entirely outside the attribute mask
    dsig = torch.randn(P, generator=g).float()
    dattr = (torch.randn(2, P, generator=g) * live).float()
    if tiny_ray:
        dsig[:S] *= TINY_RAY
    fin = (torch.randn(16, P, generator=g) * 0.3).float()
    dflow = torch.randn(6, P, generator=g).float()
    dflow[:, 128:256] = 0.0                 # a flow tile without gradient (skipped by the kernels)
    return dict(cfg=cfg, params=params, W=W, X=X, d=d, live=live, dsig=dsig, dattr=dattr, fin=fin, dflow=dflow,
                n_rays=n_rays, S=S, tc=tc)


def reference(f):
    enc, enc_e = DR.direction_encoding(f["d"])
    up = dict(dsig=f["dsig"].double(), dsig_e=torch.zeros(f["dsig"].shape, dtype=torch.float64),
              dattr=f["dattr"].double(), dattr_e=torch.zeros(f["dattr"].shape, dtype=torch.float64))
    per = {}

    def keep(p0, p1, outs):
        for k, v in outs.items():
            per.setdefault(k, []).append(v)
    out = DR.dense_reference(f["cfg"], f["W"], f["X"], f["n_rays"], f["S"], enc, enc_e, f["live"], up, f["tc"], keep,
                             chunk=2 * f["S"])
    fo = DR.flow_reference(f["W"], f["fin"], f["dflow"], f["tc"], keep, chunk=256)
    out.update(fo)
    for k, parts in per.items():
        cat = 1 if k == "attr" else 0
        out[k] = (torch.cat([p[0] for p in parts], cat), torch.cat([p[1] for p in parts], cat))
    return out


# ---- values against autograd ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [3, 10])
def test_values_match_autograd(L):
    f = fixture(L, 129, tc=False)
    ref = reference(f)
    cfg, S, N = f["cfg"], f["S"], f["n_rays"]
    K = cfg.sigma_in_dim
    leaf = {k: f["params"][k].double().clone().requires_grad_(True) for k in
            ("sigma_net.params", "intensity_net.params", "raydrop_net.params", "flow_net.mlp.0.weight",
             "flow_net.mlp.2.weight", "flow_net.mlp.4.weight")}
    X = f["X"].double().requires_grad_(True)
    fin = f["fin"].double().t().contiguous().requires_grad_(True)
    o = O.fused_mlp(X, leaf["sigma_net.params"], K, 16, 64, 1)
    sigma = O._TruncExp.apply(o[:, 0])
    geo = o[:, 1:]
    enc = DR.direction_encoding(f["d"])[0].repeat_interleave(S, 0)
    inp = torch.cat([enc, geo], 1)
    attr = [torch.sigmoid(O.fused_mlp(inp, leaf[n], cfg.attr_in_dim, 1, 64, 2)[:, 0]) * f["live"]
            for n in DR.HEADS]
    h = torch.relu(fin @ leaf["flow_net.mlp.0.weight"].t())
    h = torch.relu(h @ leaf["flow_net.mlp.2.weight"].t())
    flow = h @ leaf["flow_net.mlp.4.weight"].t()
    loss = (sigma * f["dsig"].double()).sum() + sum((a * f["dattr"][i].double()).sum() for i, a in enumerate(attr)) \
        + (flow * f["dflow"].double().t()).sum()
    loss.backward()

    def close(got, want, what):
        err = float((got.reshape(want.shape) - want).abs().max())
        assert err <= 1e-12 * max(1.0, float(want.abs().max())), (what, err)
    close(ref["sigma"][0], sigma.detach(), "sigma")
    close(ref["attr"][0], torch.stack([a.detach() for a in attr]), "attr")
    close(ref["flow"][0], flow.detach(), "flow")
    close(ref["dfeat"][0], X.grad, "dfeat")
    close(ref["dfin"][0], fin.grad, "dfin")
    for k, p in leaf.items():
        close(ref[k][0], p.grad, k)


# ---- torch emulation of the two kernel families --------------------------------------------------------------------------
def _split(x):
    hi = x.half().float()
    return hi, (x - hi).half().float()


def _pow2(am):
    """pow2_factor: maps amax into [2^5, 2^6), capped at 2^126; 1 for an all-zero tile."""
    _, e = torch.frexp(am)
    f = torch.ldexp(torch.ones_like(am), (6 - e).clamp(max=126))
    return torch.where(am > 0, f, torch.ones_like(am))


class Emu:
    """One kernel family on float32 tensors.  Deltas travel scaled by a per-tile power of two in tensor-core mode; `inv`
    [n_tiles] undoes it."""

    def __init__(self, tc: bool, tid: torch.Tensor, mutation: str = None):
        self.tc, self.tid, self.mut = tc, tid, mutation
        self.nt = int(tid.max()) + 1

    def mm(self, a, W):                          # activations times weights (forward)
        if not self.tc:
            return a @ W.t()
        h, l = _split(a)
        return h @ W.t() + l @ W.t()

    def mmT(self, d, W):                         # delta propagation d W
        if not self.tc:
            return d @ W
        h, l = _split(d)
        return h @ W + l @ W

    def amax(self, d):
        return torch.zeros(self.nt).scatter_reduce(0, self.tid, d.abs().reshape(d.shape[0], -1).amax(1), "amax")

    def scale(self, d, inv, sc, extra=1.0):
        """Re-scale a delta with its own tile amax: returns (scaled delta, inv, cumulative scale)."""
        if not self.tc:
            return d, inv, sc
        r = _pow2(self.amax(d) * extra)
        inv2 = 1.0 / (sc * r) if self.mut == "inv_product" else (inv / r)
        return d * r[self.tid][:, None], inv2, sc * r

    def wgrad(self, d, x, inv):
        """Σ over tiles of inv_t Σ_p d_p ⊗ x_p [out, in] in float32."""
        out = torch.zeros(d.shape[1], x.shape[1])
        for t in range(self.nt):
            s = self.tid == t
            if not bool(s.any()):
                continue
            if self.tc:
                dh, dl = _split(d[s])
                xh, xl = _split(x[s])
                tt = dh.t() @ xh + dl.t() @ xh
                if self.mut != "two_term":
                    tt = tt + dh.t() @ xl
            else:
                tt = d[s].t() @ x[s]
            tt = tt * inv[t]
            out = out + tt
            if self.mut == "tile_twice" and t == self.nt // 2:
                out = out + tt
        return out


def emulate(f, mutation=None):
    cfg, S, N, tc = f["cfg"], f["S"], f["n_rays"], f["tc"]
    K, ip = cfg.sigma_in_dim, cfg.sigma_in_pad
    W = {k: v.float() for k, v in f["W"].items()}
    P = N * S
    j = torch.arange(P) % S
    tid = (torch.arange(P) // S) * ((S + 127) // 128) + j // 128
    E = Emu(tc, tid, mutation)
    one = torch.ones(E.nt)
    relu = torch.relu
    xt = torch.cat([f["X"].float(), torch.ones(P, ip - K)], 1)
    z1 = E.mm(xt, W["s1"])
    m1 = (z1 > 0).float()
    h = relu(z1)
    o = E.mm(h, W["s2"])
    out = {"sigma": torch.exp(o[:, 0])}
    geo = o[:, 1:]
    arg = [((f["d"][:, dim] + 1.0) / 2.0 * float(1 << k)) * DR.PI32 + (DR.HALF_PI32 if ph else 0.0)
           for dim in range(3) for k in range(12) for ph in range(2)]
    enc = torch.sin(torch.stack(arg, -1)).float().repeat_interleave(S, 0)
    live = f["live"].float()[:, None]
    a_in = torch.cat([enc, geo, torch.ones(P, 9)], 1) * live
    dgeo = torch.zeros(P, 15)
    attr, grads = [], {}
    for net in range(2):
        za1 = E.mm(a_in, W[f"a1_{net}"])
        ha1 = relu(za1) * live
        za2 = E.mm(ha1, W[f"a2_{net}"])
        ha2 = relu(za2) * live
        w3 = W[f"a3_{net}"][0]
        a = 1.0 / (1.0 + torch.exp(-(ha2 @ w3)))
        attr.append(a * live[:, 0])
        draw = f["dattr"][net] * a * (1.0 - a)
        do, inv, sc = E.scale(draw[:, None], one, one, max(1.0, float(w3.abs().max())))
        dw3 = E.wgrad(do, ha2, inv)
        t3 = do * w3[None] * (za2 > 0).float()
        dwa2 = E.wgrad(t3, ha1, inv)
        dh1 = E.mmT(t3, W[f"a2_{net}"]) * (za1 > 0).float()
        dh1, inv, sc = E.scale(dh1, inv, sc)
        dwa1 = E.wgrad(dh1, a_in, inv)
        dgeo = dgeo + E.mmT(dh1, W[f"a1_{net}"][:, DR.ENC:DR.ENC + DR.GEO]) * inv[tid][:, None]
        name = DR.HEADS[net]
        grads[name] = torch.cat([dwa1.reshape(-1), dwa2.reshape(-1), dw3.reshape(-1), torch.zeros(15 * 64)])
    out["attr"] = torch.stack(attr)
    do = torch.cat([(f["dsig"] * torch.exp(o[:, 0].clamp(-15, 15)))[:, None], dgeo], 1)
    do, inv, sc = E.scale(do, one, one)
    dw2 = E.wgrad(do, h, inv)
    dh = E.mmT(do, W["s2"]) * m1
    dh, inv, sc = E.scale(dh, inv, sc)
    dw1 = E.wgrad(dh, xt, inv)
    if mutation == "ones_no_grad":
        dw1[:, K:] = 0.0
    out["dfeat"] = E.mmT(dh, W["s1"][:, :K]) * inv[tid][:, None]
    grads["sigma_net.params"] = torch.cat([dw1.reshape(-1), dw2.reshape(-1)])
    # flow MLP: flat tiles of 128 samples
    F = Emu(tc, torch.arange(P) // 128, mutation)
    fone = torch.ones(F.nt)
    fin = f["fin"].t().contiguous()
    y1 = F.mm(fin, W["f0"])
    h1 = relu(y1)
    y2 = F.mm(h1, W["f1"])
    h2 = relu(y2)
    out["flow"] = F.mm(h2, W["f2"])
    g, inv, sc = F.scale(f["dflow"].t().contiguous(), fone, fone)
    grads["flow_net.mlp.4.weight"] = F.wgrad(g, h2, inv)
    d2 = F.mmT(g, W["f2"]) * (y2 > 0).float()
    d2, inv, sc = F.scale(d2, inv, sc)
    grads["flow_net.mlp.2.weight"] = F.wgrad(d2, h1, inv)
    d1 = F.mmT(d2, W["f1"]) * (y1 > 0).float()
    d1, inv, sc = F.scale(d1, inv, sc)
    grads["flow_net.mlp.0.weight"] = F.wgrad(d1, fin, inv)
    out["dfin"] = F.mmT(d1, W["f0"]) * inv[F.tid][:, None]
    out.update(grads)
    return out


NAMES = ("sigma", "attr", "flow", "dfeat", "dfin", "sigma_net.params", "intensity_net.params", "raydrop_net.params",
         "flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight")


def worst(ref, emu):
    return {k: float(DR.ratio(emu[k], *ref[k]).max()) for k in NAMES}


@pytest.mark.parametrize("tc", [False, True], ids=["fp32", "tc"])
@pytest.mark.parametrize("L,S", [(8, 333), (9, 129), (10, 2)])
def test_bound_holds_for_both_kernel_families(L, S, tc):
    f = fixture(L, S, tc, tiny_ray=tc)
    ref = reference(f)
    r = worst(ref, emulate(f))
    assert max(r.values()) <= 1.0, r
    assert ref["ambiguous"] <= 1e-2 * f["n_rays"] * S, ref["ambiguous"]            # the sigma MLP
    # the bound is not vacuous: the worst entry of every output sits within a few decades of it
    assert min(v for k, v in r.items() if k != "dfeat" or not tc) > 1e-6, r
    print(f"[dense-ref] L={L} S={S} {'tc' if tc else 'fp32'}: " + " ".join(f"{k} {v:.2e}" for k, v in r.items()))


# mutation -> (fixture, outputs that must leave the bound).  Dropping a term of the hi|lo products moves each product by
# ~2^-13 of itself with random signs, so it shows where an entry has few contributions: a launch of two 3-sample rays.
MUTATIONS = {"two_term": (dict(L=8, S=3, n_rays=2), ("sigma_net.params", "flow_net.mlp.2.weight")),
             "inv_product": (dict(L=8, S=333, tiny_ray=True), ("dfeat",)),
             "ones_no_grad": (dict(L=8, S=333), ("sigma_net.params",)),
             "tile_twice": (dict(L=8, S=333), ("sigma_net.params", "intensity_net.params", "flow_net.mlp.2.weight"))}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_bound_catches_mutations(mutation):
    kw, names = MUTATIONS[mutation]
    f = fixture(tc=True, **kw)
    ref = reference(f)
    assert max(worst(ref, emulate(f)).values()) <= 1.0
    if mutation == "inv_product":
        assert ref["max_log2_scale"] > 128, ref["max_log2_scale"]
    r = worst(ref, emulate(f, mutation))
    caught = {k: r[k] for k in names}
    assert all(v > 1.0 for v in caught.values()), (mutation, r)
    print(f"[dense-ref] mutation {mutation}: " + " ".join(f"{k} {v:.3g}" for k, v in caught.items()))
