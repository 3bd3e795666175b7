"""Float64 reference of the backward's scatter stage (test infrastructure).

Given what the split pipeline's backward consumed - dL/dfeature of every sample, the forward's flow, in tensor-core mode
dL/d(flow-MLP input) - the gradients of the encoder tables are a linear function of those inputs.  This module evaluates
that function in float64, one contribution per (sample, corner or texel, feature), and returns per entry

    ref = sum of the contributions,   A = sum of their magnitudes,   n = number of contributions,

so that a kernel result can be held to |got - ref| <= (n + 16) * 2^-24 * A, a bound that holds for any summation order
(n roundings of the sum, up to 16 of each contribution's product).  Where a contribution is a product with a value that is
itself a sum (a bilinear plane sample, a difference of texels), A takes the sum of the magnitudes of its terms, so the
bound covers the rounding of those sums too.

The positions and the weights are the kernels' float32 arithmetic, restated op by op (l4d_x01, l4d_axis in
csrc/l4d_core.cuh; hash corners from the oracle's hash_indices, pinned bit-exact against the kernels): a float64 weight
would send contributions of positions within an ulp of a texel edge to the other texel.  Only the products and the sums
are float64.

Feature assembly (oracle density(), lidar4d.py:155-176): the current query takes 0.5 and each warped query 0.25, a missing
neighbour's share goes to the current query; the dynamic hash gets gradient from the current query only (the warped hash
queries are no_grad); a dynamic-hash feature is sum_k basis[k] * (w_lo * T_lo[k] + w_hi * T_hi[k]); flow-grid feature
(l, 2i + c) enters the flow MLP as basis[i] * it at input 2l + c.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import lidar4d_oracle as O

EPS32 = 2.0 ** -24
SLACK = 16                        # roundings allowed inside one contribution (the bound's "+ 16")
CHUNK = 1 << 18                   # samples per pass (keeps the float64 temporaries at a few hundred MB)
STATIC_PLANES = (0, 1, 3)         # itertools.combinations(range(4), 2): (x,y) (x,z) (y,z)
TIME_PLANES = (2, 4, 5)           # (x,t) (y,t) (z,t)
OTHER_STATIC = {0: (1, 3), 1: (0, 3), 3: (0, 1)}
STATIC_COORDS = {0: (0, 1), 1: (0, 2), 3: (1, 2)}
DYN_PAIRS = ((0, 1), (0, 2), (1, 2))


# ---- the saved buffer of a training forward (csrc/l4d_host.h saved_layout) ------------------------------------------
SAVED_FIELDS = ("feat", "flow_in", "sigma", "attr", "hidden", "flow", "dfeat", "dflow", "tstart", "hd_con", "pl_con")
BWD_SCRATCH_CTAS = 1024           # L4D_BWD_SCRATCH_CTAS
NT = 128                          # L4D_NT


def _align(v: int, a: int = 256) -> int:
    return (v + a - 1) // a * a


def saved_layout(cfg, n_rays: int, S: int) -> dict:
    """Byte offsets of the regions of the saved buffer and its total size, as l4d_saved_bytes computes them."""
    P = n_rays * S
    tiles = n_rays * ((S + 127) // 128)
    K = cfg.sigma_in_dim
    dyn_entries = sum(int(cfg.dynamic_grid(p).offset[-1]) for p in range(3))
    time_rows = 3 * sum(cfg.min_resolution * m * 8 * 3 for m in cfg.plane_scales)
    sizes = dict(feat=max(P * K * 4, tiles * ((K + 7) // 8) * 4096), flow_in=P * 16 * 4, sigma=P * 4, attr=P * 2 * 4,
                 hidden=BWD_SCRATCH_CTAS * 64 * NT * 4, flow=P * 6 * 4, dfeat=tiles * ((K + 3) // 4) * 2048,
                 dflow=P * 6 * 4, tstart=tiles * 4, hd_con=3 * dyn_entries * 4, pl_con=time_rows * 4)
    out, o = {}, 0
    for k in SAVED_FIELDS:
        out[k] = o
        o = _align(o + sizes[k])
    out["total"] = o
    return out


def decode_saved(cfg, saved: torch.Tensor, n_rays: int, S: int) -> dict:
    """Views of the saved buffer (uint8) that the split pipeline's stages read or write:
    dfeat [P, sigma_in_dim] (from the tiles [ray][tile][k/4][128][4]), flow / dflow [6, P], flow_in [16, P];
    the features, as fp32 SoA planes feat [sigma_in_dim, P] (fp32 mode) or as the raw fp16 operand tiles
    feat_tiles [ray][tile][hi|lo][k/8][128][8] (tensor-core mode; both views cover the same bytes);
    hd_con[q][p] [entries] (the contracted dynamic tables of query q = cur|fwd|bwd and plane p) and
    pl_con[q][s][t] [R, 8] (the contracted time-plane rows of query q, scale s, time plane t = (x,t)|(y,t)|(z,t))."""
    L = saved_layout(cfg, n_rays, S)
    assert saved.numel() >= L["total"], (saved.numel(), L["total"])
    P = n_rays * S
    f32 = lambda name, n, o=0: saved[L[name] + 4 * o:L[name] + 4 * (o + n)].view(torch.float32)
    nt, dq, xc = (S + 127) // 128, (cfg.sigma_in_dim + 3) // 4, (cfg.sigma_in_dim + 7) // 8
    df = f32("dfeat", n_rays * nt * dq * 128 * 4).view(n_rays, nt, dq, 128, 4)
    df = df.permute(0, 1, 3, 2, 4).reshape(n_rays, nt * 128, dq * 4)[:, :S, :cfg.sigma_in_dim].reshape(P, -1)
    tiles = saved[L["feat"]:L["feat"] + n_rays * nt * xc * 4096].view(torch.float16).view(n_rays, nt, 2, xc, 128, 8)
    ne = [int(cfg.dynamic_grid(p).offset[-1]) for p in range(3)]
    hd, o = [], 0
    for q in range(3):
        hd.append([])
        for p in range(3):
            hd[q].append(f32("hd_con", ne[p], o))
            o += ne[p]
    pl, o = [], 0
    for q in range(3):
        pl.append([])
        for s in range(cfg.n_levels_plane):
            R = cfg.min_resolution * cfg.plane_scales[s]
            pl[q].append([])
            for t in range(3):
                pl[q][s].append(f32("pl_con", R * 8, o).view(R, 8))
                o += R * 8
    return dict(dfeat=df, flow=f32("flow", 6 * P).view(6, P), dflow=f32("dflow", 6 * P).view(6, P),
                flow_in=f32("flow_in", 16 * P).view(16, P), feat=f32("feat", cfg.sigma_in_dim * P).view(-1, P),
                feat_tiles=tiles, hd_con=hd, pl_con=pl)


# ---- the kernels' float32 position arithmetic ---------------------------------------------------------------------------
def sample_x01(rays_o: torch.Tensor, rays_d: torch.Tensor, z: torch.Tensor, bound: float) -> torch.Tensor:
    """l4d_x01 of every sample: clamp(o + d * z, -bound, bound), then (p + bound) / (2 bound), float32 op by op.
    rays [N, 3], z [N, S] -> [N * S, 3]."""
    b = torch.tensor(bound, dtype=torch.float32, device=z.device)
    p = rays_o.float()[:, None, :] + rays_d.float()[:, None, :] * z.float()[:, :, None]   # two roundings, no fma
    p = torch.minimum(torch.maximum(p, -b), b)
    return ((p + b) / (b * 2.0)).reshape(-1, 3)


def point_x01(x: torch.Tensor, bound: float) -> torch.Tensor:
    """l4d_point_x01 of explicit points x [n, 3]: (x + bound) / (2 bound), float32 op by op, no clamp (points outside the
    box give coordinates outside [0, 1])."""
    b = torch.tensor(bound, dtype=torch.float32, device=x.device)
    return (x.float() + b) / (b * 2.0)


def axis(c: torch.Tensor, size: int):
    """l4d_axis: float32 coordinate in [0, 1] -> (i0, i1, w0, w1, gmult) of F.grid_sample(align_corners=True, border)."""
    c = c.float()
    g = c * 2.0 - 1.0
    ix = ((g + 1.0) / 2.0) * float(size - 1)
    mx = float(size - 1)
    gm = torch.full_like(ix, mx)
    lo, hi = ix <= 0.0, ix >= mx
    ix = torch.where(lo, torch.zeros_like(ix), torch.where(hi, torch.full_like(ix, mx), ix))
    gm = torch.where(lo | hi, torch.zeros_like(gm), gm)
    f = torch.floor(ix)
    i0 = f.long()
    i1 = i0 + 1
    w1 = ix - f
    w0 = (f + 1.0) - ix
    over = i1 > size - 1
    i1 = torch.where(over, torch.full_like(i1, size - 1), i1)
    w1 = torch.where(over, torch.zeros_like(w1), w1)
    return i0, i1, w0, w1, gm


# ---- accumulation -----------------------------------------------------------------------------------------------------
class _Sink:
    """Per-entry (sum, sum of magnitudes, count) in float64, and with carry=True a fourth column: the error bound carried
    in from the contributions' inputs."""

    def __init__(self, n: int, device, carry: bool = False):
        self.t = torch.zeros(n, 4 if carry else 3, dtype=torch.float64, device=device)

    def add(self, idx, c, a=None, e=None):
        c = c.reshape(-1)
        a = c.abs() if a is None else a.reshape(-1)
        cols = [c, a, torch.ones_like(c)]
        if self.t.shape[1] > 3:
            cols.append(torch.zeros_like(c) if e is None else e.reshape(-1))
        self.t.index_add_(0, idx.reshape(-1), torch.stack(cols, 1))

    def scaled(self, f: float):
        """The entries times a constant factor f (exact in float64 up to 2^-53)."""
        t = self.t.clone()
        t[:, 0] *= f
        t[:, 1] *= abs(f)
        if t.shape[1] > 3:
            t[:, 3] *= abs(f)
        return t


def _texels(Pt, b):
    """Values of the four texels of bilinear footprints b on a channels-last plane Pt [H, W, 8] (float64) and their
    weights: vals [C, 4, 8], wgt [C, 4] (float64 products of the float32 axis weights), ys / xs [C, 4]."""
    x0, x1, wx0, wx1, _ = b[0]
    y0, y1, wy0, wy1, _ = b[1]
    xs = torch.stack([x0, x1, x0, x1], 1)
    ys = torch.stack([y0, y0, y1, y1], 1)
    wx = torch.stack([wx0, wx1, wx0, wx1], 1).double()
    wy = torch.stack([wy0, wy0, wy1, wy1], 1).double()
    return Pt[ys, xs], wx * wy, ys, xs


def scatter_reference(cfg, params: dict, frame, x01: torch.Tensor, dfeat, flow, dfin: torch.Tensor = None,
                      dfin_err: torch.Tensor = None, dfeat_err: torch.Tensor = None) -> dict:
    """Float64 reference of the scatter stage.

    cfg FieldConfig; params: name -> fp32 master tensor (reference state_dict names); frame: geometry.FrameConstants;
    x01 [P, 3] float32 (sample_x01 or point_x01); dfeat [P, sigma_in_dim] float32; flow [6, P] float32 (the forward's);
    dfin [16, P] dL/d(flow-MLP input) or None (no flow-grid reference): the kernel's saved float32 values, or a float64
    reference with its error bound dfin_err [16, P] (tests/dense_ref.py, for the fp32 kernels, which never store it).
    dfeat_err [P, sigma_in_dim]: dfeat is itself a float64 reference with this bound (the point density backward forms
    dL/dfeature from dh without storing it); every table entry and dL/dflow then carry it in a fourth column.
    dfeat None: the flow grid alone, from a dfin produced after a first pass (the density backward's order is
    dL/dfeature -> dL/dflow -> dL/d(flow-MLP input) -> flow grid).
    Returns name -> [numel, 3] float64 (ref, A, n) per entry in the tensor's flat order, and "dflow" -> [P, 6, 3]; a fourth
    column holds a carried-in bound where dfin_err (flow grid) or dfeat_err (the others) is given (check_entries adds it)."""
    dev = x01.device
    P = x01.shape[0]
    nS, L = cfg.n_levels_plane, cfg.n_levels_hash
    row_plane_d, row_hash_s = nS * 8, 2 * nS * 8
    row_hash_d = row_hash_s + 4 * L
    T = cfg.time_resolution
    wc = 0.5 + (0.0 if frame.has_fwd else 0.25) + (0.0 if frame.has_bwd else 0.25)
    queries = [(0, wc, frame.cur)]
    if frame.has_fwd:
        queries.append((1, 0.25, frame.fwd))
    if frame.has_bwd:
        queries.append((2, 0.25, frame.bwd))
    feats = dfeat is not None
    carry = dfeat_err is not None

    gs, gf = cfg.static_grid(), cfg.flow_grid()
    gd = [cfg.dynamic_grid(p) for p in range(3)]
    fcomb = _Sink(int(gf.offset[-1]) * 2, dev) if dfin is not None else None
    ferr = torch.zeros(int(gf.offset[-1]) * 2, dtype=torch.float64, device=dev) if dfin_err is not None else None
    planes, pl64 = {}, {}
    if feats:
        static = _Sink(int(gs.offset[-1]) * 4, dev, carry)
        comb = [_Sink(int(gd[p].offset[-1]), dev, carry) for p in range(3)]    # sum of w_corner * wc * dL/dfeature
        for s in range(nS):
            for ci in range(6):
                name = f"planes_encoder.planes.{s}.{ci}"
                planes[name] = _Sink(params[name].numel(), dev, carry)
                pl64[name] = params[name].detach()[0].permute(1, 2, 0).double()         # [H, W, 8]
        dflow = torch.zeros(P, 6, 4 if carry else 3, dtype=torch.float64, device=dev)
    ar4 = torch.arange(4, device=dev)

    for h in range(0, P, CHUNK):
        x = x01[h:h + CHUNK].float()
        C = x.shape[0]

        # flow grid: feature (l, 2i + c) of a corner gets basis[i] * w_corner * dFin[2l + c]; the basis is applied below
        if fcomb is not None:
            dfi = dfin[:, h:h + CHUNK].t().double()
            for l in range(8):
                idx, w = O.hash_indices(x, gf, l)
                ent = ((idx + int(gf.offset[l])) * 2)[:, :, None] + torch.arange(2, device=dev)
                fcomb.add(ent, w.double()[:, :, None] * dfi[:, None, 2 * l:2 * l + 2])
                if ferr is not None:
                    dfe = dfin_err[2 * l:2 * l + 2, h:h + CHUNK].t().double()
                    ferr.index_add_(0, ent.reshape(-1), (w.double()[:, :, None] * dfe[:, None, :]).reshape(-1))
        if not feats:
            continue

        d = dfeat[h:h + CHUNK].double()
        de = dfeat_err[h:h + CHUNK].double() if carry else torch.zeros_like(d)
        fl = flow[:, h:h + CHUNK].t().float()
        warped = {0: x, 1: x + fl[:, 0:3], 2: x + fl[:, 3:6]}                    # float32 adds, as the kernels

        # static hash: entry (offset[l] + idx) * 4 + f gets w_corner * dL/dfeature[row_hash_s + 4 l + f]
        for l in range(L):
            idx, w = O.hash_indices(x, gs, l)
            ent = ((idx + int(gs.offset[l])) * 4)[:, :, None] + ar4
            sl = slice(row_hash_s + 4 * l, row_hash_s + 4 * l + 4)
            wd = w.double()[:, :, None]
            static.add(ent, wd * d[:, None, sl], e=wd * de[:, None, sl])

        # dynamic hash, current query: one sum per entry; the time basis and slice weights are constants of the launch
        for p, (a, b) in enumerate(DYN_PAIRS):
            x2 = x[:, [a, b]]
            for l in range(L):
                idx, w = O.hash_indices(x2, gd[p], l)
                r = row_hash_d + p * L + l
                comb[p].add(idx + int(gd[p].offset[l]), w.double() * (wc * d[:, r:r + 1]), e=w.double() * (wc * de[:, r:r + 1]))

        for s in range(nS):
            R = cfg.min_resolution * cfg.plane_scales[s]
            # static planes: product rule over (x,y) (x,z) (y,z)
            ds, dse = d[:, s * 8:s * 8 + 8], de[:, s * 8:s * 8 + 8]
            samp = {}
            for ci in STATIC_PLANES:
                ca, cb = STATIC_COORDS[ci]
                bl = (axis(x[:, ca], R), axis(x[:, cb], R))
                vals, wgt, ys, xs = _texels(pl64[f"planes_encoder.planes.{s}.{ci}"], bl)
                samp[ci] = ((wgt[:, :, None] * vals).sum(1), (wgt[:, :, None] * vals.abs()).sum(1), wgt, ys, xs, R)
            for ci in STATIC_PLANES:
                o1, o2 = OTHER_STATIC[ci]
                g = ds * samp[o1][0] * samp[o2][0]
                ga = ds.abs() * samp[o1][1] * samp[o2][1]
                ge = dse * samp[o1][1] * samp[o2][1]
                _, _, wgt, ys, xs, W = samp[ci]
                ent = torch.arange(8, device=dev)[None, None, :] * (R * R) + (ys * W + xs)[:, :, None]
                planes[f"planes_encoder.planes.{s}.{ci}"].add(ent, wgt[:, :, None] * g[:, None, :], wgt[:, :, None] * ga[:, None, :],
                                                              wgt[:, :, None] * ge[:, None, :])
            # time planes (x,t) (y,t) (z,t) at every live query; the warped queries also give dL/dflow
            dt = d[:, row_plane_d + s * 8:row_plane_d + s * 8 + 8]
            dte = de[:, row_plane_d + s * 8:row_plane_d + s * 8 + 8]
            for qi, wq, q in queries:
                pos = warped[qi]
                tau = torch.full((1,), float(q.tau), dtype=torch.float32, device=dev)
                yb = axis(tau, T)
                yb = tuple(v.expand(C) for v in yb)
                samp = []
                for t, ci in enumerate(TIME_PLANES):
                    xb = axis(pos[:, t], R)
                    Pt = pl64[f"planes_encoder.planes.{s}.{ci}"]
                    vals, wgt, ys, xs = _texels(Pt, (xb, yb))
                    x0, x1, _, _, gx = xb
                    y0, y1, _, _, _ = yb
                    wy0, wy1 = yb[2].double()[:, None], yb[3].double()[:, None]
                    gxd = gx.double()[:, None]
                    # d(sample)/d(coordinate): gmult * sum_y wy * (P[y, x1] - P[y, x0]), as two terms per texel row
                    hi_ = wy0 * Pt[y0, x1] + wy1 * Pt[y1, x1]
                    lo_ = wy0 * Pt[y0, x0] + wy1 * Pt[y1, x0]
                    dx = gxd * (hi_ - lo_)
                    dxa = gxd * (wy0 * (Pt[y0, x1].abs() + Pt[y0, x0].abs()) + wy1 * (Pt[y1, x1].abs() + Pt[y1, x0].abs()))
                    samp.append(((wgt[:, :, None] * vals).sum(1), (wgt[:, :, None] * vals.abs()).sum(1), wgt, ys, xs, dx, dxa))
                for t, ci in enumerate(TIME_PLANES):
                    o1, o2 = [u for u in range(3) if u != t]
                    g = (wq * dt) * samp[o1][0] * samp[o2][0]
                    ga = (wq * dt).abs() * samp[o1][1] * samp[o2][1]
                    ge = (wq * dte) * samp[o1][1] * samp[o2][1]
                    _, _, wgt, ys, xs, dx, dxa = samp[t]
                    ent = torch.arange(8, device=dev)[None, None, :] * (T * R) + (ys * R + xs)[:, :, None]
                    planes[f"planes_encoder.planes.{s}.{ci}"].add(ent, wgt[:, :, None] * g[:, None, :], wgt[:, :, None] * ga[:, None, :],
                                                                  wgt[:, :, None] * ge[:, None, :])
                    if qi:
                        k = 3 * (qi - 1) + t
                        dflow[h:h + C, k, 0] += (g * dx).sum(1)
                        dflow[h:h + C, k, 1] += (ga * dxa).sum(1)
                        dflow[h:h + C, k, 2] += 16.0          # 8 channels x 2 texel columns
                        if carry:
                            dflow[h:h + C, k, 3] += (ge * dxa).sum(1)

    out = {}
    if feats:
        out["hash_encoder.hash_static.params"] = static.t
        out.update({k: v.t for k, v in planes.items()})
        cur = frame.cur
        for p in range(3):
            ne = int(gd[p].offset[-1])
            for sl in range(T):
                wsl = (1.0 if sl == cur.slice_lo else 0.0) if cur.single else \
                    (float(cur.w_lo) if sl == cur.slice_lo else (float(cur.w_hi) if sl == cur.slice_hi else 0.0))
                t = torch.zeros(ne, 4, comb[p].t.shape[1], dtype=torch.float64, device=dev)
                if wsl != 0.0:
                    for k in range(4):
                        t[:, k] = comb[p].scaled(wsl * float(cur.basis[k]))
                out[f"hash_encoder.hash_dynamic.{p}.hash_t.{sl}.params"] = t.view(ne * 4, -1)
        out["dflow"] = dflow
    if fcomb is not None:
        ne = int(gf.offset[-1])
        nc = 3 if ferr is None else 4
        t = torch.zeros(ne, 4, 2, nc, dtype=torch.float64, device=dev)
        fc = fcomb.t.view(ne, 2, 3)
        for i in range(4):
            bi = float(frame.flow_basis[i])
            t[:, i, :, 0] = fc[:, :, 0] * bi
            t[:, i, :, 1] = fc[:, :, 1] * abs(bi)
            t[:, i, :, 2] = fc[:, :, 2]
            if ferr is not None:
                t[:, i, :, 3] = ferr.view(ne, 2) * abs(bi)
        out["flow_net.grid_enc.params"] = t.view(-1, nc)
    return out


def check_entries(got: torch.Tensor, ref: torch.Tensor, slack: int = SLACK):
    """Per entry: |got - ref| <= (n + slack) * 2^-24 * A (+ the carried-in bound of a fourth column), and got == 0 where
    n == 0.
    Returns (number of failing entries, worst |got - ref| / bound, index of the worst entry)."""
    g = got.detach().reshape(-1).double()
    r, a, n = ref[..., 0].reshape(-1), ref[..., 1].reshape(-1), ref[..., 2].reshape(-1)
    assert g.numel() == r.numel(), (g.numel(), r.numel())
    err = (g - r).abs()
    bound = (n + slack) * EPS32 * a
    if ref.shape[-1] > 3:
        bound = bound + ref[..., 3].reshape(-1)
    bad = (err > bound) | ((n == 0) & (g != 0))
    ratio = torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    worst = int(torch.argmax(ratio))
    return int(bad.sum()), float(ratio[worst]), worst
