"""Float64 reference of the split forward's encoder stage (test infrastructure).

The encoders of the split pipeline (k_contract_dynamic, k_contract_planes, the flow-grid gather at the top of
k_fwd_flow_tc or k_fwd_gather, k_fwd_gather with its level-major l4d_static_sweep) make no decisions once the sample
positions and the flow are given: every value they write is a sum of products of table values and float32 weights.  This
module evaluates those sums in float64 and returns per value

    ref = the exact value,   A = sum of the magnitudes of the terms of its full expansion,   n = number of those terms,

so that a float32 result can be held to |got - ref| <= (n + 16) * 2^-24 * A, whatever the association order and wherever
nvcc contracts a multiply and an add.  Features carried as fp16 hi + lo (tensor-core mode) also carry the encoding's own
error, 2^-22 * |x| + 2^-25 (fp16 rounding of the residual x - hi, which is subnormal below |x| ~ 2^-3): see tile_bound.

The tables are the working values the kernels read: fp16(master) for the three hash grids, the fp32 planes.  The
positions and all weights are the kernels' float32 arithmetic (tests/scatter_ref.py: sample_x01, axis; corners from the
oracle's hash_indices), warped positions the float32 sums x01 + flow of the saved flow; only the products and the sums are
float64.  The contracted tables are expanded from the tables themselves, so a wrong contraction shows up in the features
too.

Feature order cat([plane_s, plane_d, hash_s, hash_d]) (oracle density(), lidar4d.py:155-176):
  plane_s (s, c)   product of the bilinear samples of planes (x,y) (x,z) (y,z)                     64 terms
  plane_d (s, c)   sum over live queries q of w_q * product of the row samples of (x,t) (y,t) (z,t)   64 per query
  hash_s (l, f)    8 corners                                                                        8
  hash_d (p, l)    sum_q w_q sum_corner w_c sum_k basis_k (w_lo T_lo,k + w_hi T_hi,k)             32 per query
with the current query at 0.5 and each neighbour at 0.25, a missing neighbour's share moved to the current query; a query
whose two slices coincide (`single`) reads its slice as the lo half of pair slice_lo, or, at the last slice, as the hi
half of pair T - 2.  Flow-MLP input 2l + j = sum_i basis_i sum_c w_c e_c[2i + j] (32 terms)."""
from __future__ import annotations

import numpy as np
import torch

from lidar4d_b200.geometry import make_frame
from oracle import lidar4d_oracle as O
from scatter_ref import (EPS32, SLACK, STATIC_PLANES, TIME_PLANES, STATIC_COORDS, DYN_PAIRS, axis, _texels)

CHUNK = 1 << 18                   # samples per pass: [CHUNK, K] float64 temporaries of ~370 MB at K = 176
ENC_REL = 2.0 ** -22              # fp16 hi + lo: rounding of the residual, relative ...
ENC_ABS = 2.0 ** -25              # ... and half the spacing of fp16's subnormals


def _fp16(t: torch.Tensor) -> torch.Tensor:
    return t.detach().float().half().double()


def time_pair(q, T: int):
    """l4d_time_pair and the pair weights of l4d_contract_entry: (pair, w_lo, w_hi)."""
    pair = q.slice_lo if q.slice_lo < T - 1 else T - 2
    if q.single:
        wl = 1.0 if q.slice_lo == pair else 0.0
        return pair, wl, 1.0 - wl
    return pair, float(q.w_lo), float(q.w_hi)


def queries(frame):
    """[(index, aggregation weight, TimeQuery)] of the live queries (l4d_agg_weights)."""
    wc = 0.5 + (0.0 if frame.has_fwd else 0.25) + (0.0 if frame.has_bwd else 0.25)
    out = [(0, wc, frame.cur)]
    if frame.has_fwd:
        out.append((1, 0.25, frame.fwd))
    if frame.has_bwd:
        out.append((2, 0.25, frame.bwd))
    return out


def special_times(cfg):
    """An interior frame time whose current query is `single` (tau (T - 1) an integer) and one whose time coordinate lies on
    a time-texel row (wy1 = 0 in the kernels' float32 arithmetic), searched among the float32 neighbours of k / (T - 1)."""
    T = cfg.time_resolution
    single = row = None
    for k in range(1, T - 1):
        c = np.float32(k / (T - 1))
        for t in (c, np.nextafter(c, np.float32(0)), np.nextafter(c, np.float32(1))):
            fr = make_frame(float(t), cfg.num_frames, cfg.time_resolution)
            if single is None and fr.cur.single and 0 < fr.cur.slice_lo < T - 1:
                single = float(t)
            if row is None and float(axis(torch.tensor([float(t)]), T)[3]) == 0.0:
                row = float(t)
    assert single is not None and row is not None
    return single, row


class Tables:
    """The working tables in float64 and the float64 contractions of the launch (what k_contract_dynamic and
    k_contract_planes should write), each as (ref, A); n is 8 per hd_con entry and 2 per pl_con entry."""

    def __init__(self, cfg, params: dict, frame):
        self.cfg, self.frame = cfg, frame
        T = cfg.time_resolution
        self.hs = _fp16(params["hash_encoder.hash_static.params"]).view(-1, 4)
        self.hf = _fp16(params["flow_net.grid_enc.params"]).view(-1, 8)
        self.planes = {}
        for s in range(cfg.n_levels_plane):
            for ci in range(6):
                self.planes[s, ci] = params[f"planes_encoder.planes.{s}.{ci}"].detach()[0].permute(1, 2, 0).double()
        self.hd_con, self.pl_con = {}, {}
        for qi, _, q in queries(frame):
            pair, wl, wh = time_pair(q, T)
            b = torch.tensor([float(v) for v in q.basis], dtype=torch.float64, device=self.hs.device)
            for p in range(3):
                name = f"hash_encoder.hash_dynamic.{p}.hash_t.%d.params"
                lo = _fp16(params[name % pair]).view(-1, 4)
                hi = _fp16(params[name % (pair + 1)]).view(-1, 4)
                terms = torch.cat([(b * wl) * lo, (b * wh) * hi], 1)
                self.hd_con[qi, p] = (terms.sum(1), terms.abs().sum(1))
            tau = torch.full((1,), float(q.tau), dtype=torch.float32, device=self.hs.device)
            y0, y1, wy0, wy1, _ = axis(tau, T)
            y0, y1, wy0, wy1 = int(y0), int(y1), float(wy0), float(wy1)
            for s in range(cfg.n_levels_plane):
                for t, ci in enumerate(TIME_PLANES):
                    Pt = self.planes[s, ci]
                    a, c = wy0 * Pt[y0], wy1 * Pt[y1]
                    self.pl_con[qi, s, t] = (a + c, a.abs() + c.abs())


def feature_terms(cfg, frame) -> torch.Tensor:
    """n of every feature column [sigma_in_dim] (float64)."""
    nS, L, nq = cfg.n_levels_plane, cfg.n_levels_hash, len(queries(frame))
    return torch.tensor([64] * (8 * nS) + [64 * nq] * (8 * nS) + [8] * (4 * L) + [32 * nq] * (3 * L), dtype=torch.float64)


FLOW_TERMS = 32


def gather_reference(tabs: Tables, x01: torch.Tensor, flow: torch.Tensor, on_chunk, chunk: int = CHUNK):
    """Float64 features and flow-MLP inputs of every sample, chunk by chunk.

    x01 [P, 3] float32 (sample_x01); flow [6, P] float32 (the forward's, for the warped positions).
    on_chunk(p0, p1, {"features": (ref [C, K], A [C, K]), "flow_in": (ref [C, 16], A [C, 16])}) per chunk; n of the
    features is feature_terms(), of the flow-MLP inputs FLOW_TERMS."""
    cfg, frame = tabs.cfg, tabs.frame
    dev = x01.device
    P = x01.shape[0]
    nS, L = cfg.n_levels_plane, cfg.n_levels_hash
    K = cfg.sigma_in_dim
    row_plane_d, row_hash_s = nS * 8, 2 * nS * 8
    row_hash_d = row_hash_s + 4 * L
    gs, gf = cfg.static_grid(), cfg.flow_grid()
    gd = [cfg.dynamic_grid(p) for p in range(3)]
    qs = queries(frame)
    fb = torch.tensor([float(v) for v in frame.flow_basis], dtype=torch.float64, device=dev)

    for h in range(0, P, chunk):
        x = x01[h:h + chunk].float()
        C = x.shape[0]
        fl = flow[:, h:h + chunk].t().float()
        warped = {0: x, 1: x + fl[:, 0:3], 2: x + fl[:, 3:6]}                    # float32 adds, as the kernels
        ref = torch.empty(C, K, dtype=torch.float64, device=dev)
        mag = torch.empty_like(ref)

        for s in range(nS):
            R = cfg.min_resolution * cfg.plane_scales[s]
            # static planes: product of three bilinear samples
            r, a = 1.0, 1.0
            for ci in STATIC_PLANES:
                ca, cb = STATIC_COORDS[ci]
                vals, wgt, _, _ = _texels(tabs.planes[s, ci], (axis(x[:, ca], R), axis(x[:, cb], R)))
                r = r * (wgt[:, :, None] * vals).sum(1)
                a = a * (wgt[:, :, None] * vals).abs().sum(1)
            ref[:, s * 8:s * 8 + 8], mag[:, s * 8:s * 8 + 8] = r, a
            # time planes: per live query, the product of the row samples of the three contracted rows
            rd = torch.zeros(C, 8, dtype=torch.float64, device=dev)
            ad = torch.zeros_like(rd)
            for qi, wq, _ in qs:
                r, a = 1.0, 1.0
                for t in range(3):
                    x0, x1, wx0, wx1, _ = axis(warped[qi][:, t], R)
                    cr, ca_ = tabs.pl_con[qi, s, t]
                    w0, w1 = wx0.double()[:, None], wx1.double()[:, None]
                    r = r * (w0 * cr[x0] + w1 * cr[x1])
                    a = a * (w0.abs() * ca_[x0] + w1.abs() * ca_[x1])
                rd += wq * r
                ad += wq * a
            ref[:, row_plane_d + s * 8:row_plane_d + s * 8 + 8], mag[:, row_plane_d + s * 8:row_plane_d + s * 8 + 8] = rd, ad

        # static hash: 8 corners per level
        for l in range(L):
            idx, w = O.hash_indices(x, gs, l)
            v = tabs.hs[idx + int(gs.offset[l])]                                 # [C, 8, 4]
            t = w.double()[:, :, None] * v
            ref[:, row_hash_s + 4 * l:row_hash_s + 4 * l + 4] = t.sum(1)
            mag[:, row_hash_s + 4 * l:row_hash_s + 4 * l + 4] = t.abs().sum(1)

        # dynamic hash: per live query, 4 corners of the float64 contraction of the query's pair records
        for p, (a_, b_) in enumerate(DYN_PAIRS):
            for l in range(L):
                r = torch.zeros(C, dtype=torch.float64, device=dev)
                a = torch.zeros_like(r)
                for qi, wq, _ in qs:
                    idx, w = O.hash_indices(warped[qi][:, [a_, b_]], gd[p], l)
                    cr, ca_ = tabs.hd_con[qi, p]
                    e = idx + int(gd[p].offset[l])
                    wd = w.double()
                    r += wq * (wd * cr[e]).sum(1)
                    a += wq * (wd.abs() * ca_[e]).sum(1)
                ref[:, row_hash_d + p * L + l], mag[:, row_hash_d + p * L + l] = r, a

        # flow-MLP inputs: input 2l + j = sum_i basis_i sum_c w_c e_c[2i + j]
        fr = torch.empty(C, 16, dtype=torch.float64, device=dev)
        fa = torch.empty_like(fr)
        for l in range(8):
            idx, w = O.hash_indices(x, gf, l)
            e = tabs.hf[idx + int(gf.offset[l])].view(C, 8, 4, 2)               # [C, corner, i, j]
            t = w.double()[:, :, None, None] * fb[None, None, :, None] * e
            fr[:, 2 * l:2 * l + 2] = t.sum((1, 2))
            fa[:, 2 * l:2 * l + 2] = t.abs().sum((1, 2))
        on_chunk(h, h + C, {"features": (ref, mag), "flow_in": (fr, fa)})


def bound32(A: torch.Tensor, n, slack: int = SLACK) -> torch.Tensor:
    """(n + slack) * 2^-24 * A: a float32 evaluation of a sum of n products, in any order, with or without fma."""
    return (torch.as_tensor(n, dtype=torch.float64, device=A.device) + slack) * EPS32 * A


def tile_bound(ref: torch.Tensor, A: torch.Tensor, n) -> torch.Tensor:
    """Bound of hi + lo, the fp16 pair that carries a float32 feature x: bound32 plus fp16 rounding of the residual
    x - hi, relative 2^-22 of |x| and absolute 2^-25 where the residual is an fp16 subnormal."""
    b = bound32(A, n)
    return b + ENC_REL * (ref.abs() + b) + ENC_ABS


def ratio(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> torch.Tensor:
    """|got - ref| / bound, inf where the bound is 0 and got differs (NaN counts as a failure)."""
    err = (got.double() - ref).abs()
    r = torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    return torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)


def check_table(got: torch.Tensor, ref_a, n: int):
    """A contracted table against (ref, A): (number of failing entries, worst fraction of the bound, entries)."""
    ref, A = ref_a
    r = ratio(got.reshape(ref.shape), ref, bound32(A, n))
    return int((r > 1).sum()), float(r.max()), r.numel()


# ---- the fp16 hi + lo operand tiles ------------------------------------------------------------------------------------
def ulp16(h: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 at h (float64): 2^(e - 10) for normal |h| in [2^e, 2^(e+1)), 2^-24 below 2^-14."""
    a = h.double().abs()
    e = torch.frexp(a).exponent.double() - 1                    # a = m 2^(e + 1), m in [0.5, 1)
    return torch.where(a >= 2.0 ** -14, torch.exp2(e - 10), torch.full_like(a, 2.0 ** -24))


def tile_rows(cfg, tiles: torch.Tensor, S: int):
    """feat_tiles [N][nt][hi|lo][k/8][128][8] -> hi, lo [N, nt * 128, 8 * x_chunks] (fp16; rows >= S are padding)."""
    N, nt, _, xc = tiles.shape[:4]
    t = tiles.permute(0, 1, 4, 2, 3, 5).reshape(N, nt * 128, 2, xc * 8)
    return t[:, :, 0], t[:, :, 1]


def check_tile_structure(cfg, tiles: torch.Tensor, S: int, rays_per_pass: int = 256) -> dict:
    """Structural checks of the operand tiles; returns counts of violations per check (all must be 0):
      nonfinite  an inf or NaN anywhere in a tile;
      padding    a row j >= S of a ray's last tile that is not +0 in both halves;
      ones       a column sigma_in_dim .. 8 x_chunks - 1 of a live row whose hi is not 1.0 or whose lo is not +0;
      split      a live feature whose |lo| exceeds half an fp16 ulp of hi, or whose hi is not a nearest fp16 value of
                 hi + lo: fp16_rn(hi + lo) == hi, except at an exact tie |lo| = ulp(hi) / 2, where round-to-even of the
                 sum may pick the other neighbour (fp16_rn of a residual just below half an ulp can round up to it)."""
    K = cfg.sigma_in_dim
    out = dict(nonfinite=0, padding=0, ones=0, split=0)
    for r0 in range(0, tiles.shape[0], rays_per_pass):
        hi, lo = tile_rows(cfg, tiles[r0:r0 + rays_per_pass], S)
        out["nonfinite"] += int((~torch.isfinite(hi)).sum() + (~torch.isfinite(lo)).sum())
        out["padding"] += int((hi[:, S:].view(torch.int16) != 0).sum() + (lo[:, S:].view(torch.int16) != 0).sum())
        out["ones"] += int((hi[:, :S, K:] != 1.0).sum() + (lo[:, :S, K:].view(torch.int16) != 0).sum())
        h, l = hi[:, :S, :K], lo[:, :S, :K]
        half = 0.5 * ulp16(h)
        la = l.double().abs()
        back = (h.float() + l.float()).half()                   # hi + lo is exact in float32
        out["split"] += int(((la > half) | ((back != h) & (la != half))).sum())
    return out


def emulate_tile_emit(x: np.ndarray):
    """l4d_tile_emit's split of float32 values: hi = fp16_rn(x), lo = fp16_rn(x - hi) (x - hi is exact in float32)."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo
