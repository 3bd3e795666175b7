"""ORACLE (test infrastructure, NOT product code) - CPU restatement of the
LiDAR4D per-ray volume-rendering hot path in plain PyTorch.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this.  The product (lidar4d_b200/) never does and
fails loudly when its CUDA library is missing.

Parity status: **parity unpinned by upstream tests** - the reference ships no
tests or golden vectors for this path and its arithmetic for hash grids /
frequency encoding / fused MLPs lives in tiny-cuda-nn (un-vendored, un-pinned:
/root/reference/README.md:88-91).  This oracle is pinned instead against the
reference's *own* python modules (renderer.py, planes_field.py, lidar4d.py,
hash_field.py, flow_field.py, imported unchanged) running on top of
oracle/tcnn_shim.py in the build container; tests/golden/make_golden.py is the
generating script and tests/golden/*.npz the committed vectors.

Numeric spec ("L4D spec v1", SURVEY.md §8(c)):
  * hash tables: fp32 master params, fp16-rounded working values (as tcnn),
    corner weights and blends in fp32 (tcnn blends in fp16 - we are more exact)
  * pos = fmaf(scale_l, x, 0.5) with a single rounding; uint32 hash
    (c0*1) ^ (c1*2654435761) ^ (c2*805459861); dense index when the level fits
  * planes: fp32, F.grid_sample(bilinear, align_corners=True, border)
  * MLPs: bias-free, inputs padded to x16 with 1.0, fp32 math
  * compositing fp32 exactly as model/renderer.py:98-129
Each function cites the reference lines it restates (paths relative to
/root/reference).
"""
from __future__ import annotations

import itertools
import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from lidar4d_b200.geometry import (FieldConfig, FrameConstants, GridGeometry, TimeQuery,
                                   make_frame, HASH_PRIMES)

PI32 = float(np.float32(np.pi))
HALF_PI32 = float(np.float32(np.pi / 2))


# =============================================================================
# tiny-cuda-nn semantics [tcnn-ext]  (spec: SURVEY.md §8(c))
# =============================================================================
def hash_indices(x: torch.Tensor, geo: GridGeometry, level: int):
    """uint32 corner indices + fp32 corner weights of one level.

    tcnn kernel_grid / grid_index [tcnn-ext]; call sites hash_field.py:47-57,
    :107-117, flow_field.py:67-77.  Returns (idx int64 [N, 2^D] already taken
    modulo the level's entries, w float32 [N, 2^D]).
    """
    D = geo.n_dims
    assert x.shape[-1] == D
    scale = float(geo.scale[level])
    res = int(geo.resolution[level])
    entries = int(geo.entries[level])
    # pos = fmaf(scale, x, 0.5f): exact in float64, one rounding to float32
    pos = (x.detach().to(torch.float64) * scale + 0.5).to(torch.float32)
    g = torch.floor(pos)
    w = pos - g                                           # fp32
    cell = g.to(torch.int64) & 0xFFFFFFFF                 # (uint32)(int)floorf(pos)
    idx_list, w_list = [], []
    for corner in range(1 << D):
        wc = None
        c = []
        for d in range(D):
            if (corner >> d) & 1:
                f = w[:, d]
                c.append((cell[:, d] + 1) & 0xFFFFFFFF)
            else:
                f = 1.0 - w[:, d]
                c.append(cell[:, d])
            wc = f if wc is None else wc * f
        # grid_index: dense stride walk while stride <= hashmap_size
        stride, index, d = 1, torch.zeros_like(c[0]), 0
        while d < D and stride <= entries:
            index = (index + c[d] * stride) & 0xFFFFFFFF
            stride = (stride * res) & 0xFFFFFFFF          # uint32 wrap like the C++ code
            d += 1
        if entries < stride:                              # hashed level
            index = torch.zeros_like(c[0])
            for dd in range(D):
                index = index ^ ((c[dd] * HASH_PRIMES[dd]) & 0xFFFFFFFF)
        idx_list.append(index % entries)
        w_list.append(wc)
    return torch.stack(idx_list, -1), torch.stack(w_list, -1)


def working_table(params: torch.Tensor, table_dtype: str) -> torch.Tensor:
    """fp16-rounded working copy with straight-through gradient to the fp32
    master (tcnn keeps fp32 masters and casts per call [tcnn-ext])."""
    if table_dtype == "fp32":
        return params
    q = params.detach().to(torch.float32).to(torch.float16).to(params.dtype)
    return params + (q - params.detach())


def hash_encode(x: torch.Tensor, params: torch.Tensor, geo: GridGeometry,
                table_dtype: str = "fp16", compute_dtype=torch.float32) -> torch.Tensor:
    """tcnn HashGrid forward: [N,D] -> [N, L*F] level-major."""
    Fd = geo.n_features
    table = working_table(params, table_dtype).view(-1, Fd)
    outs = []
    for l in range(geo.n_levels):
        idx, w = hash_indices(x, geo, l)
        rows = table[(idx + int(geo.offset[l])).reshape(-1)].view(idx.shape[0], idx.shape[1], Fd)
        outs.append((rows.to(compute_dtype) * w.to(compute_dtype).unsqueeze(-1)).sum(1))
    return torch.cat(outs, -1)


def frequency_encode(x: torch.Tensor, degree: int) -> torch.Tensor:
    """tcnn Frequency encoding [tcnn-ext]: out[:, dim*2n + 2k + {0:sin,1:cos}]
    = sin(2^k*pi*x + phase), fp32 with mul-then-add (no fma)."""
    N, D = x.shape
    out = []
    for dim in range(D):
        for k in range(degree):
            xs = x[:, dim] * float(2 ** k)
            for p in range(2):
                arg = xs * PI32 + (HALF_PI32 if p else 0.0)
                out.append(torch.sin(arg))
    return torch.stack(out, -1)


def mlp_layers(params: torch.Tensor, n_in_pad: int, hidden: int, n_hidden_layers: int,
               n_out_pad: int = 16) -> List[torch.Tensor]:
    """Split a tcnn FullyFusedMLP flat param vector into [out,in] matrices."""
    mats, o = [], 0
    dims = [n_in_pad] + [hidden] * n_hidden_layers + [n_out_pad]
    for i in range(len(dims) - 1):
        n = dims[i + 1] * dims[i]
        mats.append(params[o:o + n].view(dims[i + 1], dims[i]))
        o += n
    assert o == params.numel()
    return mats


def fused_mlp(x: torch.Tensor, params: torch.Tensor, n_in: int, n_out: int, hidden: int,
              n_hidden_layers: int, weight_dtype: str = "fp32") -> torch.Tensor:
    """tcnn FullyFusedMLP [tcnn-ext]: pad inputs with ones to x16, ReLU hidden,
    linear output padded to 16 and sliced.  fp32 math."""
    n_in_pad = (n_in + 15) // 16 * 16
    mats = mlp_layers(working_table(params, weight_dtype), n_in_pad, hidden, n_hidden_layers)
    if n_in_pad > n_in:
        x = torch.cat([x, torch.ones(x.shape[0], n_in_pad - n_in, dtype=x.dtype, device=x.device)], -1)
    h = x
    for i, W in enumerate(mats):
        h = h @ W.to(h.dtype).t()
        if i < len(mats) - 1:
            h = torch.relu(h)
    return h[:, :n_out]


class _TruncExp(torch.autograd.Function):
    """model/activation.py:6-20."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(-15, 15))


trunc_exp = _TruncExp.apply


def _texel_axis(u: torch.Tensor, size: int):
    """One axis of F.grid_sample(bilinear, align_corners=True, border) for a float64 coordinate u in [0, 1]: the texel
    pair is chosen from the float32 value of the coordinate by grid_sample's float32 arithmetic, the weights are float64
    (and differentiable).  A warped position x + flow within float32 rounding of a texel edge therefore falls in the
    texel the float32 evaluation picks, where d(sample)/d(position) is that texel's slope."""
    m = float(size - 1)
    ix32 = (u.detach().float() * 2.0 - 1.0 + 1.0) / 2.0 * m
    ix = (u * 2.0 - 1.0 + 1.0) / 2.0 * m
    inside = (ix32 > 0.0) & (ix32 < m)                 # border padding: no gradient on or beyond the edge texels
    ix = torch.where(inside, ix, ix.detach().clamp(0.0, m))
    ix32 = ix32.clamp(0.0, m)
    i0 = torch.floor(ix32).long().clamp(max=size - 1)
    i1 = (i0 + 1).clamp(max=size - 1)
    w1 = ix - i0.to(ix.dtype)
    return i0, i1, 1.0 - w1, w1


def _grid_sample_texels32(grid: torch.Tensor, cx: torch.Tensor, cy: torch.Tensor) -> torch.Tensor:
    """Bilinear sample of grid [1, C, H, W] at (cx -> W, cy -> H) in [0, 1]: [P, C], texels selected as in float32."""
    _, C, H, W = grid.shape
    x0, x1, wx0, wx1 = _texel_axis(cx, W)
    y0, y1, wy0, wy1 = _texel_axis(cy, H)
    g = grid[0]
    return ((g[:, y0, x0] * (wx0 * wy0) + g[:, y0, x1] * (wx1 * wy0)) +
            (g[:, y1, x0] * (wx0 * wy1) + g[:, y1, x1] * (wx1 * wy1))).t()


# =============================================================================
# counter-based jitter RNG shared with the CUDA kernels (spec of this repo; the
# reference uses torch.rand, renderer.py:84, which no other code can reproduce)
# =============================================================================
def jitter_uniform(seed: int, ray_index: np.ndarray, n_steps: int) -> np.ndarray:
    """u[ray, j] in [0,1): splitmix64 of (seed, global ray index, sample index)."""
    ray = ray_index.astype(np.uint64).reshape(-1, 1)
    j = np.arange(n_steps, dtype=np.uint64).reshape(1, -1)
    with np.errstate(over="ignore"):
        z = (ray << np.uint64(32)) | j
        z = z + np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return ((z >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)).astype(np.float32)


def sample_lin(n_steps: int) -> np.ndarray:
    """torch.linspace(0,1,S) exactly as the CUDA kernel computes it (the reference renders on the GPU,
    renderer.py:77): step*j below the midpoint, fma(-step, S-1-j, 1) - ONE rounding - above it.  Pinned against the
    real thing: tests/golden/cuda_linspace.npz was dumped from torch.linspace(device="cuda") on a GPU."""
    if n_steps < 2:                                  # torch.linspace(0, 1, 1) == [0.]
        return np.zeros(n_steps, np.float32)
    step = np.float32(1.0) / np.float32(n_steps - 1)
    j = np.arange(n_steps)
    lo = (step * j.astype(np.float32)).astype(np.float32)
    hi = (1.0 - np.float64(step) * (n_steps - 1 - j).astype(np.float64)).astype(np.float32)   # exact product, one rounding
    return np.where(j < n_steps // 2, lo, hi).astype(np.float32)


# =============================================================================
# the model
# =============================================================================
class OracleLiDAR4D(nn.Module):
    """Same parameter names / shapes as the reference LiDAR4D.state_dict()
    (SURVEY.md §8(b)), so state dicts move freely between the reference-on-shim
    model, this oracle and the CUDA module."""

    def __init__(self, cfg: Optional[FieldConfig] = None, table_dtype: str = "fp16", **kw):
        super().__init__()
        self.cfg = cfg or FieldConfig(**kw)
        c = self.cfg
        c.validate()
        self.table_dtype = table_dtype
        self.mlp_dtype = "fp32"          # "fp16": MLP weights as fp16-rounded working copies (tcnn keeps half params)
        self.cd = torch.float32          # compute dtype; float64 = "truth" mode (see to_float64)
        self.g_static = c.static_grid()
        self.g_dynamic = [c.dynamic_grid(p) for p in range(3)]
        self.g_flow = c.flow_grid()

        P = nn.ParameterDict()
        # planes_field.py:32-53 init_grid_param, :169-190 multi-scale
        self.coo_combs = list(itertools.combinations(range(4), 2))
        for s, mult in enumerate(c.plane_scales):
            reso = [c.min_resolution * mult] * 3 + [c.time_resolution]
            for ci, comb in enumerate(self.coo_combs):
                shape = [1, c.n_features_per_level_plane] + [reso[cc] for cc in comb[::-1]]
                t = torch.empty(shape)
                if 3 in comb:
                    nn.init.ones_(t)
                else:
                    nn.init.uniform_(t, a=0.1, b=0.5)
                P[f"planes_encoder.planes.{s}.{ci}".replace(".", "/")] = nn.Parameter(t)
        P["hash_encoder/hash_static/params"] = nn.Parameter(
            torch.empty(self.g_static.n_params).uniform_(-1e-4, 1e-4))
        for p in range(3):
            for s in range(c.time_resolution):
                P[f"hash_encoder/hash_dynamic/{p}/hash_t/{s}/params"] = nn.Parameter(
                    torch.empty(self.g_dynamic[p].n_params).uniform_(-1e-4, 1e-4))
        P["view_encoder/params"] = nn.Parameter(torch.zeros(0))
        P["flow_net/grid_enc/params"] = nn.Parameter(
            torch.empty(self.g_flow.n_params).uniform_(-1e-4, 1e-4))
        fin = c.flow_n_levels * c.flow_n_features // 4
        dims = [fin, c.hidden_dim_flow, c.hidden_dim_flow, 6]
        for li, idx in enumerate([0, 2, 4]):
            lin = nn.Linear(dims[li], dims[li + 1], bias=False)
            if li == 2:
                nn.init.normal_(lin.weight.data, 0, 0.001)     # flow_field.py:100
            P[f"flow_net/mlp/{idx}/weight"] = nn.Parameter(lin.weight.data.clone())
        P["sigma_net/params"] = nn.Parameter(self._xavier_mlp(c.sigma_in_pad, 64, 1))
        P["intensity_net/params"] = nn.Parameter(self._xavier_mlp(c.attr_in_pad, 64, 2))
        P["raydrop_net/params"] = nn.Parameter(self._xavier_mlp(c.attr_in_pad, 64, 2))
        self.P = P
        b = c.bound
        self.register_buffer("aabb", torch.tensor([-b, -b, -b, b, b, b], dtype=torch.float32))

    # -- naming ---------------------------------------------------------------
    @staticmethod
    def _xavier_mlp(n_in_pad, hidden, n_hidden_layers, n_out_pad=16):
        dims = [n_in_pad] + [hidden] * n_hidden_layers + [n_out_pad]
        chunks = []
        for i in range(len(dims) - 1):
            s = math.sqrt(6.0 / (dims[i] + dims[i + 1]))
            chunks.append(torch.empty(dims[i + 1] * dims[i]).uniform_(-s, s))
        return torch.cat(chunks)

    def p(self, name: str) -> torch.Tensor:
        return self.P[name.replace(".", "/")]

    def to_float64(self) -> "OracleLiDAR4D":
        """Truth mode: parameters and all smooth arithmetic in float64.  The
        quantities the spec pins in float32 (sample positions, x01, hash cell
        selection / corner weights, the frequency-encoding argument, fp16 table
        rounding, the plane texel that each position - warped positions x + flow included - falls in) stay exactly
        as in float32, so this is the infinitely-precise
        evaluation of the SAME function; use it to tell which of two float32
        results is the noisy one."""
        self.double()
        self.cd = torch.float64
        return self

    def ref_state_dict(self) -> Dict[str, torch.Tensor]:
        """state_dict with the reference's key names."""
        d = {k.replace("/", "."): v.detach().clone() for k, v in self.P.items()}
        d["aabb"] = self.aabb.clone()
        return d

    def load_ref_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        with torch.no_grad():
            for k, v in self.P.items():
                key = k.replace("/", ".")
                if key in sd:
                    v.copy_(sd[key].to(v.dtype).view_as(v))

    def ref_named_grads(self) -> Dict[str, torch.Tensor]:
        return {k.replace("/", "."): (v.grad.detach().clone() if v.grad is not None
                                      else torch.zeros_like(v)) for k, v in self.P.items()}

    # -- encoders -------------------------------------------------------------
    def interp_t(self, feat: torch.Tensor, n_levels: int, n_feat: int, basis) -> torch.Tensor:
        """hash_field.py:65-74 / flow_field.py:102-111: view [N,L,F], chunk F
        into 4 node groups, sum_i L_i(t)*chunk_i, flatten level-major."""
        x = feat.view(-1, n_levels, n_feat)
        chunks = torch.chunk(x, 4, dim=-1)
        out = None
        for i in range(4):
            term = float(basis[i]) * chunks[i]
            out = term if out is None else out + term
        return out.reshape(feat.shape[0], -1)

    def hash_static(self, x01):
        """hash_field.py:141-144."""
        return hash_encode(x01, self.p("hash_encoder.hash_static.params"), self.g_static, self.table_dtype, self.cd)

    def hash_dynamic(self, x, q: TimeQuery):
        """hash_field.py:146-158 with HashGridT.forward :76-88."""
        c = self.cfg
        pairs = [(0, 1), (0, 2), (1, 2)]
        outs = []
        for p, (a, b) in enumerate(pairs):
            x2 = x[:, [a, b]]
            name = f"hash_encoder.hash_dynamic.{p}.hash_t.%d.params"
            f_lo = hash_encode(x2, self.p(name % q.slice_lo), self.g_dynamic[p], self.table_dtype, self.cd)
            if q.single:
                f = f_lo
            else:
                f_hi = hash_encode(x2, self.p(name % q.slice_hi), self.g_dynamic[p], self.table_dtype, self.cd)
                f = float(q.w_lo) * f_lo + float(q.w_hi) * f_hi
            outs.append(self.interp_t(f, c.n_levels_hash, c.n_features_per_level_hash, q.basis))
        return torch.cat(outs, -1)

    def _plane(self, s, ci):
        return self.p(f"planes_encoder.planes.{s}.{ci}")

    def planes(self, xt: torch.Tensor, which: str):
        """planes_field.py:87-141 interpolate_ms_features with
        grid_sample_wrapper :56-84 (bilinear, align_corners=True, border), product over
        the 3 static / 3 dynamic planes per scale, concat over scales."""
        feats = []
        for s in range(self.cfg.n_levels_plane):
            prod = None
            for ci, comb in enumerate(self.coo_combs):
                dyn = 3 in comb
                if dyn != (which == "dynamic"):
                    continue
                grid = self._plane(s, ci)
                if xt.dtype == torch.float64:
                    v = _grid_sample_texels32(grid.to(xt.dtype), xt[:, comb[0]], xt[:, comb[1]])
                else:
                    coords = xt[:, list(comb)].view(1, 1, -1, 2) * 2.0 - 1
                    v = F.grid_sample(grid.to(xt.dtype), coords, align_corners=True, mode="bilinear",
                                      padding_mode="border")
                    v = v.view(grid.shape[1], -1).t()
                prod = v if prod is None else prod * v
            feats.append(prod)
        return torch.cat(feats, -1)

    def flow_field(self, x01: torch.Tensor, basis) -> torch.Tensor:
        """flow_field.py:113-130: grid -> interpT at the frame time -> 3 bias-free Linear."""
        c = self.cfg
        e = hash_encode(x01, self.p("flow_net.grid_enc.params"), self.g_flow, self.table_dtype, self.cd)
        h = self.interp_t(e, c.flow_n_levels, c.flow_n_features, basis)
        self._dbg_flow_in = h
        W = lambda n: working_table(self.p(n), self.mlp_dtype)
        h = torch.relu(h @ W("flow_net.mlp.0.weight").t())
        h = torch.relu(h @ W("flow_net.mlp.2.weight").t())
        return h @ W("flow_net.mlp.4.weight").t()

    # -- LiDAR4D.flow / density / attribute ------------------------------------
    def flow(self, x: torch.Tensor, t) -> Dict[str, torch.Tensor]:
        """lidar4d.py:124-137."""
        b = self.cfg.bound
        x01 = (x.float() + b) / (2 * b)
        fr = make_frame(float(t), self.cfg.num_frames, self.cfg.time_resolution)
        fl = self.flow_field(x01, fr.flow_basis)
        return {"forward": fl[:, :3], "backward": fl[:, 3:]}

    def density(self, x: torch.Tensor, fr: FrameConstants, return_features=False):
        """lidar4d.py:139-188."""
        c = self.cfg
        b = c.bound
        x01 = ((x.float() + b) / (2 * b)).to(self.cd)      # float32 arithmetic (lidar4d.py:141), then promote
        N = x01.shape[0]
        hash_s = self.hash_static(x01)
        hash_d = self.hash_dynamic(x01, fr.cur)
        tcol = torch.full((N, 1), float(fr.time), dtype=x01.dtype, device=x01.device)
        xt = torch.cat([x01, tcol], -1)
        plane_s = self.planes(xt, "static")
        plane_d = self.planes(xt, "dynamic")
        flow = self.flow_field(x01, fr.flow_basis)
        hash_1 = hash_2 = hash_d
        plane_1 = plane_2 = plane_d
        if fr.has_fwd:
            x1 = x01 + flow[:, :3]
            with torch.no_grad():
                hash_1 = self.hash_dynamic(x1, fr.fwd)
            xt1 = torch.cat([x1, torch.full((N, 1), float(fr.fwd.tau), dtype=x01.dtype, device=x01.device)], -1)
            plane_1 = self.planes(xt1, "dynamic")
        if fr.has_bwd:
            x2 = x01 + flow[:, 3:]
            with torch.no_grad():
                hash_2 = self.hash_dynamic(x2, fr.bwd)
            xt2 = torch.cat([x2, torch.full((N, 1), float(fr.bwd.tau), dtype=x01.dtype, device=x01.device)], -1)
            plane_2 = self.planes(xt2, "dynamic")
        plane_d = 0.5 * plane_d + 0.25 * (plane_1 + plane_2)
        hash_d = 0.5 * hash_d + 0.25 * (hash_1 + hash_2)
        feats = torch.cat([plane_s, plane_d, hash_s, hash_d], -1)
        h = fused_mlp(feats, self.p("sigma_net.params"), c.sigma_in_dim, 1 + c.geo_feat_dim, 64, 1, self.mlp_dtype)
        sigma = trunc_exp(h[:, 0])
        geo = h[:, 1:]
        out = {"sigma": sigma, "geo_feat": geo}
        if return_features:
            out.update(features=feats, flow=flow, flow_in=self._dbg_flow_in)
        return out

    def attribute(self, d: torch.Tensor, geo: torch.Tensor, mask: Optional[torch.Tensor]):
        """lidar4d.py:191-223 (x is unused by the reference's attribute heads)."""
        c = self.cfg
        N = d.shape[0]
        out = torch.zeros(N, c.out_lidar_dim, dtype=self.cd, device=d.device)
        if mask is not None:
            if not bool(mask.any()):
                return out
            d, geo = d[mask], geo[mask]
        enc = frequency_encode((d.float() + 1) / 2, c.view_degree).to(self.cd)
        inp = torch.cat([enc, geo], -1)
        inten = torch.sigmoid(fused_mlp(inp, self.p("intensity_net.params"), c.attr_in_dim, 1, 64, 2, self.mlp_dtype))
        drop = torch.sigmoid(fused_mlp(inp, self.p("raydrop_net.params"), c.attr_in_dim, 1, 64, 2, self.mlp_dtype))
        h = torch.cat([drop, inten], -1)
        if mask is not None:
            out[mask] = h.to(out.dtype)                    # lidar4d.py:219 (fp16 under autocast -> the fp32 output)
            return out
        return h

    # -- LiDAR_Renderer.run ----------------------------------------------------
    def render(self, rays_o: torch.Tensor, rays_d: torch.Tensor, time, num_steps: int = 768,
               perturb: bool = False, seed: int = 0, ray_offset: int = 0, lin: Optional[np.ndarray] = None,
               return_stages: bool = False, mask_override: Optional[torch.Tensor] = None):
        """model/renderer.py:44-140 on [N,3] rays.  mask_override [N,S] bool replaces the (non-differentiable)
        `weights > 1e-4` attribute mask: parity tests align it with the implementation under test when a weight sits
        within fp32 rounding of the threshold, where either decision is a correct evaluation of the reference."""
        c = self.cfg
        rays_o = rays_o.reshape(-1, 3).float()
        rays_d = rays_d.reshape(-1, 3).float()
        N = rays_o.shape[0]
        fr = make_frame(float(time), c.num_frames, c.time_resolution)
        near, far = np.float32(c.near_lidar), np.float32(c.far_lidar)
        lin = sample_lin(num_steps) if lin is None else lin
        z1 = (near + (far - near) * lin).astype(np.float32)                     # renderer.py:79
        z = torch.from_numpy(np.broadcast_to(z1, (N, num_steps)).copy()).to(rays_o.device)
        sample_dist = np.float32((far - near) / np.float32(num_steps))          # :82
        if perturb:
            u = jitter_uniform(seed, np.arange(N) + ray_offset, num_steps)
            z = z + (torch.from_numpy(u).to(rays_o.device) - 0.5) * float(sample_dist)           # :84
        xyz = rays_o.unsqueeze(-2) + rays_d.unsqueeze(-2) * z.unsqueeze(-1)     # :88
        xyz = torch.min(torch.max(xyz, self.aabb[:3]), self.aabb[3:])           # :89
        dens = self.density(xyz.reshape(-1, 3), fr, return_features=return_stages)
        sigma = dens["sigma"].view(N, num_steps)
        deltas = z[:, 1:] - z[:, :-1]                                           # :98 (float32 like the reference)
        deltas = torch.cat([deltas, float(sample_dist) * torch.ones_like(deltas[:, :1])], -1).to(self.cd)
        z = z.to(self.cd)
        k = 2.0 if c.active_sensor else 1.0
        alphas = 1 - torch.exp(-k * deltas * c.density_scale * sigma)           # :100-102
        shifted = torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-15], -1)
        weights = alphas * torch.cumprod(shifted, -1)[:, :-1]                   # :104
        mask = weights > 1e-4                                                   # :110
        if mask_override is not None:
            mask = mask_override.to(mask.device).view_as(mask)
        dirs = rays_d.view(-1, 1, 3).expand(N, num_steps, 3).reshape(-1, 3)
        attr = self.attribute(dirs, dens["geo_feat"], mask.reshape(-1)).view(N, num_steps, -1)
        wsum = weights.sum(-1)                                                  # :121
        depth = (weights * z).sum(-1)                                           # :126
        image = (weights.unsqueeze(-1) * attr).sum(-2)                          # :129
        out = {"depth_lidar": depth, "image_lidar": image, "weights_sum_lidar": wsum,
               "weights": weights, "z_vals": z}
        if return_stages:
            out.update(sigma=sigma, geo_feat=dens["geo_feat"], features=dens["features"],
                       flow=dens["flow"], flow_in=dens["flow_in"], mask=mask, attr=attr, xyz=xyz)
        return out


def randomize_parameters(model: OracleLiDAR4D, seed: int = 0, hash_range: float = 0.5,
                         plane_noise: float = 0.1, flow_last_std: float = 0.05) -> None:
    """Parity / throughput initialisation of SURVEY.md §8(d): tcnn's own
    U(-1e-4,1e-4) hash init makes every feature ~0 and hides bugs."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k, v in model.P.items():
            if "hash" in k or "grid_enc" in k:
                v.copy_((torch.rand(v.shape, generator=g) - 0.5) * 2 * hash_range)
            elif "planes" in k:
                v.add_(torch.randn(v.shape, generator=g) * plane_noise)
            elif k.endswith("mlp/4/weight"):
                v.copy_(torch.randn(v.shape, generator=g) * flow_last_std)


MLP_PARAM_NAMES = ("sigma_net/params", "intensity_net/params", "raydrop_net/params",
                   "flow_net/mlp/0/weight", "flow_net/mlp/2/weight", "flow_net/mlp/4/weight")


def snap_mlp_weights_fp16(model: OracleLiDAR4D) -> OracleLiDAR4D:
    """Round every MLP master weight to an fp16-representable value.  With such masters the fp32-weight function
    (the reference's python modules on the shim) and the fp16-working-copy function (tiny-cuda-nn's FullyFusedMLP,
    the tensor-core kernels) are the same function, so one fixture pins both."""
    with torch.no_grad():
        for k in MLP_PARAM_NAMES:
            v = model.P[k]
            v.copy_(v.to(torch.float16).to(v.dtype))
    return model


def band_limit_tables(model: OracleLiDAR4D) -> OracleLiDAR4D:
    """Scale hash level l by resolution_0 / resolution_l ("trained-like" tables: the amplitude of a level falls with its
    cell size, so every level contributes the same slope).  With the white-noise tables of randomize_parameters one ulp
    (6e-8) of a warped coordinate x + flow moves a 32769-cell level by 2e-3 cells = a 1e-3 feature change: two correct
    fp32 implementations then differ by ~5e-5 in the weights and disagree on ReLU / texel decisions of individual
    samples, which shows up as per-entry differences of sparse table gradients (observed on a GPU:
    profiles/r02_parity_*).  Band-limited tables keep that amplification at 1 and gradients comparable entry by entry."""
    with torch.no_grad():
        for k, v in model.P.items():
            if "hash_static" in k:
                geo = model.g_static
            elif "grid_enc" in k:
                geo = model.g_flow
            elif "hash_dynamic" in k:
                geo = model.g_dynamic[int(k.split("/")[2])]
            else:
                continue
            t = v.view(-1, geo.n_features)
            for l in range(geo.n_levels):
                t[int(geo.offset[l]):int(geo.offset[l + 1])] *= float(geo.resolution[0]) / float(geo.resolution[l])
    return model


def projection_vector(n: int) -> np.ndarray:
    """Deterministic float64 direction for gradient fingerprints of tables too big to store (regenerated on the
    GPU box from the formula; the golden-ratio stride keeps it aperiodic)."""
    return np.cos(np.arange(n, dtype=np.float64) * 0.6180339887498949 + 0.25)


def sample_entries(g: np.ndarray, n_top: int = 2048, n_nz: int = 4096, n_zero: int = 1024) -> np.ndarray:
    """Entries of a big gradient to store element-wise: the largest ones, an even stride through the touched
    ones and an even stride through the untouched ones (stray writes show up there)."""
    a = np.abs(g)
    nz = np.flatnonzero(a)
    zz = np.flatnonzero(a == 0)
    pick = [nz[np.argsort(a[nz])[-n_top:]]] if nz.size else []
    if nz.size:
        pick.append(nz[np.linspace(0, nz.size - 1, min(n_nz, nz.size)).astype(np.int64)])
    if zz.size:
        pick.append(zz[np.linspace(0, zz.size - 1, min(n_zero, zz.size)).astype(np.int64)])
    return np.unique(np.concatenate(pick)) if pick else np.zeros(0, np.int64)


def build_seeded(cfg: FieldConfig, seed: int, table_dtype: str = "fp16", **rand_kw) -> OracleLiDAR4D:
    """Deterministic model for a seed: constructor draws from torch's global CPU
    generator seeded here, then randomize_parameters() with its own generator."""
    torch.manual_seed(seed)
    m = OracleLiDAR4D(cfg, table_dtype=table_dtype)
    randomize_parameters(m, seed=seed, **rand_kw)
    return m
