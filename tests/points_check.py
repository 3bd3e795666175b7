"""Holds the explicit-point kernels - LiDAR4D.flow (k_flow_fwd / k_flow_bwd), LiDAR4D.density (k_density_train /
k_density_bwd) and LiDAR4D.attribute (k_attribute / k_attribute_bwd) - to a float64 evaluation of their own inputs
(test infrastructure, shared by the host-build test on the CPU and tests/test_gpu_points_exact.py).

Each hold_* function takes what a launch consumed and produced - points, frame, upstream gradients, the saved flow-MLP
input and features, the outputs and the parameter gradients - and checks every output entry against tests/gather_ref.py
(features, flow-MLP inputs), tests/dense_ref.py (the point entry points of the MLPs) and tests/scatter_ref.py (the table
gradients).  Values the kernels keep private are taken from the reference with their bound carried on: dL/dfeature
(dense_ref's dfeat) into the scatter, the scattered dL/dflow into the flow MLP, its dL/d(flow-MLP input) into the flow
grid.  Each returns {output: worst fraction of its bound} and the ambiguous-unit counts, and fails when an entry lies
outside its bound or when an entry without a contribution is not exactly 0.  Callers cap the ambiguous points of the
sigma and flow MLPs at MAX_AMBIGUOUS of all the points they hold (a cap per launch would be noise at n = 129)."""
from __future__ import annotations

import torch

import dense_ref as DR
import gather_ref as GR
import scatter_ref as SR
from lidar4d_b200.geometry import make_frame

FLOW_MLP = ("flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight")
HEADS = ("intensity_net.params", "raydrop_net.params")
MAX_AMBIGUOUS = 1e-2          # fraction of points with a sigma- or flow-MLP unit within its bound of the kink


def density_saved_views(cfg, saved: torch.Tensor, n: int):
    """flow_in [16, n] and feat [sigma_in_dim, n] of a density training forward's saved buffer (density_saved_layout)."""
    al = lambda v: (v + 255) // 256 * 256
    o_feat = al(n * 16 * 4)
    f = saved[:o_feat + n * cfg.sigma_in_dim * 4]
    return f[:n * 64].view(torch.float32).view(16, n), f[o_feat:].view(torch.float32).view(cfg.sigma_in_dim, n)


class Holder:
    """Worst |got - ref| / bound per output, and where it was."""

    def __init__(self, what: str):
        self.what, self.worst, self.at = what, {}, {}

    def value(self, name, got, v, b, prefill=None):
        got = got.double().reshape(v.shape)
        if prefill is not None:         # the kernel added into a gradient that held values: one rounding of the sum
            b = b + DR.EPS32 * got.abs()
            got = got - prefill.double().reshape(v.shape)
        r = GR.ratio(got, v, b).reshape(-1)
        i = int(torch.argmax(r))
        if float(r[i]) >= self.worst.get(name, -1.0):
            self.worst[name] = float(r[i])
            self.at[name] = (i, float(got.reshape(-1)[i]), float(v.reshape(-1)[i]), float(b.reshape(-1)[i]))

    def entries(self, name, got, ref, prefill=None):
        """A table gradient against scatter_ref's (ref, A, n[, carried bound]) columns."""
        r = ref.reshape(-1, ref.shape[-1])
        b = (r[:, 2] + SR.SLACK) * SR.EPS32 * r[:, 1]
        if r.shape[1] > 3:
            b = b + r[:, 3]
        b = b + DR.FTZ * r[:, 2] * (r[:, 1] > 0)          # each contribution is one float atomic, which flushes subnormals
        self.value(name, got.reshape(-1), r[:, 0], b, None if prefill is None else prefill.reshape(-1))

    def check(self):
        bad = {k: f"{v:.3g} x bound at {self.at[k]}" for k, v in self.worst.items() if not v <= 1.0}
        assert not bad, f"{self.what}: {bad}"

    def line(self):
        return " ".join(f"{k.replace('.params', '').replace('.weight', '')} {v:.2e}"
                        for k, v in self.worst.items())


def _pf(prefill, k):
    return None if prefill is None else prefill[k]


def _flow_grid(h: Holder, cfg, params, fr, x01, dfin, dfin_e, grads, prefill):
    ref = SR.scatter_reference(cfg, params, fr, x01, None, None, dfin, dfin_e)["flow_net.grid_enc.params"]
    h.entries("flow_grid", grads["flow_net.grid_enc.params"], ref, _pf(prefill, "flow_net.grid_enc.params"))
    # entries of a basis slot whose Lagrange weight is exactly 0 get exactly 0 (their bound is 0 above)
    return sum(int(grads["flow_net.grid_enc.params"].view(-1, 4, 2)[:, i].count_nonzero() == 0)
               for i in range(4) if float(fr.flow_basis[i]) == 0.0)


def hold_flow(cfg, params, fp16: bool, t: float, x, flow, fin, g_flow=None, grads=None, prefill=None, what=""):
    """LiDAR4D.flow on points x [n, 3]: flow [n, 6] and the saved flow-MLP input fin [16, n] the forward wrote; with
    g_flow [n, 6] the backward's gradients (name -> tensor) of flow_net.mlp.* and the flow grid."""
    h = Holder(what)
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    W = DR.working_weights(cfg, params, fp16)
    x01 = SR.point_x01(x, cfg.bound)
    tabs = GR.Tables(cfg, params, fr)

    def on_gather(p0, p1, o):
        fr_, fa = o["flow_in"]
        h.value("flow_in", fin[:, p0:p1].t(), fr_, GR.bound32(fa, GR.FLOW_TERMS))
    GR.gather_reference(tabs, x01, flow.t(), on_gather)
    n = x.shape[0]
    dfin = torch.zeros(16, n, dtype=torch.float64, device=x.device)
    dfin_e = torch.zeros_like(dfin)

    def on_flow(p0, p1, o):
        h.value("flow", flow[p0:p1], *o["flow"])
        dfin[:, p0:p1], dfin_e[:, p0:p1] = o["dfin"][0].t(), o["dfin"][1].t()
    g = g_flow.t() if g_flow is not None else torch.zeros(6, n, device=x.device)
    ref = DR.flow_reference(W, fin, g, False, on_flow, points=True)
    zero_slots = 0
    if g_flow is not None:
        for k in FLOW_MLP:
            h.value(k, grads[k].reshape(-1), ref[k][0].reshape(-1), ref[k][1].reshape(-1), _pf(prefill, k))
        zero_slots = _flow_grid(h, cfg, params, fr, x01, dfin, dfin_e, grads, prefill)
    h.check()
    return dict(holder=h, ambiguous=ref["ambiguous"], zero_slots=zero_slots)


def hold_density(cfg, params, fp16: bool, t: float, x, out: dict, fin, feat, g_sigma=None, g_geo=None, grads=None,
                 prefill=None, what=""):
    """LiDAR4D.density on points x [n, 3]: out = sigma [n], geo_feat [n, 15], features [n, K], flow [n, 6]; fin [16, n]
    and feat [K, n] from the saved buffer; the upstream gradients (None for one the kernel did not get) and the
    backward's gradients of every parameter."""
    h = Holder(what)
    dev = x.device
    n = x.shape[0]
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    W = DR.working_weights(cfg, params, fp16)
    x01 = SR.point_x01(x, cfg.bound)
    nt = GR.feature_terms(cfg, fr).to(dev)

    def on_gather(p0, p1, o):
        r, a = o["features"]
        b = GR.bound32(a, nt)
        h.value("features", out["features"][p0:p1], r, b)
        h.value("saved_feat", feat[:, p0:p1].t(), r, b)
        fr_, fa = o["flow_in"]
        h.value("flow_in", fin[:, p0:p1].t(), fr_, GR.bound32(fa, GR.FLOW_TERMS))
    GR.gather_reference(GR.Tables(cfg, params, fr), x01, out["flow"].t(), on_gather)
    dfeat = torch.zeros(n, cfg.sigma_in_dim, dtype=torch.float64, device=dev)
    dfeat_e = torch.zeros_like(dfeat)

    def on_sigma(p0, p1, o):
        h.value("sigma", out["sigma"][p0:p1], *o["sigma"])
        h.value("geo", out["geo_feat"][p0:p1], *o["geo"])
        dfeat[p0:p1], dfeat_e[p0:p1] = o["dfeat"]
    dref = DR.density_point_reference(cfg, W, feat.t(), g_sigma, g_geo, on_sigma)
    amb = dref["ambiguous"]
    backward = g_sigma is not None or g_geo is not None
    if backward:
        h.value("sigma_net.params", grads["sigma_net.params"], *dref["sigma_net.params"], _pf(prefill, "sigma_net.params"))
        sref = SR.scatter_reference(cfg, params, fr, x01, dfeat, out["flow"].t(), dfeat_err=dfeat_e)
        for k, r in sref.items():
            if k != "dflow":
                h.entries("hash_dynamic" if "hash_dynamic" in k else ("planes" if "planes" in k else k), grads[k], r,
                          _pf(prefill, k))
        d = sref["dflow"]
        dflow, dflow_e = d[..., 0].t(), ((d[..., 2] + SR.SLACK) * SR.EPS32 * d[..., 1] + d[..., 3]).t()
    else:
        dflow = dflow_e = torch.zeros(6, n, dtype=torch.float64, device=dev)
    dfin = torch.zeros(16, n, dtype=torch.float64, device=dev)
    dfin_e = torch.zeros_like(dfin)

    def on_flow(p0, p1, o):
        h.value("flow", out["flow"][p0:p1], *o["flow"])
        dfin[:, p0:p1], dfin_e[:, p0:p1] = o["dfin"][0].t(), o["dfin"][1].t()
    fref = DR.flow_reference(W, fin, dflow, False, on_flow, dflow_err=dflow_e, points=True)
    amb += fref["ambiguous"]
    if backward:
        for k in FLOW_MLP:
            h.value(k, grads[k].reshape(-1), fref[k][0].reshape(-1), fref[k][1].reshape(-1), _pf(prefill, k))
        _flow_grid(h, cfg, params, fr, x01, dfin, dfin_e, grads, prefill)
        for k in HEADS:
            got = grads[k] if prefill is None else grads[k] - prefill[k]
            assert float(got.abs().max()) == 0.0, f"{what}: {k} touched by the density backward"
    h.check()
    return dict(holder=h, ambiguous=amb)


def hold_attribute(cfg, params, fp16: bool, d, geo, mask, out, g_out=None, g_geo=None, grads=None, prefill=None, what=""):
    """LiDAR4D.attribute on n points: out [n, 2] (None: the backward alone); with g_out [n, 2] the backward's dL/dgeo
    [n, 15] and head gradients."""
    h = Holder(what)
    dev = d.device
    n = d.shape[0]
    W = DR.working_weights(cfg, params, fp16)

    def on_chunk(p0, p1, o):
        if out is not None:
            h.value("attr", out[p0:p1].t(), *o["attr"])
        if g_out is not None:
            h.value("dgeo", g_geo[p0:p1], *o["dgeo"])
    dattr = g_out if g_out is not None else torch.zeros(n, 2, device=dev)
    ref = DR.attribute_point_reference(cfg, W, d, geo, mask, dattr, on_chunk)
    if g_out is not None:
        for k in HEADS:
            h.value(k, grads[k], *ref[k], _pf(prefill, k))
    h.check()
    return dict(holder=h, ambiguous=ref["ambiguous_attr"])
