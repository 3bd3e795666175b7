"""CPU: the explicit-point density / attribute backwards (lidar4d_b200/csrc/l4d_points.cuh) against oracle autograd, through
the host build of their per-sample phases (tests/hostsim), and the argument checks of the new C-ABI entry points."""
import ctypes as C

import pytest
import torch

import hostsim_util as H
import points_hostsim_util as PH
from lidar4d_b200 import _capi
from lidar4d_b200.geometry import make_frame
from oracle import lidar4d_oracle as O
from parity_util import small_config, rel_err, relu_margin

TOL = 1e-4
MIN_RELU_MARGIN = 1e-8      # see tests/test_hostsim_parity.py
TIMES = [0.4, 0.0, 1.0]     # interior frame, first frame (no backward neighbour), last frame (no forward neighbour)
_HEAD = ("intensity_net.params", "raydrop_net.params")


def _grad_tables(hs):
    grads = {k: torch.zeros_like(v) for k, v in hs.params.items()}
    tab = _capi.L4DMasterGrads()
    _capi.fill_pointer_table(tab, hs.cfg, lambda n: grads[n].data_ptr())
    work = torch.zeros(hs.L.hs_grad_work_bytes(C.byref(hs.ccfg)), dtype=torch.uint8)
    return grads, tab, work


def hs_density_grads(hs, x, t, g_sigma, g_geo):
    """host-sim l4d_density_forward_ex + l4d_density_backward + l4d_unstage_grads"""
    fr = hs.frame(t)
    x = x.float().contiguous()
    n = x.shape[0]
    sigma, geo = torch.zeros(n), torch.zeros(n, 15)
    feats, flow = torch.zeros(n, hs.cfg.sigma_in_dim), torch.zeros(n, 6)
    saved = torch.zeros(PH.lib().hs_density_saved_bytes(C.byref(hs.ccfg), n), dtype=torch.uint8)
    rc = PH.lib().hs_density_forward_ex(C.byref(hs.ccfg), hs.staged.data_ptr(), C.byref(fr), x.data_ptr(), n, sigma.data_ptr(),
                                         geo.data_ptr(), feats.data_ptr(), flow.data_ptr(), saved.data_ptr())
    assert rc == 0, PH.lib().hs_points_last_error()
    grads, tab, work = _grad_tables(hs)
    gs = None if g_sigma is None else g_sigma.float().contiguous()
    gg = None if g_geo is None else g_geo.float().contiguous()
    rc = PH.lib().hs_density_backward(C.byref(hs.ccfg), hs.staged.data_ptr(), C.byref(fr), x.data_ptr(), n, saved.data_ptr(),
                                       gs.data_ptr() if gs is not None else None, gg.data_ptr() if gg is not None else None,
                                       C.byref(tab), work.data_ptr())
    assert rc == 0, PH.lib().hs_points_last_error()
    assert hs.L.hs_unstage_grads(C.byref(hs.ccfg), work.data_ptr(), C.byref(tab)) == 0
    return dict(sigma=sigma, geo_feat=geo, features=feats, flow=flow), grads


def hs_attribute_grads(hs, d, geo, mask, g_out):
    d, geo, g_out = d.float().contiguous(), geo.float().contiguous(), g_out.float().contiguous()
    n = d.shape[0]
    m8 = None if mask is None else mask.to(torch.uint8).contiguous()
    g_geo = torch.full((n, 15), float("nan"))
    grads, tab, work = _grad_tables(hs)
    rc = PH.lib().hs_attribute_backward(C.byref(hs.ccfg), hs.staged.data_ptr(), d.data_ptr(), geo.data_ptr(),
                                         m8.data_ptr() if m8 is not None else None, n, g_out.data_ptr(), g_geo.data_ptr(),
                                         C.byref(tab), work.data_ptr())
    assert rc == 0, PH.lib().hs_points_last_error()
    assert hs.L.hs_unstage_grads(C.byref(hs.ccfg), work.data_ptr(), C.byref(tab)) == 0
    return g_geo, grads


def attr_margin(orc, d, geo, mask) -> float:
    """smallest |pre-activation| of the four hidden layers of the attribute heads on the masked points"""
    c = orc.cfg
    with torch.no_grad():
        if mask is not None:
            d, geo = d[mask], geo[mask]
        if d.shape[0] == 0:
            return float("inf")
        enc = O.frequency_encode((d.float() + 1) / 2, c.view_degree)
        inp = torch.cat([enc, geo.float(), torch.ones(d.shape[0], c.attr_in_pad - c.attr_in_dim)], -1)
        m = float("inf")
        for net in ("intensity_net.params", "raydrop_net.params"):
            W1, W2, _ = O.mlp_layers(orc.p(net).float(), c.attr_in_pad, 64, 2)
            y1 = inp @ W1.t()
            m = min(m, float(y1.abs().min()), float((torch.relu(y1) @ W2.t()).abs().min()))
    return m


def density_case(seed, fp16):
    orc = O.build_seeded(small_config(), seed, flow_last_std=0.02)
    if fp16:
        orc.mlp_dtype = "fp16"
    return orc


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("t", TIMES)
def test_density_backward_against_oracle(t, fp16):
    orc = density_case(21, fp16)
    hs = H.HostSim(orc, mlp_fp16=fp16)
    g = torch.Generator().manual_seed(4)
    n = 300                                                     # two full tiles of 128 and a ragged one
    x = torch.rand(n, 3, generator=g) * 2 - 1
    g_s, g_g = torch.randn(n, generator=g), torch.randn(n, 15, generator=g)
    ref = orc.density(x, make_frame(t, orc.cfg.num_frames, orc.cfg.time_resolution), return_features=True)
    assert relu_margin(orc, ref) > MIN_RELU_MARGIN, "pick another seed: a ReLU sits on its kink"
    ((ref["sigma"] * g_s).sum() + (ref["geo_feat"] * g_g).sum()).backward()
    og = orc.ref_named_grads()
    out, hg = hs_density_grads(hs, x, t, g_s, g_g)
    for k in ("sigma", "geo_feat", "features", "flow"):
        assert rel_err(out[k], ref[k]) < TOL, k
    errs = {k: rel_err(hg[k], og[k]) for k in hg if og[k].numel()}
    bad = {k: v for k, v in errs.items() if not v < TOL}
    assert not bad, bad
    for k in _HEAD:
        assert float(hg[k].abs().max()) == 0.0, k
    # the flow net is reached through the warped time planes only: nothing at the first / last frame's missing side,
    # something whenever a neighbour exists
    assert float(hg["flow_net.mlp.0.weight"].abs().max()) > 0
    assert float(hg["sigma_net.params"].abs().max()) > 0


def test_density_backward_one_upstream_at_a_time():
    """g_sigma alone and g_geo alone (the other NULL) add up to the joint backward."""
    orc = density_case(21, False)
    hs = H.HostSim(orc)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(150, 3, generator=g) * 2 - 1
    g_s, g_g = torch.randn(150, generator=g), torch.randn(150, 15, generator=g)
    _, both = hs_density_grads(hs, x, 0.4, g_s, g_g)
    _, a = hs_density_grads(hs, x, 0.4, g_s, None)
    _, b = hs_density_grads(hs, x, 0.4, None, g_g)
    for k in both:
        if both[k].numel():
            assert rel_err(a[k] + b[k], both[k]) < 1e-5, k


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("mask_kind", ["none", "partial", "empty"])
def test_attribute_backward_against_oracle(mask_kind, fp16):
    orc = O.build_seeded(small_config(), 14)
    if fp16:
        orc.mlp_dtype = "fp16"
    hs = H.HostSim(orc, mlp_fp16=fp16)
    g = torch.Generator().manual_seed(2)
    n = 301
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    geo = torch.randn(n, 15, generator=g)
    mask = {"none": None, "partial": torch.rand(n, generator=g) > 0.4, "empty": torch.zeros(n, dtype=torch.bool)}[mask_kind]
    g_out = torch.randn(n, 2, generator=g)
    assert attr_margin(orc, d, geo, mask) > MIN_RELU_MARGIN, "pick another seed: a ReLU sits on its kink"
    geo_t = geo.clone().requires_grad_(True)
    ref = orc.attribute(d, geo_t, mask)
    if mask_kind != "empty":
        (ref * g_out.to(ref.dtype)).sum().backward()
    og = orc.ref_named_grads()
    ref_geo = geo_t.grad if geo_t.grad is not None else torch.zeros(n, 15)
    got_geo, hg = hs_attribute_grads(hs, d, geo, mask, g_out)
    if mask_kind == "empty":
        assert float(got_geo.abs().max()) == 0.0
        assert all(float(v.abs().max()) == 0.0 for v in hg.values() if v.numel())
        return
    assert rel_err(got_geo, ref_geo) < TOL
    if mask is not None:
        assert float(got_geo[~mask].abs().max()) == 0.0
    for k in _HEAD:
        assert rel_err(hg[k], og[k]) < TOL, k
    for k, v in hg.items():                                     # nothing else is touched
        if k not in _HEAD and v.numel():
            assert float(v.abs().max()) == 0.0, k


# ---- C-ABI: symbols and argument checks (no GPU needed: every call below returns before touching the device) ------------
def test_point_entry_points_exported_and_checked():
    lib = _capi.load_library()
    for sym in ("l4d_density_saved_bytes", "l4d_density_forward_ex", "l4d_density_backward", "l4d_attribute_backward"):
        assert sym in _capi.EXPORTS and hasattr(lib, sym), sym
    cfg = small_config()
    cc = _capi.make_config(cfg)
    n = 1000
    need = lib.l4d_density_saved_bytes(C.byref(cc), n)
    assert need >= n * (16 + cfg.sigma_in_dim) * 4
    assert lib.l4d_density_saved_bytes(C.byref(cc), 2 * n) > need
    assert lib.l4d_density_saved_bytes(C.byref(cc), 0) == 0
    assert need == PH.lib().hs_density_saved_bytes(C.byref(cc), n)
    bad = _capi.make_config(cfg)
    bad.sigma_in_dim += 1
    assert lib.l4d_density_saved_bytes(C.byref(bad), n) == 0
    wb = lib.l4d_grad_work_bytes(C.byref(cc))
    fake = 256                                                  # never dereferenced: every call fails its checks first
    fr = _capi.make_frame_struct(make_frame(0.4, cfg.num_frames, cfg.time_resolution))
    full = _capi.L4DMasterGrads()
    _capi.fill_pointer_table(full, cfg, lambda name: fake)
    st = None
    EINVAL, ESIZE = -1, -3
    # density forward with a saved buffer
    assert lib.l4d_density_forward_ex(C.byref(cc), None, C.byref(fr), fake, n, fake, fake, None, None, fake, need, st) == EINVAL
    assert lib.l4d_density_forward_ex(C.byref(cc), fake, C.byref(fr), fake, n, None, fake, None, None, fake, need, st) == EINVAL
    assert lib.l4d_density_forward_ex(C.byref(cc), fake, C.byref(fr), fake, n, fake, fake, None, None, fake, need - 1, st) == ESIZE
    # density backward
    args = lambda **o: [C.byref(cc), o.get("staged", fake), C.byref(fr), o.get("x", fake), n, o.get("saved", fake),
                        o.get("saved_bytes", need), fake, fake, C.byref(o.get("grads", full)), o.get("work", fake),
                        o.get("work_bytes", wb), st]
    assert lib.l4d_density_backward(*args(saved=None)) == EINVAL
    assert lib.l4d_density_backward(*args(x=None)) == EINVAL
    assert lib.l4d_density_backward(*args(work=None)) == EINVAL
    assert lib.l4d_density_backward(*args(saved_bytes=need - 1)) == ESIZE
    assert lib.l4d_density_backward(*args(work_bytes=wb - 1)) == ESIZE
    for hole in ("hash_static", "flow_grid", "sigma_net"):
        g = _capi.L4DMasterGrads()
        _capi.fill_pointer_table(g, cfg, lambda name: fake)
        setattr(g, hole, None)
        assert lib.l4d_density_backward(*args(grads=g)) == EINVAL, hole
    g = _capi.L4DMasterGrads()
    _capi.fill_pointer_table(g, cfg, lambda name: fake)
    g.hash_dynamic[1][cfg.time_resolution - 1] = None
    assert lib.l4d_density_backward(*args(grads=g)) == EINVAL
    # attribute backward: only the head buffers are required
    heads = _capi.L4DMasterGrads()
    heads.intensity_net = heads.raydrop_net = fake
    aargs = lambda **o: [C.byref(cc), fake, o.get("d", fake), fake, None, n, o.get("g_out", fake), None,
                         C.byref(o.get("grads", heads)), fake, o.get("work_bytes", wb), st]
    assert lib.l4d_attribute_backward(*aargs(d=None)) == EINVAL
    assert lib.l4d_attribute_backward(*aargs(g_out=None)) == EINVAL
    assert lib.l4d_attribute_backward(*aargs(work_bytes=wb - 1)) == ESIZE
    assert lib.l4d_attribute_backward(*aargs(grads=_capi.L4DMasterGrads())) == EINVAL
    # n == 0 is a no-op once the arguments are valid
    assert lib.l4d_attribute_backward(C.byref(cc), fake, fake, fake, None, 0, fake, None, C.byref(heads), fake, wb, st) == 0
    assert lib.l4d_density_backward(C.byref(cc), fake, C.byref(fr), fake, 0, fake, 0, fake, None, C.byref(full), fake, wb, st) == 0


# ---- the float64 point references (tests/dense_ref.py, tests/points_check.py) ------------------------------------------
def _hs_flow(hs, x, t, g_flow):
    """host-sim l4d_flow_forward (with its saved flow-MLP input) + l4d_flow_backward"""
    fr = hs.frame(t)
    x = x.float().contiguous()
    n = x.shape[0]
    flow, fin = torch.zeros(n, 6), torch.zeros(16, n)
    assert hs.L.hs_flow_forward(C.byref(hs.ccfg), hs.staged.data_ptr(), C.byref(fr), x.data_ptr(), n, flow.data_ptr(),
                                fin.data_ptr()) == 0
    grads, tab, work = _grad_tables(hs)
    g = g_flow.float().contiguous()
    assert hs.L.hs_flow_backward(C.byref(hs.ccfg), hs.staged.data_ptr(), C.byref(fr), x.data_ptr(), n, fin.data_ptr(),
                                 g.data_ptr(), C.byref(tab), work.data_ptr()) == 0
    assert hs.L.hs_unstage_grads(C.byref(hs.ccfg), work.data_ptr(), C.byref(tab)) == 0
    return flow, fin, grads


def _hs_density_saved(hs, x, t, g_sigma, g_geo):
    """hs_density_grads that also returns the saved flow-MLP input and features"""
    import points_check as PC
    fr = hs.frame(t)
    x = x.float().contiguous()
    n = x.shape[0]
    out = dict(sigma=torch.zeros(n), geo_feat=torch.zeros(n, 15), features=torch.zeros(n, hs.cfg.sigma_in_dim),
               flow=torch.zeros(n, 6))
    saved = torch.zeros(PH.lib().hs_density_saved_bytes(C.byref(hs.ccfg), n), dtype=torch.uint8)
    assert PH.lib().hs_density_forward_ex(C.byref(hs.ccfg), hs.staged.data_ptr(), C.byref(fr), x.data_ptr(), n,
                                          out["sigma"].data_ptr(), out["geo_feat"].data_ptr(), out["features"].data_ptr(),
                                          out["flow"].data_ptr(), saved.data_ptr()) == 0
    grads, tab, work = _grad_tables(hs)
    gs = None if g_sigma is None else g_sigma.float().contiguous()
    gg = None if g_geo is None else g_geo.float().contiguous()
    assert PH.lib().hs_density_backward(C.byref(hs.ccfg), hs.staged.data_ptr(), C.byref(fr), x.data_ptr(), n,
                                        saved.data_ptr(), gs.data_ptr() if gs is not None else None,
                                        gg.data_ptr() if gg is not None else None, C.byref(tab), work.data_ptr()) == 0
    assert hs.L.hs_unstage_grads(C.byref(hs.ccfg), work.data_ptr(), C.byref(tab)) == 0
    fin, feat = PC.density_saved_views(hs.cfg, saved, n)
    return out, fin.clone(), feat.clone(), grads


@pytest.mark.parametrize("t", TIMES)
def test_point_references_equal_autograd(t):
    """density_point_reference, flow_reference and attribute_point_reference against torch.autograd.grad through the
    float64 oracle on the same inputs: features, flow-MLP inputs, directions and geo.  The density / flow values agree
    to float64 rounding (the references' inputs are the oracle's own); the attribute nets agree within the reference's
    bound (the oracle rounds the direction encoding's sine to float32, the reference keeps it in float64)."""
    import dense_ref as DR
    cfg = small_config()
    orc = O.build_seeded(cfg, 21, flow_last_std=0.05)
    params32 = {k: v.detach().clone().float() for k, v in orc.ref_state_dict().items()}
    orc.to_float64()
    fr = make_frame(t, cfg.num_frames, cfg.time_resolution)
    g = torch.Generator().manual_seed(3)
    n = 700
    x = torch.rand(n, 3, generator=g) * 2 - 1
    out = orc.density(x, fr, return_features=True)
    gs, gg, gf = (torch.randn(n, generator=g).double(), torch.randn(n, 15, generator=g).double(),
                  torch.randn(n, 6, generator=g).double())
    feats, fin = out["features"], out["flow_in"]
    names = ["sigma_net.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight"]
    loss = (out["sigma"] * gs).sum() + (out["geo_feat"] * gg).sum() + (out["flow"] * gf).sum()
    want = torch.autograd.grad(loss, [orc.p(k) for k in names] + [feats, fin])
    W = DR.working_weights(cfg, params32, False)
    kept = {}
    dref = DR.density_point_reference(cfg, W, feats.detach(), gs, gg, lambda p0, p1, o: kept.update(o))
    fref = DR.flow_reference(W, fin.detach().t(), gf.t(), False, lambda p0, p1, o: kept.update(o), points=True)
    # loss reaches the flow MLP both through flow (gf) and, via the features, through the warped queries; the flow
    # reference takes the first part only, so compare it with autograd of (flow * gf) alone
    want_flow = torch.autograd.grad((orc.density(x, fr, return_features=True)["flow"] * gf).sum(),
                                    [orc.p(k) for k in names[1:]])

    def close(got, ref, bound, what):
        err = (got.double().reshape(-1) - ref.double().reshape(-1)).abs()
        tol = 1e-9 * bound.reshape(-1) + 1e-12 * float(ref.detach().abs().max())
        assert bool((err <= tol).all()), (what, float(err.max()), float(bound.max()))
    close(kept["sigma"][0], out["sigma"], kept["sigma"][1], "sigma")
    close(kept["geo"][0], out["geo_feat"], kept["geo"][1], "geo")
    close(kept["dfeat"][0], want[-2], kept["dfeat"][1], "dfeat")
    close(dref["sigma_net.params"][0], want[0], dref["sigma_net.params"][1], "sigma_net.params")
    close(kept["flow"][0], out["flow"], kept["flow"][1], "flow")
    for k, w in zip(names[1:], want_flow):
        close(fref[k][0], w, fref[k][1], k)
    assert float(dref["sigma_net.params"][0].abs().max()) > 0 and float(fref[names[1]][0].abs().max()) > 0
    # attribute nets on a partial mask
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    d[:6] = torch.tensor([[1.0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0], [0, -1.0, 0], [0, 0, 1.0], [0, 0, -1.0]])
    geo = torch.randn(n, 15, generator=g).double()
    mask = torch.rand(n, generator=g) > 0.3
    go = torch.randn(n, 2, generator=g).double()
    geo_t = geo.clone().requires_grad_(True)
    a = orc.attribute(d, geo_t, mask)
    heads = [orc.p(k) for k in DR.HEADS]
    wa = torch.autograd.grad((a * go).sum(), heads + [geo_t])
    aref = DR.attribute_point_reference(cfg, W, d, geo, mask, go, lambda p0, p1, o: kept.update(o))
    for got, ref, b, what in [(kept["attr"][0].t(), a, kept["attr"][1].t(), "attr"),
                              (kept["dgeo"][0], wa[-1], kept["dgeo"][1], "dgeo")] + \
            [(aref[k][0], w, aref[k][1], k) for k, w in zip(DR.HEADS, wa)]:
        err = (got.reshape(-1) - ref.detach().double().reshape(-1)).abs()
        assert bool((err <= b.reshape(-1) + 1e-12 * float(ref.detach().abs().max())).all()), \
            (what, float((err - b.reshape(-1)).max()))
    assert float(kept["attr"][0][:, ~mask].abs().max()) == 0 and float(kept["dgeo"][0][~mask].abs().max()) == 0


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("t", TIMES)
def test_host_build_within_point_bounds(t, fp16):
    """The host build of the point kernels (float32, contraction off) stays inside every bound of tests/points_check.py:
    flow, density and attribute, forward and backward, on 300 points in and outside the box (|x| up to 1.5 bound)."""
    import points_check as PC
    cfg = small_config(bound=0.75)
    orc = O.build_seeded(cfg, 21, flow_last_std=0.02)
    if fp16:
        orc.mlp_dtype = "fp16"
    hs = H.HostSim(orc, mlp_fp16=fp16)
    params = hs.params
    g = torch.Generator().manual_seed(6)
    n = 300
    x = (torch.rand(n, 3, generator=g) * 3 - 1.5) * cfg.bound
    gf = torch.randn(n, 6, generator=g)
    flow, fin, grads = _hs_flow(hs, x, t, gf)
    st = PC.hold_flow(cfg, params, fp16, t, x, flow, fin, gf, grads, what=f"host flow t={t}")
    gs, gg = torch.randn(n, generator=g), torch.randn(n, 15, generator=g)
    out, fin, feat, grads = _hs_density_saved(hs, x, t, gs, gg)
    sd = PC.hold_density(cfg, params, fp16, t, x, out, fin, feat, gs, gg, grads, what=f"host density t={t}")
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    geo = out["geo_feat"]
    mask = torch.rand(n, generator=g) > 0.4
    go = torch.randn(n, 2, generator=g)
    g_geo, grads = hs_attribute_grads(hs, d, geo, mask, go)
    # the host build has no attribute forward entry point: its forward is held on the GPU only
    sa = PC.hold_attribute(cfg, params, fp16, d, geo, mask, None, go, g_geo, grads, what="host attribute")
    assert st["ambiguous"] + sd["ambiguous"] <= PC.MAX_AMBIGUOUS * 2 * n, (st["ambiguous"], sd["ambiguous"])
    print(f"[points-host] t={t} fp16={fp16}: flow {st['holder'].line()}; density {sd['holder'].line()}; "
          f"attribute {sa['holder'].line()}")
