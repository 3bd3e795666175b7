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
