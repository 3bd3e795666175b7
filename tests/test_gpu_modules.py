"""GPU: LiDAR4D's encoder and MLP submodules called on their own (csrc/l4d_modules.cuh): every call of the reference's
module surface against the oracle's restatement of it, forward and backward, in both MLP precisions and both grad modes;
every call against the results of the reference's own modules (tests/golden/modules_ref.npz); the submodule-composed
density against model.density; launch sizes, determinism, argument rules, EMA swaps and the stale-forward error."""
import os

import numpy as np
import pytest
import torch

import modules_golden_util as U
from oracle import lidar4d_oracle as O
from lidar4d_b200 import LiDAR4D
from lidar4d_b200.geometry import lagrange_basis, make_time_query
from parity_util import small_config, rel_err, cuda_model_from_oracle

pytestmark = pytest.mark.gpu
TOL = 1e-4                                   # as tests/test_gpu_point_grads.py
# t on a slice node, between nodes, the ends and the warped-query times (k +- 1) / num_frames of frame k = 20
TIMES = [3 / 7, 0.4, 0.0, 1.0, 21 / 51, 19 / 51]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def case(fp16, seed=31):
    orc = O.build_seeded(small_config(), seed, flow_last_std=0.02)
    if fp16:
        orc.mlp_dtype = "fp16"
    return orc


def points(n, d, seed=5, edges=True):
    """n points in [0,1]^d with the edge cases 0, 1, 1-eps and points outside [0,1] in the first rows"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g)
    if edges and n >= 6:
        e = np.float32(1.0) - np.finfo(np.float32).eps
        x[0], x[1], x[2] = 0.0, 1.0, float(e)
        x[3] = -0.03
        x[4] = 1.04
        x[5, 0] = 1.2
    return x


def model_grads(m, loss_fn, grad_mode, x=None):
    """parameter gradients of loss_fn(m) (and x.grad when x is given) through .grad (arena) or torch.autograd.grad"""
    m.grad_mode = grad_mode
    m.zero_grad(set_to_none=True)
    loss = loss_fn(m)
    names, params = zip(*m.named_parameters())
    if grad_mode == "arena":
        loss.backward()
        return {k: (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)) for k, p in zip(names, params)}
    extra = (x,) if x is not None else ()
    gs = torch.autograd.grad(loss, params + extra, allow_unused=True)
    if x is not None:
        x.grad = gs[-1]
    return {k: (g.detach().clone() if g is not None else torch.zeros_like(p)) for k, p, g in zip(names, params, gs)}


def assert_grads(got, og, keys, tol=TOL):
    errs = {k: rel_err(got[k], og[k]) for k in keys if og[k].numel()}
    bad = {k: v for k, v in errs.items() if not v < tol}
    assert not bad, f"failing: {bad}"


def L(orc):
    return orc.cfg.n_levels_hash


def oracle_hash_t(orc, x2, p, t):
    q = make_time_query(t, orc.cfg.time_resolution)
    x3 = torch.zeros(x2.shape[0], 3)
    a, b = [(0, 1), (0, 2), (1, 2)][p]
    x3[:, a], x3[:, b] = x2[:, 0], x2[:, 1]
    return orc.hash_dynamic(x3, q)[:, p * L(orc):(p + 1) * L(orc)]


def oracle_flow(orc, xt):
    return orc.flow_field(xt[:, :3], lagrange_basis(np.float32(xt[0, 3])))


# (name, module getter, oracle function, input width, parameter keys, gives an input gradient)
def calls(t):
    Lt = lambda o: o.cfg.time_resolution
    return [
        ("hash_static", lambda m: m.hash_encoder.hash_static, lambda o, x: o.hash_static(x), 3,
         ["hash_encoder.hash_static.params"], False),
        ("forward_static", lambda m: m.hash_encoder.forward_static, lambda o, x: o.hash_static(x), 3,
         ["hash_encoder.hash_static.params"], False),
        ("forward_dynamic", lambda m: (lambda x: m.hash_encoder.forward_dynamic(x, torch.tensor(t, device=x.device))),
         lambda o, x: o.hash_dynamic(x, make_time_query(t, Lt(o))), 3,
         [f"hash_encoder.hash_dynamic.{p}.hash_t.{s}.params" for p in range(3) for s in range(8)], False),
        ("hash_t1", lambda m: (lambda x: m.hash_encoder.hash_dynamic[1](x, t)), lambda o, x: oracle_hash_t(o, x, 1, t), 2,
         [f"hash_encoder.hash_dynamic.1.hash_t.{s}.params" for s in range(8)], False),
        ("hash_slice", lambda m: m.hash_encoder.hash_dynamic[2].hash_t[7],
         lambda o, x: O.hash_encode(x, o.p("hash_encoder.hash_dynamic.2.hash_t.7.params"), o.g_dynamic[2]), 2,
         ["hash_encoder.hash_dynamic.2.hash_t.7.params"], False),
        ("planes_static", lambda m: m.planes_encoder.forward_static, lambda o, x: o.planes(x, "static"), 4,
         [f"planes_encoder.planes.{s}.{c}" for s in range(4) for c in (0, 1, 3)], True),
        ("planes_dynamic", lambda m: m.planes_encoder.forward_dynamic, lambda o, x: o.planes(x, "dynamic"), 4,
         [f"planes_encoder.planes.{s}.{c}" for s in range(4) for c in (2, 4, 5)], True),
        ("flow_grid", lambda m: m.flow_net.grid_enc,
         lambda o, x: O.hash_encode(x, o.p("flow_net.grid_enc.params"), o.g_flow), 3, ["flow_net.grid_enc.params"], False),
        ("flow_net", lambda m: m.flow_net, oracle_flow, 4,
         ["flow_net.grid_enc.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight"], False),
    ]


def mlp_calls():
    c = small_config()
    return [
        ("sigma_net", c.sigma_in_dim, 16, "sigma_net.params", 1),
        ("intensity_net", c.attr_in_dim, 1, "intensity_net.params", 2),
        ("raydrop_net", c.attr_in_dim, 1, "raydrop_net.params", 2),
    ]


def prepare_input(name, x, t):
    if name in ("planes_dynamic", "planes_static"):
        x = x.clone()
        x[6:, 3] = torch.linspace(0, 1, x.shape[0] - 6)            # rows with their own times
    if name == "flow_net":
        x = x.clone()
        x[0, 3] = t
        x[1:, 3] = torch.rand(x.shape[0] - 1)                       # only row 0's time counts
    return x


@pytest.mark.parametrize("grad_mode", ["arena", "autograd"])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("t", TIMES)
@pytest.mark.parametrize("idx", range(9))
def test_encoders_against_oracle(dev, idx, t, fp16, grad_mode):
    name, get, ofn, d, keys, xgrad = calls(t)[idx]
    orc = case(fp16)
    m = cuda_model_from_oracle(orc)
    n = 333
    x = prepare_input(name, points(n, d), t)
    ref_x = x.clone().requires_grad_(xgrad)
    ref = ofn(orc, ref_x)
    g = torch.randn(ref.shape, generator=torch.Generator().manual_seed(9))
    (ref * g).sum().backward()
    og = orc.ref_named_grads()
    xd = x.to(dev).requires_grad_(xgrad)

    def loss(mm):
        out = get(mm)(xd)
        assert out.dtype == torch.float32 and out.shape == ref.shape
        assert rel_err(out, ref) < TOL, (name, rel_err(out, ref))
        return (out * g.to(dev)).sum()
    got = model_grads(m, loss, grad_mode, xd if xgrad else None)
    assert_grads(got, og, keys)
    if xgrad:
        assert rel_err(xd.grad, ref_x.grad) < TOL, rel_err(xd.grad, ref_x.grad)


@pytest.mark.parametrize("grad_mode", ["arena", "autograd"])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("idx", range(3))
def test_mlps_against_oracle(dev, idx, fp16, grad_mode):
    name, n_in, n_out, key, layers = mlp_calls()[idx]
    orc = case(fp16)
    m = cuda_model_from_oracle(orc)
    n = 333
    x = torch.randn(n, n_in, generator=torch.Generator().manual_seed(3)) * 0.5
    ref_x = x.clone().requires_grad_(True)
    ref = O.fused_mlp(ref_x, orc.p(key), n_in, n_out, 64, layers, orc.mlp_dtype)
    g = torch.randn(ref.shape, generator=torch.Generator().manual_seed(8))
    (ref * g).sum().backward()
    og = orc.ref_named_grads()
    xd = x.to(dev).requires_grad_(True)

    def loss(mm):
        out = getattr(mm, name)(xd)
        assert out.shape == (n, n_out)
        assert rel_err(out, ref) < TOL
        return (out * g.to(dev)).sum()
    got = model_grads(m, loss, grad_mode, xd)
    assert_grads(got, og, [key])
    assert rel_err(xd.grad, ref_x.grad) < TOL


def test_view_encoder(dev):
    orc = case(False)
    m = cuda_model_from_oracle(orc)
    d = torch.rand(333, 3) * 2 - 1
    v = (d + 1) / 2
    out = m.view_encoder(v.to(dev))
    assert out.shape == (333, 72)
    assert rel_err(out, O.frequency_encode(v, 12)) < 1e-5


def test_static_features_bit_for_bit(dev):
    orc = case(True)
    m = cuda_model_from_oracle(orc)
    c = orc.cfg
    x = (torch.rand(333, 3) * 2 - 1).to(dev)
    t = 0.4
    with torch.no_grad():
        f = m.density(x, torch.tensor([[t]]), return_features=True)["features"]
        x01 = (x + 1.0) / 2.0
        xt = torch.cat([x01, torch.full_like(x01[:, :1], t)], -1)
        ps = m.planes_encoder.forward_static(xt)
        hs = m.hash_encoder.hash_static(x01)
    nS = c.n_levels_plane * 8
    assert torch.equal(ps, f[:, :nS])
    assert torch.equal(hs, f[:, 2 * nS:2 * nS + 4 * c.n_levels_hash])


@pytest.mark.parametrize("n", [0, 1, 333, "wrap"])
def test_sizes_and_determinism(dev, n):
    orc = case(False)
    m = cuda_model_from_oracle(orc)
    if n == "wrap":
        n = wrap_size()
    x = points(n, 3, edges=False)
    with torch.no_grad():
        a = m.hash_encoder.hash_static(x.to(dev))
        b = m.hash_encoder.hash_static(x.to(dev))
        s = m.sigma_net(torch.rand(n, orc.cfg.sigma_in_dim, device=dev))
    assert a.shape == (n, 4 * L(orc)) and s.shape == (n, 16)
    assert torch.equal(a, b)
    if n:
        idx = torch.linspace(0, n - 1, min(n, 4000)).long()
        assert rel_err(a.cpu()[idx], orc.hash_static(x[idx])) < TOL


def test_input_grad_not_implemented(dev):
    m = cuda_model_from_oracle(case(False))
    x = torch.rand(10, 3, device=dev, requires_grad=True)
    xt = torch.rand(10, 4, device=dev, requires_grad=True)
    for f, a in [(m.hash_encoder.hash_static, x), (lambda v: m.hash_encoder.forward_dynamic(v, 0.4), x),
                 (m.view_encoder, x), (m.flow_net, xt), (m.flow_net.grid_enc, x)]:
        with pytest.raises(NotImplementedError):
            f(a)


def test_backward_after_step_raises(dev):
    m = cuda_model_from_oracle(case(False))
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    xt = torch.rand(50, 4, device=dev)
    out = m.planes_encoder.forward_static(xt)
    out.sum().backward()
    opt.step()
    out = m.sigma_net(torch.rand(50, m.cfg.sigma_in_dim, device=dev))
    opt.step()
    m.sigma_net(torch.rand(5, m.cfg.sigma_in_dim, device=dev))        # re-stages the working set
    with pytest.raises(RuntimeError, match="changed between this forward and its backward"):
        out.sum().backward()


def test_no_host_sync(dev):
    m = cuda_model_from_oracle(case(False))
    x = torch.rand(64, 3, device=dev)
    xt = torch.rand(64, 4, device=dev)
    m.hash_encoder(x, 0.4)[1].sum().backward()                       # stage and attach once
    m.flow_net(xt).sum().backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = m.hash_encoder(x, 0.4)
        (a[0].sum() + a[1].sum()).backward()
        m.flow_net(xt).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")


# ---- the end-to-end check: density written with the submodules only ------------------------------------------------
class ComposedLiDAR4D(LiDAR4D):
    """density(x, t) built from the submodules: the frame's neighbours at (k +- 1) / num_frames are reached along the
    flow, their dynamic hash features without gradient, their time planes with gradient into the flow field."""

    def density(self, x, t=None, return_features=False):
        x01 = (x + self.bound) / (2 * self.bound)
        tt = float(np.asarray(t).reshape(-1)[0]) if not torch.is_tensor(t) else float(t.reshape(-1)[0])
        F = self.num_frames
        k = int(np.float32(np.float32(tt) * np.float32(F - 1)))
        col = lambda v: torch.full_like(x01[:, :1], float(np.float32(v)))
        xt = torch.cat([x01, col(tt)], -1)
        h_s, h_d = self.hash_encoder(x01, tt)
        p_s, p_d = self.planes_encoder(xt)
        flow = self.flow_net(xt)
        h_f = h_b = h_d
        p_f = p_b = p_d
        if k < F - 1:
            tf = (k + 1) / F
            xf = x01 + flow[:, :3]
            with torch.no_grad():
                h_f = self.hash_encoder.forward_dynamic(xf, tf)
            p_f = self.planes_encoder.forward_dynamic(torch.cat([xf, col(tf)], -1))
        if k > 0:
            tb = (k - 1) / F
            xb = x01 + flow[:, 3:]
            with torch.no_grad():
                h_b = self.hash_encoder.forward_dynamic(xb, tb)
            p_b = self.planes_encoder.forward_dynamic(torch.cat([xb, col(tb)], -1))
        p_d = 0.5 * p_d + 0.25 * (p_f + p_b)
        h_d = 0.5 * h_d + 0.25 * (h_f + h_b)
        h = self.sigma_net(torch.cat([p_s, p_d, h_s, h_d], -1))
        return {"sigma": O.trunc_exp(h[:, 0]), "geo_feat": h[:, 1:]}


def composed_from_oracle(orc, dev):
    m = cuda_model_from_oracle(orc)
    cm = ComposedLiDAR4D(min_resolution=orc.cfg.min_resolution, base_resolution=orc.cfg.base_resolution,
                         max_resolution=orc.cfg.max_resolution, time_resolution=orc.cfg.time_resolution,
                         n_levels_plane=orc.cfg.n_levels_plane, n_levels_hash=orc.cfg.n_levels_hash,
                         log2_hashmap_size=orc.cfg.log2_hashmap_size, num_frames=orc.cfg.num_frames,
                         hash_size_dynamic=orc.cfg.hash_size_dynamic,
                         flow_base_resolution=orc.cfg.flow_base_resolution,
                         flow_max_resolution=orc.cfg.flow_max_resolution,
                         flow_log2_hashmap_size=orc.cfg.flow_log2_hashmap_size)
    cm.load_state_dict(m.state_dict())
    cm.set_mlp_fp16(orc.mlp_dtype == "fp16")
    return m, cm.to(dev)


@pytest.mark.parametrize("grad_mode", ["arena", "autograd"])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("t", [0.0, 0.4, 1.0])
def test_composed_density(dev, t, fp16, grad_mode):
    orc = case(fp16, seed=21)
    m, cm = composed_from_oracle(orc, dev)
    ro, rd = torch.rand(1, 16, 3, device=dev) * 0.1, torch.nn.functional.normalize(torch.randn(1, 16, 3, device=dev), dim=-1)
    with torch.no_grad():
        before = cm.render(ro, rd, torch.tensor([[t]]), num_steps=64)
    x = (torch.rand(300, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1).to(dev)
    g = torch.randn(300, 15, generator=torch.Generator().manual_seed(3)).to(dev)

    def loss(mm):
        out = mm.density(x, torch.tensor([[t]]))
        return out["sigma"].sum() + (out["geo_feat"] * g).sum()
    ref = m.density(x, torch.tensor([[t]]))
    got = cm.density(x, torch.tensor([[t]]))
    assert rel_err(got["sigma"], ref["sigma"]) < TOL and rel_err(got["geo_feat"], ref["geo_feat"]) < TOL
    g_ref = model_grads(m, loss, grad_mode)
    g_got = model_grads(cm, loss, grad_mode)
    assert_grads(g_got, g_ref, [k for k in g_ref if "raydrop" not in k and "intensity" not in k])
    with torch.no_grad():
        after = cm.render(ro, rd, torch.tensor([[t]]), num_steps=64)    # the model whose submodules ran
    for k in ("depth_lidar", "image_lidar"):
        assert torch.equal(before[k], after[k])


def wrap_size():
    """every CTA of a launch strides at least twice: more than 16 resident CTAs of 128 points per SM"""
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * 16 * 128


@pytest.mark.parametrize("name", ["sigma_net", "flow_net", "planes_dynamic"])
def test_backward_at_wrap_size(dev, name):
    """the backwards with block-wide barriers inside the grid-stride loop (flow field, networks) and the planes backward,
    at a size where every CTA takes several tiles: the forward against the oracle, the gradients against the sum of the
    same kernels' gradients over the two halves of the points (same per-point arithmetic, other tiles and CTAs), and for
    the networks and planes against the oracle too.  (With 5e5 random points some flow-MLP pre-activation lies within
    fp32 noise of its ReLU kink, where two correct evaluations take different sub-gradients: the flow field is held to
    the halves only.)"""
    orc = case(False)
    m = cuda_model_from_oracle(orc)
    n = wrap_size()
    if name == "sigma_net":
        x = torch.randn(n, orc.cfg.sigma_in_dim, generator=torch.Generator().manual_seed(3)) * 0.5
        ofn = lambda xx: O.fused_mlp(xx, orc.p("sigma_net.params"), orc.cfg.sigma_in_dim, 16, 64, 1)
        keys, xgrad = ["sigma_net.params"], True
    elif name == "flow_net":
        x = points(n, 4, edges=False)
        x[:, 3] = 0.4                                                # both halves read the same row-0 time
        ofn = lambda xx: oracle_flow(orc, xx)
        keys, xgrad = ["flow_net.grid_enc.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight",
                       "flow_net.mlp.4.weight"], False
    else:
        x = points(n, 4, edges=False)
        ofn = lambda xx: orc.planes(xx, "dynamic")
        keys, xgrad = [f"planes_encoder.planes.{s}.{c}" for s in range(4) for c in (2, 4, 5)], True
    ref_x = x.clone().requires_grad_(xgrad)
    ref = ofn(ref_x)
    g = torch.randn(ref.shape, generator=torch.Generator().manual_seed(9))
    (ref * g).sum().backward()
    og = orc.ref_named_grads()
    get = {"sigma_net": lambda mm: mm.sigma_net, "flow_net": lambda mm: mm.flow_net,
           "planes_dynamic": lambda mm: mm.planes_encoder.forward_dynamic}[name]

    def run(lo, hi):
        xd = x[lo:hi].to(dev).requires_grad_(xgrad)

        def loss(mm):
            out = get(mm)(xd)
            assert rel_err(out, ref[lo:hi]) < TOL
            return (out * g[lo:hi].to(dev)).sum()
        return model_grads(m, loss, "arena"), xd.grad
    got, gx = run(0, n)
    h1, gx1 = run(0, n // 2)
    h2, gx2 = run(n // 2, n)
    assert_grads(got, {k: h1[k] + h2[k] for k in keys}, keys)
    if name != "flow_net":
        assert_grads(got, og, keys)
    if xgrad:
        assert torch.equal(gx, torch.cat([gx1, gx2]))               # per-point: no accumulation across points
        assert rel_err(gx, ref_x.grad) < TOL


def test_ema_swap_detected(dev):
    """torch_ema's copy_to() / restore() write through .data (no version counter moves): a no-grad submodule call after
    copy_to() sees the EMA weights, a grad-mode call after restore() the trained ones, with the fused Adam's staging"""
    from lidar4d_b200.optim import Adam
    orc, ema = case(False), case(False, seed=32)
    m = cuda_model_from_oracle(orc)
    xt = points(333, 4)
    xd = xt.to(dev)
    m.planes_encoder.forward_static(xd).sum().backward()
    opt = Adam(m, m.get_params(1e-3), betas=(0.9, 0.99), eps=1e-15)
    opt.step()                                                       # re-stages inside the step
    trained = m.planes_encoder.forward_static(xd)                    # grad mode: the content it saw is recorded
    backup = {k: p.detach().clone() for k, p in m.named_parameters()}
    sd = ema.ref_state_dict()
    with torch.no_grad():                                            # ema.copy_to()
        for k, p in m.named_parameters():
            p.data.copy_(sd[k].view_as(p))
        assert rel_err(m.planes_encoder.forward_static(xd), ema.planes(xt, "static")) < TOL
        h = torch.rand(50, orc.cfg.sigma_in_dim)
        assert rel_err(m.sigma_net(h.to(dev)), O.fused_mlp(h, ema.p("sigma_net.params"), orc.cfg.sigma_in_dim, 16, 64, 1)) < TOL
        for k, p in m.named_parameters():                            # ema.restore()
            p.data.copy_(backup[k])
    assert torch.equal(m.planes_encoder.forward_static(xd), trained)


# ---- against the reference modules' own results (tests/golden/modules_ref.npz) ----------------------------------------
@pytest.mark.parametrize("grad_mode", ["arena", "autograd"])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("name", list(U.CONFIGS))
def test_against_reference_golden(dev, name, fp16, grad_mode):
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", U.GOLDEN))
    cfg = U.config(name)
    m = cuda_model_from_oracle(U.oracle(name)).set_mlp_fp16(fp16)
    m.grad_mode = grad_mode
    params = dict(m.named_parameters())
    inp = {k: torch.from_numpy(gold[f"{name}/in/{k}"]).to(dev) for k in U.inputs(cfg)}
    bad = []
    for ci, (key, fn, names, xkey) in enumerate(U.calls(cfg)):
        m.zero_grad(set_to_none=True)
        i = dict(inp)
        if xkey:
            i[xkey] = inp[xkey].clone().requires_grad_(True)
        outs = fn(m, i)
        loss = sum((o * g.to(dev)).sum() for o, g in zip(outs, U.upstream(outs, 100 + ci)))
        for j, o in enumerate(outs):
            e = rel_err(o, torch.from_numpy(gold[f"{name}/{key}/out{j}"]))
            if not e < TOL:
                bad.append((key, f"out{j}", e))
        if not loss.requires_grad:
            continue
        wrt = [params[n] for n in names] + ([i[xkey]] if xkey else [])
        if grad_mode == "arena":
            loss.backward()
            gs = [p.grad if p.grad is not None else torch.zeros_like(p) for p in wrt[:len(names)]]
            gx = i[xkey].grad if xkey else None
        else:
            got = torch.autograd.grad(loss, wrt, allow_unused=True)
            gs = [g if g is not None else torch.zeros_like(p) for g, p in zip(got, wrt)]
            gx = gs[-1] if xkey else None
        for r, n in enumerate(names):
            if not U.fp_close(U.fingerprint(gs[r]), gold[f"{name}/{key}/fp"][r], TOL):
                bad.append((key, n))
        if xkey:
            e = rel_err(gx, torch.from_numpy(gold[f"{name}/{key}/gx"]))
            if not e < TOL:
                bad.append((key, "gx", e))
    assert not bad, bad
