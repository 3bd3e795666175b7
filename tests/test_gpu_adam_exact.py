"""GPU: the fused Adam step is torch's fused Adam (torch 2.11, ``torch._fused_adam_`` / ``torch.optim.Adam(fused=True)``)
bit for bit - parameters, exp_avg and exp_avg_sq compared as int32 after every step - and the fp16 hash tables it writes
in the same pass are byte for byte a from-scratch staging of the updated masters.

  a. synthetic arenas straight through l4d_adam_step, in every value regime of tests/test_adam_hostsim.py and the arena
     layouts where a grid-stride chunk kernel goes wrong (partial quads, gaps, 64 segments, the grid cap), with a
     power-of-two inv_scale against torch's grad_scale and zero_grad=1;
  b. lidar4d_b200.optim.Adam against torch.optim.Adam(fused=True) on clones of a model's parameters, with seeded
     gradients written into the .grad views (no render, so no atomics noise), the recipe's LambdaLR, per-group rates
     that diverge mid-run, moments driven subnormal by zero gradients, and a state_dict round trip mid-run;
  c. after each of b's steps, the staged buffer against l4d_stage_params_ex(TABLES | SMALL) into a zero-filled buffer
     and every table region against torch's .half() of the masters."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

from lidar4d_b200 import _capi, LiDAR4D
from lidar4d_b200.geometry import FieldConfig
from parity_util import SMALL, FULL
from test_adam_hostsim import B1, B2, EPS, STEPS, regime

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bits(t):
    return t.contiguous().view(torch.int32)


def _ndiff(a, b):
    return int((_bits(a) != _bits(b)).sum())


# ---- a. synthetic arenas --------------------------------------------------------------------------------------------
def _arena(n, seed, regimes=("magnitudes", "g_zero", "g_tiny", "update_subnormal", "v_large", "g_huge", "nonfinite")):
    """p, m, v, g of n floats: runs of 1024 floats drawn from the value regimes in turn"""
    rng = np.random.default_rng(seed)
    out = [np.empty(n, np.float32) for _ in range(4)]
    pos, k = 0, 0
    while pos < n:
        run = min(n - pos, 1024 * int(rng.integers(1, 5)))
        p, m, v, g, _ = regime(regimes[k % len(regimes)], rng, run)
        for o, x in zip(out, (p, m, v, g)):
            o[pos:pos + run] = x
        pos, k = pos + run, k + 1
    return [torch.from_numpy(x).to(DEV) for x in out]


def _adam_step(arena, segs, step, inv_scale=1.0, zero_grad=0):
    lib = _capi.load_library()
    cfg = _capi.make_config(FieldConfig())
    p, m, v, g = arena
    arr = (_capi.L4DAdamGroup * len(segs))()
    for i, (b, e, lr) in enumerate(segs):
        arr[i].begin, arr[i].end, arr[i].lr = b, e, lr
    rc = lib.l4d_adam_step(C.byref(cfg), p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), arr,
                           len(segs), float(B1), float(B2), float(EPS), step, inv_scale, zero_grad, None, None, 0,
                           torch.cuda.current_stream().cuda_stream)
    _capi.check(lib, rc, "l4d_adam_step")


def _torch_step(arena, segs, step, grad_scale=None):
    p, m, v, g = arena
    for lr in sorted({s[2] for s in segs}):
        mine = [(b, e) for b, e, l in segs if l == lr]
        torch._fused_adam_([p[b:e] for b, e in mine], [g[b:e] for b, e in mine], [m[b:e] for b, e in mine],
                           [v[b:e] for b, e in mine], [], [torch.tensor(float(step), device=DEV) for _ in mine],
                           lr=lr, beta1=float(B1), beta2=float(B2), weight_decay=0.0, eps=float(EPS), amsgrad=False,
                           maximize=False, grad_scale=grad_scale, found_inf=None)


def _layouts():
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    cap = sm * 16                                   # k_adam_flat's grid cap, in chunks
    rng = np.random.default_rng(3)
    out = {"single_chunk": (1024, [(0, 1024, 1e-2)]),
           "ends_at_4_mod_1024": (8 * 1024, [(0, 1028, 1e-2), (2048, 3076, 1e-3), (4096, 8 * 1024 - 1020, 1e-2)]),
           "gaps": (16 * 1024, [(2048, 3000, 1e-2), (5120, 9216, 1e-3), (12288, 12292, 3e-4)])}
    b, segs = 0, []
    for i in range(64):
        e = b + 4 * int(rng.integers(1, 1024 * 3 // 4))
        segs.append((b, e, (1e-2, 1e-3)[i % 2] if i % 5 else 2e-3))
        b = (e + 1023) // 1024 * 1024 + 1024 * int(rng.integers(0, 2))
    out["64_segments"] = (b, segs)
    for nc in (cap - 1, cap, cap + 1, 2 * cap + 3):
        out[f"chunks_{nc}"] = (nc * 1024, [(0, 1024 * (nc // 2), 1e-2), (1024 * (nc // 2), nc * 1024 - 8, 1e-3)])
    return out


@pytest.mark.parametrize("layout", ["single_chunk", "ends_at_4_mod_1024", "gaps", "64_segments", "cap-1", "cap", "cap+1",
                                    "2cap+3"])
def test_adam_step_equals_torch_fused_adam_on_synthetic_arenas(layout):
    lays = _layouts()
    cap = torch.cuda.get_device_properties(0).multi_processor_count * 16
    key = {"cap-1": cap - 1, "cap": cap, "cap+1": cap + 1, "2cap+3": 2 * cap + 3}.get(layout)
    n, segs = lays[f"chunks_{key}"] if key is not None else lays[layout]
    covered = torch.zeros(n, dtype=torch.bool, device=DEV)
    for b, e, _ in segs:
        covered[b:e] = True
    for si, step in enumerate(STEPS):
        ours = _arena(n, 1000 + si)
        ref = [x.clone() for x in ours]
        before = [x.clone() for x in ours]
        _adam_step(ours, segs, step)
        _torch_step(ref, segs, step)
        for what, a, r, b0 in zip("pmvg", ours, ref, before):
            assert _ndiff(a, r) == 0, (layout, step, what, _ndiff(a, r))
            assert torch.equal(_bits(a)[~covered], _bits(b0)[~covered]), (layout, step, what, "outside the groups")
    torch.cuda.synchronize()


@pytest.mark.parametrize("k", [-16, -7, -1, 0, 1, 5, 16])
def test_inv_scale_equals_torch_grad_scale(k):
    n, segs = _layouts()["ends_at_4_mod_1024"]
    for step in (1, 3, 100):
        ours = _arena(n, 50 + k + 17 * step, regimes=("magnitudes", "g_tiny", "update_subnormal", "v_large"))
        ours[3] *= 2.0 ** -k                          # the scaled gradient; exact: powers of two
        ref = [x.clone() for x in ours]
        _adam_step(ours, segs, step, inv_scale=2.0 ** k)
        _torch_step(ref, segs, step, grad_scale=torch.tensor(2.0 ** -k, device=DEV))
        for what, a, r in zip("pmv", ours[:3], ref[:3]):
            assert _ndiff(a, r) == 0, (k, step, what)


def test_zero_grad_clears_exactly_the_covered_ranges():
    n, segs = _layouts()["gaps"]
    ours = _arena(n, 77)
    g0 = ours[3].clone()
    ref = [x.clone() for x in ours]
    _adam_step(ours, segs, 2, zero_grad=1)
    _torch_step(ref, segs, 2)
    covered = torch.zeros(n, dtype=torch.bool, device=DEV)
    for b, e, _ in segs:
        covered[b:e] = True
    assert int((_bits(ours[3])[covered] != 0).sum()) == 0                  # +0.0 everywhere it covered
    assert torch.equal(_bits(ours[3])[~covered], _bits(g0)[~covered])
    for what, a, r in zip("pmv", ours[:3], ref[:3]):
        assert _ndiff(a, r) == 0, what


# ---- b./c. the optimiser class against torch.optim.Adam(fused=True) ------------------------------------------------
def _model(kind):
    torch.manual_seed(0)
    if kind == "small":
        m = LiDAR4D(**SMALL)
    elif kind == "t2":
        m = LiDAR4D(**dict(SMALL, time_resolution=2))
    else:
        m = LiDAR4D(n_levels_hash=16, **FULL)            # the benchmarked configuration: L = 16, 2^19 tables
    return m.to(DEV)


def _torch_twin(model, lr, lambdas):
    named = dict(model.named_parameters())
    by_id = {id(p): n for n, p in named.items()}
    clones = {n: p.detach().clone().requires_grad_() for n, p in named.items() if n in model._engine.names}
    groups = [{"params": [clones[by_id[id(p)]] for p in g["params"] if p.numel() and by_id[id(p)] in clones],
               "lr": g["lr"]} for g in model.get_params(lr)]
    opt = torch.optim.Adam(groups, betas=(0.9, 0.99), eps=1e-15, fused=True)
    return clones, opt, torch.optim.lr_scheduler.LambdaLR(opt, lambdas)


def _ours(model, lr, lambdas):
    from lidar4d_b200.optim import Adam
    opt = Adam(model, model.get_params(lr), betas=(0.9, 0.99), eps=1e-15)
    return opt, torch.optim.lr_scheduler.LambdaLR(opt, lambdas)


def _table_regions(model):
    """(name, staged byte range, expected fp16 bytes) of every hash table: static / flow plain casts, dynamic slice-pair
    records k = {slice k | slice k+1}, 4 halves each (include/lidar4d_b200.h, l4d_stage_params_ex)"""
    eng, T = model._engine, model.cfg.time_resolution
    ts = eng.tensors()
    up = lambda x: (x + 255) // 256 * 256
    out, o = [], 0
    hs = ts["hash_encoder.hash_static.params"].detach()
    out.append(("hash_static", o, hs.half()))
    o = up(o + hs.numel() * 2)
    for p in range(3):
        sl = [ts[f"hash_encoder.hash_dynamic.{p}.hash_t.{t}.params"].detach().half().view(-1, 4) for t in range(T)]
        pairs = torch.stack([torch.stack([sl[k], sl[k + 1]], 1) for k in range(T - 1)])      # [T-1][ne][2][4]
        out.append((f"hash_dynamic.{p}", o, pairs))
        o = up(o + pairs.numel() * 2)
    hf = ts["flow_net.grid_enc.params"].detach()
    out.append(("flow_grid", o, hf.half()))
    return out


def _check_staged(model):
    eng = model._engine
    lib = eng._lib()
    fresh = torch.zeros_like(eng.staged)
    rc = lib.l4d_stage_params_ex(C.byref(eng.ccfg), C.byref(eng.master_table()), fresh.data_ptr(), fresh.numel(),
                                 _capi.STAGE_TABLES | _capi.STAGE_SMALL, eng.stream())
    _capi.check(lib, rc, "l4d_stage_params_ex")
    assert torch.equal(eng.staged, fresh), "fused table refresh != from-scratch staging"
    for name, off, exp in _table_regions(model):
        got = eng.staged[off:off + exp.numel() * 2]
        assert torch.equal(got, exp.reshape(-1).view(torch.uint8)), name


def _compare(model, clones, opt, topt, step):
    eng = model._engine
    bad = []
    ts = eng.tensors()
    for n, q in clones.items():
        o, k = eng.offsets[n]
        if k == 0:
            continue
        st = topt.state[q]
        for what, a, b in (("param", ts[n].detach().reshape(-1), q.detach().reshape(-1)),
                           ("exp_avg", opt._exp_avg[o:o + k], st["exp_avg"].reshape(-1)),
                           ("exp_avg_sq", opt._exp_avg_sq[o:o + k], st["exp_avg_sq"].reshape(-1))):
            d = _ndiff(a, b)
            if d:
                bad.append((n, what, d))
    assert not bad, (step, bad[:8])


def _grads(model, clones, gen, step, quiet):
    """seeded gradients, identical on both sides; tensors in `quiet` get tiny gradients at step 1 and zeros after"""
    ts = model._engine.tensors()
    for n, q in clones.items():
        k = q.numel()
        if k == 0:
            continue
        if n in quiet:
            g = (torch.rand(k, device=DEV, generator=gen) * 1e-20 if step == 1 else torch.zeros(k, device=DEV))
            if step == 1:
                g[::2] *= 1e-10
        else:
            g = torch.randn(k, device=DEV, generator=gen) * 10.0 ** float(torch.empty(()).uniform_(-6, 1, generator=None))
        ts[n].grad.view(-1).copy_(g)
        q.grad = g.view(q.shape).clone()


def _run(kind, n_steps, per_group=False, resume_at=None, quiet=()):
    torch.manual_seed(1)
    model = _model(kind)
    eng = model._engine
    iters = max(n_steps, 20)
    base = lambda it: 0.1 ** min(it / iters, 1)                                 # main_lidar4d.py:302-305
    if per_group:                      # equal rates (groups 0-2, groups 3-6) split apart after step 8
        lambdas = [lambda it, i=i: base(it) * (1.0 if it < 8 else 0.5 ** (i % 3)) for i in range(7)]
    else:
        lambdas = base
    clones, topt, tsched = _torch_twin(model, 1e-2, lambdas)
    opt, sched = _ours(model, 1e-2, lambdas)
    eng.attach_grads()
    eng.ensure_staged()                                   # staged working set present: the step refreshes the tables
    gen = torch.Generator(device=DEV).manual_seed(7)
    for step in range(1, n_steps + 1):
        _grads(model, clones, gen, step, quiet)
        opt.step()
        topt.step()
        sched.step()
        tsched.step()
        _compare(model, clones, opt, topt, step)
        if step <= 3 or step % 25 == 0 or step == n_steps:
            _check_staged(model)
        if step == resume_at:
            buf = io.BytesIO()
            torch.save({"opt": opt.state_dict(), "sched": sched.state_dict()}, buf)
            buf.seek(0)
            sd = torch.load(buf, weights_only=False)
            opt, sched = _ours(model, 1e-2, lambdas)
            opt.load_state_dict(sd["opt"])
            sched.load_state_dict(sd["sched"])
            assert [g["lr"] for g in opt.param_groups] == [g["lr"] for g in topt.param_groups]
    torch.cuda.synchronize()
    return model, opt


def test_optim_adam_equals_torch_fused_adam_small_config():
    _run("small", 24, resume_at=11)


def test_optim_adam_per_group_rates_diverging_mid_run():
    _run("small", 20, per_group=True)


def test_optim_adam_subnormal_moments_after_hundreds_of_zero_gradient_steps():
    quiet = ("hash_encoder.hash_static.params", "hash_encoder.hash_dynamic.1.hash_t.3.params", "sigma_net.params")
    model, opt = _run("small", 400, quiet=quiet)
    o, k = model._engine.offsets[quiet[0]]
    for mom in (opt._exp_avg[o:o + k].abs(), opt._exp_avg_sq[o:o + k]):
        assert bool(((mom > 0) & (mom < 2.0 ** -126)).any())


def test_optim_adam_single_slice_pair():
    _run("t2", 20)


def test_optim_adam_equals_torch_fused_adam_benchmark_config():
    _run("full", 20, resume_at=9)
