"""CPU: the train-step losses after the flow loss (model/runner.py:255-369).

- The torch restatement (tests/loss_ref.py) reproduces what the UNMODIFIED reference Trainer.train_step computed
  (tests/golden/train_losses.npz, written by tests/golden/make_loss_golden.py), value and gradients, on every option set.
- The kernels' per-patch / per-sample math (l4d_losses.cuh, compiled for the CPU by tests/hostsim/losssim.cu) matches
  the restatement, value and gradient, on the golden's inputs and on synthetic patch batches of several shapes."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

import __graft_entry__
import loss_ref
from lidar4d_b200.losses import GRAD_CRITERIA

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "train_losses.npz"), allow_pickle=False)
NAMES = [str(s) for s in GOLD["names"]]
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(__graft_entry__.build_losssim())
        P, F, U = C.c_void_p, C.c_float, C.c_uint32
        L.ls_patch.argtypes = [P, P, U, U, U, F, U, U, F, F, F, F, P, P]
        L.ls_los.argtypes = [P, P, P, U, U, C.c_double, F, P, P]
        L.ls_patch.restype = L.ls_los.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data


def sim_patch(depth, gt, patch_size, **kw):
    o = dict(loss_ref.DEFAULTS)
    o.update({k: v for k, v in kw.items() if k in o})
    px, py = (patch_size, patch_size) if isinstance(patch_size, int) else (tuple(patch_size) * 2)[:2] if len(patch_size) == 1 \
        else tuple(patch_size)
    d = np.ascontiguousarray(depth, np.float32).reshape(-1)
    g = np.ascontiguousarray(gt, np.float32).reshape(-1, 3)
    flags = (1 if o["sobel_grad"] else 0) | (2 if o["grad_loss"] else 0) | (4 if o["grad_norm_smooth"] else 0) | \
        (8 if o["spatial_smooth"] else 0) | (16 if o["tv_loss"] else 0)
    loss = np.zeros(1, np.float32)
    gd = np.zeros_like(d)
    lib().ls_patch(_p(d), _p(g), d.size, px, py, o["scale"], GRAD_CRITERIA[o["depth_grad_loss"]], flags, o["alpha_grad"],
                   o["alpha_grad_norm"], o["alpha_spatial"], o["alpha_tv"], _p(loss), _p(gd))
    return float(loss[0]), gd


def sim_los(w, z, gt, eps, g_in=1.0):
    w, z = np.ascontiguousarray(w, np.float32), np.ascontiguousarray(z, np.float32)
    g = np.ascontiguousarray(gt, np.float32).reshape(-1, 3)
    loss = np.zeros(1, np.float32)
    gw = np.zeros_like(w)
    lib().ls_los(_p(w), _p(z), _p(g), w.shape[0], w.shape[1], eps, g_in, _p(loss), _p(gw))
    return float(loss[0]), gw


def ref_patch(depth, gt, patch_size, **kw):
    """The restatement on inputs divided by scale beforehand, with scale 1: torch on the CPU divides by scale exactly,
    the kernels (and torch on CUDA) multiply by its fp32 reciprocal, and one ulp of depth / scale ~ 65 is 1e-4 of the
    differences the branch takes.  With m in {0, 1}, (x * m) * (1/scale) == (x * (1/scale)) * m, so both sides then see
    the same pred and gt_d bits; the gradient is scaled back by 1/scale."""
    scale = kw.get("scale", loss_ref.DEFAULTS["scale"])
    inv = np.float32(1) / np.float32(scale)
    g = np.array(gt, np.float32).reshape(-1, 3)
    g[:, 2] *= inv
    d = torch.tensor(np.asarray(depth, np.float32).reshape(-1) * inv, requires_grad=True)
    kw = dict(kw, scale=1.0)
    loss = loss_ref.patch_ref(d, torch.from_numpy(g), patch_size, huber_delta=0.2 * scale, **kw)
    if loss.requires_grad:
        loss.backward()
    return float(loss), (d.grad.numpy() * inv if d.grad is not None else np.zeros(d.shape, np.float32))


def ref_los(w, z, gt, eps):
    wt = torch.tensor(np.asarray(w, np.float32), requires_grad=True)
    loss = loss_ref.line_of_sight_ref(wt, torch.from_numpy(np.asarray(z, np.float32)), torch.from_numpy(np.asarray(gt)), eps)
    loss.backward()
    return float(loss), wt.grad.numpy()


def cos_term_scale(depth, gt, patch, scale=0.01, sobel_grad=False, alpha_grad=0.1, **_):
    """The largest single term of the cosine criterion's gradient, alpha_grad * |stencil| / scale / max(|a_p|, eps) over
    patches p (a_p = the masked predicted x differences).  Where a_p has one nonzero entry, a_p and b_p are parallel,
    the gradient is 0 in exact arithmetic and any two roundings of it differ by a few ulps of such terms."""
    import torch.nn.functional as F
    px, py = (patch, patch) if isinstance(patch, int) else (list(patch) * 2)[:2] if len(patch) == 1 else patch
    g = torch.from_numpy(np.asarray(gt, np.float32).reshape(-1, 3))
    P = (torch.from_numpy(np.asarray(depth, np.float32)) * g[:, 0] / scale).view(-1, 1, px, py)
    G = (g[:, 2] * g[:, 0] / scale).view(-1, 1, px, py)
    if sobel_grad:
        k = torch.tensor([[-1, 0, 1], [-2, 0, 2], [-1, 0, 1]], dtype=torch.float32)[None, None]
        a, b, m = F.conv2d(P, k, padding=1), F.conv2d(G, k, padding=1), g[:, 0].view(-1, 1, px, py)
    else:
        a, b, m = (P[..., :-1] - P[..., 1:]).abs(), G[..., :-1] - G[..., 1:], g[:, 0].view(-1, 1, px, py)[..., :-1]
    a = (a * m * (b.abs() < 0.01)).flatten(1)
    na = a.norm(dim=1).clamp_min(1e-8)
    return float(alpha_grad * 8 / scale / na.min()) if a.shape[0] else 0.0


def close(a, b, rel=1e-5):
    return a == pytest.approx(b, rel=rel, abs=1e-7)


def grad_close(a, b, tol=1e-6):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() <= tol * max(np.abs(b).max(), 1e-30)


def golden_opt(name):
    kw = dict(patch_size_lidar=[2, 8], urf_loss=False, iters=int(GOLD["iters"]), **loss_ref.DEFAULTS)
    kw.update(loss_ref.OPTION_SETS[name])
    return types.SimpleNamespace(**kw)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_reference_trainer(name):
    """runner.py:255-369 restated == the reference's train_step on the same render outputs (value and gradients)."""
    d = torch.tensor(GOLD["depth_lidar"], requires_grad=True)
    w = torch.tensor(GOLD["weights"], requires_grad=True)
    z = torch.from_numpy(GOLD["z_vals"])
    gt = torch.from_numpy(GOLD["images"])
    opt = golden_opt(name)
    loss = loss_ref.extra_losses_ref({"depth_lidar": d, "weights": w, "z_vals": z}, gt, opt, int(GOLD["global_step"]))
    loss.backward()
    assert loss.item() == pytest.approx(float(GOLD[f"{name}/loss"]), rel=1e-6)
    g_d = d.grad.numpy()
    # the stored weights gradient includes the path through depth_lidar = sum(weights * z_vals)
    g_w = (w.grad if w.grad is not None else torch.zeros_like(w)) + z * d.grad.view(-1, 1)
    assert grad_close(g_d, GOLD[f"{name}/g_depth"])
    assert grad_close(g_w.numpy(), GOLD[f"{name}/g_weights"])


@pytest.mark.parametrize("name", NAMES)
def test_kernel_math_matches_restatement_on_golden_inputs(name):
    opt = golden_opt(name)
    d, gt = GOLD["depth_lidar"].reshape(-1), GOLD["images"].reshape(-1, 3)
    v_sim, g_sim = sim_patch(d, gt, opt.patch_size_lidar, **vars(opt))
    v_ref, g_ref = ref_patch(d, gt, opt.patch_size_lidar, **vars(opt))
    assert close(v_sim, v_ref)
    assert grad_close(g_sim, g_ref)
    if opt.urf_loss:
        eps = loss_ref.los_eps(int(GOLD["global_step"]), opt.iters)
        v_sim, g_sim = sim_los(GOLD["weights"], GOLD["z_vals"], gt, eps)
        v_ref, g_ref = ref_los(GOLD["weights"], GOLD["z_vals"], gt, eps)
        assert close(v_sim, v_ref)
        assert grad_close(g_sim, g_ref)


PATCH_CASES = [([2, 8], 24), (4, 10), ([3, 5], 13), ([1, 8], 6), ([8], 3), ([2, 1], 9)]
OPTION_CASES = [dict(depth_grad_loss=c, sobel_grad=s) for c in GRAD_CRITERIA for s in (False, True)] + \
    [dict(grad_norm_smooth=True, spatial_smooth=True, tv_loss=True, sobel_grad=s) for s in (False, True)] + \
    [dict(grad_loss=False, tv_loss=True), dict(spatial_smooth=True, alpha_spatial=0.37, alpha_grad=0.2)]


@pytest.mark.parametrize("patch,n_patch", PATCH_CASES)
@pytest.mark.parametrize("opts", OPTION_CASES, ids=lambda o: "-".join(f"{k}={v}" for k, v in o.items()))
def test_patch_math_matches_restatement(patch, n_patch, opts):
    px, py = (patch, patch) if isinstance(patch, int) else (patch * 2)[:2] if len(patch) == 1 else patch
    gt = loss_ref.patch_gt(n_patch, px, py, seed=n_patch).numpy()
    rng = np.random.default_rng(7)
    # predictions near the gt so the criteria see small and large differences, with exact ties to the gt here and there
    depth = loss_ref.quantize(gt[:, 2] + rng.normal(0, 3e-5, gt.shape[0]) * (rng.random(gt.shape[0]) > 0.2))
    v_sim, g_sim = sim_patch(depth, gt, patch, **opts)
    v_ref, g_ref = ref_patch(depth, gt, patch, **opts)
    if np.isnan(v_ref):                     # the mean over an empty dx / dy (py == 1 or px == 1 without Sobel) is nan
        assert np.isnan(v_sim)
        return
    assert close(v_sim, v_ref)
    if opts.get("depth_grad_loss") == "cos":
        assert np.abs(g_sim - g_ref).max() <= 1e-6 * max(np.abs(g_ref).max(), cos_term_scale(depth, gt, patch, **opts))
    else:
        assert grad_close(g_sim, g_ref)


def test_all_masked_patch_gives_one_and_no_gradient():
    gt = loss_ref.patch_gt(4, 2, 8, seed=3).numpy()
    gt[:16, 0] = 0.0                               # the first patch's rays all dropped
    depth = np.random.default_rng(0).random(gt.shape[0]).astype(np.float32)
    v_sim, g_sim = sim_patch(depth, gt, [2, 8], depth_grad_loss="cos")
    v_ref, g_ref = ref_patch(depth, gt, [2, 8], depth_grad_loss="cos")
    assert close(v_sim, v_ref) and np.all(g_sim[:16] == 0) and grad_close(g_sim, g_ref)


def los_case(n, S, seed, inside=False, no_valid=False):
    g = np.random.default_rng(seed)
    gt = np.stack([(g.random(n) > 0.2), g.random(n), 0.05 + 0.6 * g.random(n)], -1).astype(np.float32)
    if no_valid:
        gt[:, 0] = 0.0
    gd = gt[:, 2] * gt[:, 0]
    if inside:                                     # every sample within eps of its ray's gt depth
        z = gd[:, None] + g.uniform(-0.015, 0.015, (n, S))
    else:
        z = np.sort(g.uniform(0.01, 0.85, (n, S)), axis=1)
        z[:, :4] = gd[:, None] + g.uniform(-0.015, 0.015, (n, 4))
    w = g.random((n, S)) ** 4
    return w.astype(np.float32), z.astype(np.float32), gt


@pytest.mark.parametrize("n,S,kind", [(16, 48, "normal"), (64, 768, "normal"), (16, 48, "inside"), (32, 7, "inside")])
def test_line_of_sight_math_matches_restatement(n, S, kind):
    w, z, gt = los_case(n, S, seed=n + S, inside=kind == "inside")
    eps = 0.02
    v_sim, g_sim = sim_los(w, z, gt, eps)
    v_ref, g_ref = ref_los(w, z, gt, eps)
    assert close(v_sim, v_ref)
    assert grad_close(g_sim, g_ref)
    # the scaled backward is the same gradient times the scale
    _, g_big = sim_los(w, z, gt, eps, g_in=65536.0)
    assert grad_close(g_big, g_ref * 65536.0)


def test_line_of_sight_without_valid_rays_is_the_references_inf_or_nan():
    w, z, gt = los_case(16, 48, seed=1, no_valid=True)
    v_sim, _ = sim_los(w, z, gt, 0.02)
    v_ref, _ = ref_los(w, z, gt, 0.02)
    assert not np.isfinite(v_ref) and (np.isnan(v_sim) == np.isnan(v_ref)) and (np.isinf(v_sim) == np.isinf(v_ref))
