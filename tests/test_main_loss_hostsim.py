"""CPU: the main LiDAR loss of train_step (model/runner.py:193-220, with the chamfer term) and eval_step's loss (:409-421).

- The torch restatement (tests/main_loss_ref.py) reproduces what the UNMODIFIED reference Trainer computed
  (tests/golden/main_loss_ref.npz, written by tests/golden/make_main_loss_golden.py), loss and gradients, on every case.
- The kernels' per-element, cosine and fold math (l4d_losses.cuh, compiled for the CPU by tests/hostsim/mainlosssim.cu)
  matches the restatement on the same cases, with the chamfer oracle supplying the distances and their gradient."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import __graft_entry__
import main_loss_ref as R
from lidar4d_b200.losses import GRAD_CRITERIA
from oracle import chamfer_oracle

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "main_loss_ref.npz"), allow_pickle=False)
CASES = {c[0]: c for c in R.case_list()}
TRAIN = [k for k in CASES if CASES[k][1] == "train"]
EVAL = [k for k in CASES if CASES[k][1] == "eval"]
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(__graft_entry__.build_mainlosssim())
        P, F, U, D = C.c_void_p, C.c_float, C.c_uint32, C.c_double
        L.ms_train.argtypes = [P, P, P, P, U, P, P, D, F, F, P, P, P, P, P]
        L.ms_train.restype = None
        L.ms_finish.argtypes = [P, P, U, F, D, P, P, P, P, P]
        L.ms_finish.restype = F
        L.ms_eval.argtypes = [P, P, P, P, U, U, U, P, P, F]
        L.ms_eval.restype = F
        _LIB = L
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data


def oracle_cham_fn(a, b):
    """chamfer_3DDist on the CPU through oracle/chamfer_oracle.py (the reference kernel's rule, ties to the smallest index)."""
    class Fn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, y):
            d1, d2, i1, i2 = chamfer_oracle.chamfer_forward(x.detach().numpy(), y.detach().numpy())
            ctx.save_for_backward(x, y)
            ctx.idx = (i1, i2)
            return torch.from_numpy(d1), torch.from_numpy(d2), torch.from_numpy(i1), torch.from_numpy(i2)

        @staticmethod
        def backward(ctx, g1, g2, *_):
            x, y = ctx.saved_tensors
            gx, gy = chamfer_oracle.chamfer_backward(x.numpy(), y.numpy(), g1.numpy(), g2.numpy(), *ctx.idx)
            return torch.from_numpy(gx), torch.from_numpy(gy)
    return Fn.apply(a.contiguous(), b.contiguous())


def restated(name, recip=False):
    """The restatement on the case's rebuilt inputs: loss and (for train) d loss / d (depth, image)."""
    _, kind, combo, scale, size, _, seed, extra = CASES[name]
    if kind == "train":
        depth, image, gt, rays_d = R.train_inputs(size, seed, ties=extra == "ties")
        assert R.sha(depth, image, gt, rays_d) == str(GOLD[f"{name}/sha"])
        d = torch.from_numpy(depth).requires_grad_(True)
        im = torch.from_numpy(image).requires_grad_(True)
        loss = R.train_ref(d, im, torch.from_numpy(gt), combo, scale, torch.from_numpy(rays_d), oracle_cham_fn,
                           recip=recip)
        loss.backward()
        return loss.item(), d.grad.numpy(), im.grad.numpy()
    B, H, W = size
    depth, image, gt, r = R.eval_inputs(B, H, W, seed, torch.float16 if extra else None, nan=extra == "unet_nan")
    assert R.sha(depth, image, gt, *(() if r is None else (r.float().numpy(),))) == str(GOLD[f"{name}/sha"])
    loss = R.eval_ref(torch.from_numpy(depth), torch.from_numpy(image), torch.from_numpy(gt), combo, scale, raydrop=r)
    return loss.item(), None, None


def grad_tol(combo, *refs):
    """1e-6 of the largest entry.  A cos term's gradient, b / (|a| |b|) - a cos / |a|^2, is the difference of two nearly
    equal fp32 terms when the vectors are nearly parallel (torch rounds them in fp32 too, in another order): 1e-5 of
    the largest entry then, plus 1e-8 for the single-ray cosine, whose gradient is zero and both sides' rounding noise."""
    m = max(float(np.abs(r).max()) for r in refs)
    return 1e-5 * m + 1e-8 if "cos" in combo else 1e-6 * m


def _close(a, b, rel=1e-6):
    if np.isnan(b):
        return np.isnan(a)
    return abs(a - b) <= rel * abs(b)


def test_golden_covers_the_cases():
    assert sorted(str(s) for s in GOLD["names"]) == sorted(CASES)
    combos = {CASES[k][2] for k in TRAIN}
    for slot in range(3):
        assert {c[slot] for c in combos} == set(R.CRITERIA)
    assert {CASES[k][3] for k in TRAIN} == set(R.SCALES)


@pytest.mark.parametrize("name", TRAIN + EVAL)
def test_restatement_reproduces_reference(name):
    """Same ops in the same order as the reference's train_step / eval_step: the same bits."""
    loss, gd, gi = restated(name)
    gl = float(GOLD[f"{name}/loss"])
    assert (np.isnan(gl) and np.isnan(loss)) or np.float32(loss) == np.float32(gl)
    if gd is not None:
        np.testing.assert_array_equal(gd, GOLD[f"{name}/g_depth"])
        np.testing.assert_array_equal(gi, GOLD[f"{name}/g_image"])


def sim_train(name):
    _, _, combo, scale, n, _, seed, extra = CASES[name]
    depth, image, gt, rays_d = R.train_inputs(n, seed, ties=extra == "ties")
    crit = np.array([GRAD_CRITERIA[c] for c in combo], np.uint32)
    alpha = np.array([1.0, 0.01, 0.1], np.float32)
    s = np.zeros(1, np.float64)
    g_pd = np.zeros(n, np.float32)
    gi = np.zeros((1, n, 2), np.float32)
    pred = np.zeros((n, 3), np.float32)
    gtc = np.zeros((n, 3), np.float32)
    lib().ms_train(_p(depth), _p(image), _p(gt), _p(rays_d), n, _p(crit), _p(alpha), 0.2, scale, 0.2 * scale, _p(s),
                   _p(g_pd), _p(gi), _p(pred), _p(gtc))
    d1, d2, i1, i2 = chamfer_oracle.chamfer_forward(pred[None], gtc[None])
    gdist = np.full((1, n), np.float32(0.5) / np.float32(n), np.float32)
    gx1, _ = chamfer_oracle.chamfer_backward(pred[None], gtc[None], gdist, gdist, i1, i2)
    gd = np.zeros((1, n), np.float32)
    loss = lib().ms_finish(_p(gt), _p(rays_d), n, scale, float(s[0]), _p(d1), _p(d2), _p(np.ascontiguousarray(gx1[0])),
                           _p(g_pd), _p(gd))
    # the clouds: torch's `rays_d * pred_depth.unsqueeze(-1) / scale` on the CPU divides; ATen on CUDA (and the kernel)
    # multiplies by the fp32 reciprocal - compare against that form
    m = gt[..., 0]
    inv = np.float32(1) / np.float32(scale)
    np.testing.assert_array_equal(pred, ((rays_d * (depth * m)[..., None]) * inv)[0])
    np.testing.assert_array_equal(gtc, ((rays_d * (gt[..., 2] * m)[..., None]) * inv)[0])
    return loss, gd, gi


@pytest.mark.parametrize("name", TRAIN)
def test_hostsim_train_matches_restatement(name):
    """Against the restatement with the clouds formed as on CUDA (times the fp32 reciprocal of scale; torch on the CPU
    divides, which moves a point by an ulp and a short distance between two points ~80 apart by ~1e-5 relative).
    Loss within 1e-6 relative: the kernel sums in double where torch sums in fp32.  Gradients: grad_tol."""
    loss, gd, gi = sim_train(name)
    ref, rgd, rgi = restated(name, recip=True)
    assert _close(loss, ref), (loss, ref)
    tol = grad_tol(CASES[name][2], rgd, rgi)
    assert np.abs(gi - rgi).max() <= tol
    assert np.abs(gd - rgd).max() <= tol


@pytest.mark.parametrize("name", TRAIN)
def test_hostsim_without_chamfer_matches_restatement(name):
    _, _, combo, scale, n, _, seed, extra = CASES[name]
    depth, image, gt, _ = R.train_inputs(n, seed, ties=extra == "ties")
    crit = np.array([GRAD_CRITERIA[c] for c in combo], np.uint32)
    alpha = np.array([1.0, 0.01, 0.1], np.float32)
    s = np.zeros(1, np.float64)
    g_pd = np.zeros(n, np.float32)
    gi = np.zeros((1, n, 2), np.float32)
    gd = np.zeros((1, n), np.float32)
    lib().ms_train(_p(depth), _p(image), _p(gt), None, n, _p(crit), _p(alpha), 0.2, scale, 0.2 * scale, _p(s), _p(g_pd),
                   _p(gi), None, None)
    loss = lib().ms_finish(_p(gt), None, n, scale, float(s[0]), None, None, None, _p(g_pd), _p(gd))
    d = torch.from_numpy(depth).requires_grad_(True)
    im = torch.from_numpy(image).requires_grad_(True)
    ref = R.train_ref(d, im, torch.from_numpy(gt), combo, scale)
    ref.backward()
    assert _close(loss, ref.item())
    if combo == R.COMBOS["defaults"]:       # the elementwise criteria evaluate torch's expressions op by op
        np.testing.assert_array_equal(gd, d.grad.numpy())
        np.testing.assert_array_equal(gi, im.grad.numpy())
    tol = grad_tol(combo, d.grad.numpy(), im.grad.numpy())
    assert np.abs(gd - d.grad.numpy()).max() <= tol and np.abs(gi - im.grad.numpy()).max() <= tol


@pytest.mark.parametrize("name", EVAL)
def test_hostsim_eval_matches_reference(name):
    _, _, combo, scale, (B, H, W), _, seed, extra = CASES[name]
    depth, image, gt, r = R.eval_inputs(B, H, W, seed, torch.float16 if extra else None, nan=extra == "unet_nan")
    crit = np.array([GRAD_CRITERIA[c] for c in combo], np.uint32)
    alpha = np.array([1.0, 0.01, 0.1], np.float32)
    rf = None if r is None else np.ascontiguousarray(r.float().numpy())
    loss = lib().ms_eval(_p(depth), _p(image), _p(gt), _p(rf), B, H, W, _p(crit), _p(alpha), 0.2 * scale)
    assert _close(loss, float(GOLD[f"{name}/loss"])), (loss, float(GOLD[f"{name}/loss"]))
