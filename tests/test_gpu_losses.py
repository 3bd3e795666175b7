"""GPU: the patch losses and the line-of-sight loss as CUDA ops (lidar4d_b200.losses), against the torch restatement of
model/runner.py:255-369 (tests/loss_ref.py) on identical CUDA tensors, and through a Trainer mirror against the
unmodified reference Trainer's values (tests/golden/train_losses.npz)."""
import os

import numpy as np
import pytest
import torch

import loss_ref
from lidar4d_b200.losses import GRAD_CRITERIA, lidar_patch_loss, line_of_sight_loss
from trainer_mirror import MirrorTrainer, default_opt, default_criterion
from parity_util import small_config, cuda_model_from_oracle
from oracle import lidar4d_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "train_losses.npz"), allow_pickle=False)


def launches():
    from lidar4d_b200 import _capi
    return int(_capi.load_library().l4d_launch_count())


def _grad_close(a, b, tol=1e-6):
    a, b = a.double(), b.double()
    return float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-30)


def _run(fn, x, *args, g_out=1.0, **kw):
    x = x.detach().clone().requires_grad_(True)
    loss = fn(x, *args, **kw)
    if not loss.requires_grad:                 # the restatement's px == 1: a constant 0
        return loss.detach(), torch.zeros_like(x)
    loss.backward(torch.tensor(g_out, device=DEV))
    return loss.detach(), x.grad


@pytest.fixture(autouse=True)
def _fp32_conv():
    """The restatement's Sobel conv2d in fp32, not TF32 (cuDNN's default on the H100): the reference's own CPU run and
    these ops compute it in fp32, and TF32 would round depth / scale ~ 65 to 0.03."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def patch_inputs(n, px, py, seed, mask_first=False):
    n_patch = max(1, n // (px * py))
    gt = loss_ref.patch_gt(n_patch, px, py, seed=seed)
    if mask_first:
        gt[: px * py, 0] = 0.0
    rng = np.random.default_rng(seed + 1)
    m = gt.shape[0]
    depth = loss_ref.quantize(gt[:, 2].numpy() + rng.normal(0, 3e-5, m) * (rng.random(m) > 0.2))
    return torch.from_numpy(depth).to(DEV), gt.to(DEV)


PATCHES = [[2, 8], 4, [3, 5], [1, 8]]
OPTIONS = [dict(depth_grad_loss=c, sobel_grad=s) for c in GRAD_CRITERIA for s in (False, True)] + \
    [dict(grad_norm_smooth=True, spatial_smooth=True, tv_loss=True, sobel_grad=s) for s in (False, True)]


def _cos_scale(depth, gt, patch, **opts):
    from test_losses_hostsim import cos_term_scale
    return cos_term_scale(depth.cpu().numpy(), gt.cpu().numpy(), patch, **opts)


@pytest.mark.parametrize("n", [16, 1024, 65536])
@pytest.mark.parametrize("patch", PATCHES, ids=str)
@pytest.mark.parametrize("opts", OPTIONS, ids=lambda o: "-".join(f"{k}={v}" for k, v in o.items()))
def test_patch_loss_matches_restatement(n, patch, opts):
    px, py = (patch, patch) if isinstance(patch, int) else patch
    depth, gt = patch_inputs(n, px, py, seed=n + px * 10 + py, mask_first=True)
    for g_out in (1.0, 65536.0):
        v, g = _run(lidar_patch_loss, depth, gt, patch, 0.01, g_out=g_out, **opts)
        v_r, g_r = _run(loss_ref.patch_ref, depth, gt, patch, g_out=g_out, **opts)
        if torch.isnan(v_r):           # the mean over an empty dx or dy is nan in the reference as well
            assert torch.isnan(v)
            continue
        assert float(v) == pytest.approx(float(v_r), rel=1e-5, abs=1e-7)
        if opts.get("depth_grad_loss") == "cos":
            bound = 1e-6 * g_out * max(float(g_r.abs().max()) / g_out, _cos_scale(depth, gt, patch, **opts))
            assert float((g - g_r).abs().max()) <= bound
        else:
            assert _grad_close(g, g_r)
        if opts == dict(depth_grad_loss="l1", sobel_grad=False):
            # sign-type derivatives: equal wherever the restatement's is not an exact zero of a sum of signs
            nz = g_r != 0
            assert torch.equal(g[nz], g_r[nz])


def test_patch_loss_all_masked_patches_and_launches():
    depth, gt = patch_inputs(1024, 2, 8, seed=3)
    gt[:, 0] = 0.0                                         # every ray dropped: every patch all-masked
    before = launches()
    v, g = _run(lidar_patch_loss, depth, gt, [2, 8], 0.01, depth_grad_loss="cos")
    assert launches() - before == 2                        # forward one launch, backward one launch
    assert float(v) == pytest.approx(0.1 * 64) and torch.count_nonzero(g) == 0


def test_patch_loss_is_deterministic_and_rejects_bad_input():
    depth, gt = patch_inputs(65536, 2, 8, seed=5)
    a = _run(lidar_patch_loss, depth, gt, [2, 8], 0.01, sobel_grad=True, spatial_smooth=True)
    b = _run(lidar_patch_loss, depth, gt, [2, 8], 0.01, sobel_grad=True, spatial_smooth=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    with pytest.raises(RuntimeError):
        lidar_patch_loss(depth.cpu(), gt.cpu(), [2, 8], 0.01)
    with pytest.raises(ValueError):
        lidar_patch_loss(depth[:-1], gt[:-1], [2, 8], 0.01)           # not a whole number of patches
    with pytest.raises(ValueError):
        lidar_patch_loss(depth, gt[:-1], [2, 8], 0.01)
    with pytest.raises(ValueError):
        lidar_patch_loss(depth, gt, [2, 8], 0.01, depth_grad_loss="l2")


def los_inputs(n, S, seed, inside=False, no_valid=False):
    g = np.random.default_rng(seed)
    gt = np.stack([(g.random(n) > 0.2), g.random(n), 0.05 + 0.6 * g.random(n)], -1).astype(np.float32)
    if no_valid:
        gt[:, 0] = 0.0
    gd = gt[:, 2] * gt[:, 0]
    if inside:
        z = gd[:, None] + g.uniform(-0.015, 0.015, (n, S))
    else:
        z = np.sort(g.uniform(0.01, 0.85, (n, S)), axis=1)
        z[:, :4] = gd[:, None] + g.uniform(-0.015, 0.015, (n, 4))
    w = g.random((n, S)) ** 4
    return (torch.from_numpy(w.astype(np.float32)).to(DEV), torch.from_numpy(z.astype(np.float32)).to(DEV),
            torch.from_numpy(gt).to(DEV))


@pytest.mark.parametrize("n", [16, 1024, 65536])
@pytest.mark.parametrize("S", [48, 768])
def test_line_of_sight_matches_restatement(n, S):
    w, z, gt = los_inputs(n, S, seed=n + S)
    eps = loss_ref.los_eps(1500, 30000)
    for g_out in (1.0, 65536.0):
        v, g = _run(line_of_sight_loss, w, z, gt, eps, g_out=g_out)
        v_r, g_r = _run(loss_ref.line_of_sight_ref, w, z, gt, eps, g_out=g_out)
        assert float(v) == pytest.approx(float(v_r), rel=1e-5)
        assert _grad_close(g, g_r)


@pytest.mark.parametrize("n,S", [(16, 48), (1024, 768)])
def test_line_of_sight_all_samples_in_window(n, S):
    """No sample lies outside its window: max(distr) < its peak, the second launch re-reads [n, S]."""
    w, z, gt = los_inputs(n, S, seed=7, inside=True)
    v, g = _run(line_of_sight_loss, w, z, gt, 0.02)
    v_r, g_r = _run(loss_ref.line_of_sight_ref, w, z, gt, 0.02)
    assert float(v) == pytest.approx(float(v_r), rel=1e-5)
    assert _grad_close(g, g_r)


def test_line_of_sight_without_valid_rays_determinism_and_launches():
    w, z, gt = los_inputs(64, 48, seed=2, no_valid=True)
    v, _ = _run(line_of_sight_loss, w, z, gt, 0.02)
    v_r, _ = _run(loss_ref.line_of_sight_ref, w, z, gt, 0.02)
    assert not torch.isfinite(v_r) and torch.isnan(v) == torch.isnan(v_r) and torch.isinf(v) == torch.isinf(v_r)
    w, z, gt = los_inputs(65536, 768, seed=4)
    before = launches()
    a = _run(line_of_sight_loss, w, z, gt, 0.02)
    assert launches() - before == 3                        # forward two launches, backward one
    b = _run(line_of_sight_loss, w, z, gt, 0.02)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    with pytest.raises(RuntimeError):
        line_of_sight_loss(w.cpu(), z.cpu(), gt.cpu(), 0.02)
    with pytest.raises(ValueError):
        line_of_sight_loss(w, z[:, :-1], gt, 0.02)


# ---- the Trainer path -------------------------------------------------------------------------------------------------
class LossMirrorTrainer(MirrorTrainer):
    """MirrorTrainer + runner.py:255-369: the restated torch expressions, or the fused CUDA ops with `fused = True`."""
    fused = False

    def train_step(self, data):
        o, cap = self.opt, {}
        render = self.model.render

        def capture(*a, **k):
            cap.update(render(*a, **k))
            return cap
        self.model.render = capture
        try:
            res = super().train_step(data)
        finally:
            del self.model.render
        loss, gt = res[4], data["images_lidar"]
        if self.fused:
            if o.urf_loss:
                loss = loss + line_of_sight_loss(cap["weights"], cap["z_vals"], gt, loss_ref.los_eps(self.global_step, o.iters))
            loss = loss + lidar_patch_loss(cap["depth_lidar"], gt, o.patch_size_lidar, **vars(o))
        else:
            loss = loss + loss_ref.extra_losses_ref(cap, gt, o, self.global_step)
        return (*res[:4], loss)


def _zero(a, b):
    return a * 0.0


def _golden_trainer(name, fused):
    orc = O.build_seeded(small_config(), int(GOLD["seed"]), flow_last_std=0.02)
    model = cuda_model_from_oracle(orc)
    model.jitter_seed = int(GOLD["seed"])
    kw = dict(num_frames=6, num_steps=int(GOLD["num_steps"]), near_lidar=0.0105, far_lidar=0.851, fp16=False,
              iters=int(GOLD["iters"]), patch_size_lidar=[2, 8], flow_loss=False, **loss_ref.DEFAULTS)
    kw.update(loss_ref.OPTION_SETS[name])
    # the main-loss criteria and the chamfer distances are zero, as in tests/golden/make_loss_golden.py
    crit = {"depth": _zero, "raydrop": _zero, "intensity": _zero, "grad": None}
    tr = LossMirrorTrainer(default_opt(**kw), model, lambda a, b: (a[..., 0] * 0.0, b[..., 0] * 0.0, None, None),
                           criterion=crit, device=DEV)
    tr.fused = fused
    tr.global_step = int(GOLD["global_step"])
    data = {"rays_o_lidar": torch.from_numpy(GOLD["rays_o"]).to(DEV), "rays_d_lidar": torch.from_numpy(GOLD["rays_d"]).to(DEV),
            "time": torch.from_numpy(GOLD["time"]).to(DEV), "images_lidar": torch.from_numpy(GOLD["images"]).to(DEV)}
    return tr, model, data


@pytest.mark.parametrize("name", [str(s) for s in GOLD["names"]])
def test_trainer_mirror_reproduces_reference_losses(name):
    losses, grads = {}, {}
    for fused in (False, True):
        tr, model, data = _golden_trainer(name, fused)
        model._jitter_calls = 0
        loss = tr.train_step(data)[4]
        loss.backward()
        torch.cuda.synchronize()
        losses[fused] = float(loss)
        grads[fused] = [p.grad.detach().clone() for p in model.parameters() if p.grad is not None]
    assert losses[False] == pytest.approx(float(GOLD[f"{name}/loss"]), rel=2e-4)
    assert losses[True] == pytest.approx(losses[False], rel=1e-5)
    assert len(grads[True]) == len(grads[False]) > 0
    for a, b in zip(grads[True], grads[False]):
        assert _grad_close(a, b, tol=1e-5)


def test_trainer_trains_through_fused_losses_with_fp16_autocast():
    from lidar4d_b200.chamfer import chamfer_3DDist
    from lidar4d_b200.optim import Adam
    from lidar4d_b200.rays import get_lidar_rays
    orc = O.build_seeded(small_config(), 31, flow_last_std=0.02)
    model = cuda_model_from_oracle(orc)
    opt = default_opt(num_frames=6, num_steps=48, near_lidar=0.0105, far_lidar=0.851, fp16=True, flow_loss=False,
                      patch_size_lidar=[2, 8], urf_loss=True)
    tr = LossMirrorTrainer(opt, model, chamfer_3DDist(), criterion=default_criterion(), device=DEV, fp16=True,
                           optimizer=lambda m: Adam(m, m.get_params(1e-2), betas=(0.9, 0.99), eps=1e-15))
    tr.fused = True
    g = np.random.default_rng(0)
    img = np.stack([g.random((8, 32)) > 0.15, g.random((8, 32)) * 0.5, 0.05 + 0.6 * g.random((8, 32))], -1)
    pose = torch.eye(4, device=DEV)[None]
    pose[0, 0, 3] = -0.05
    torch.manual_seed(0)
    r = get_lidar_rays(pose, (2.0, 26.9), 8, 32, N=256, patch_size=[2, 8],
                       images=torch.from_numpy(img.astype(np.float32))[None].to(DEV))
    data = {"rays_o_lidar": r["rays_o"], "rays_d_lidar": r["rays_d"], "time": torch.tensor([[0.4]], device=DEV),
            "images_lidar": r["gt"]}
    losses = [tr.train_iteration(data) for _ in range(3)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
