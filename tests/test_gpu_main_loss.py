"""GPU: the main LiDAR loss ops (lidar4d_b200.losses.lidar_main_loss / lidar_eval_loss) against the torch restatement
(tests/main_loss_ref.py, pinned to the reference Trainer by tests/test_main_loss_hostsim.py) on identical CUDA tensors,
with lidar4d_b200.chamfer.chamfer_3DDist as the restatement's chamfer function."""
import ctypes as C

import numpy as np
import pytest
import torch

import main_loss_ref as R
from trainer_mirror import MirrorTrainer, default_opt

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SIZES = [(1, None), (37, None), (1024, None), (4096, None), (65536, None), (32, (2, 8)), (1024, (4, 16))]


def cham_fn():
    from lidar4d_b200.chamfer import chamfer_3DDist
    return chamfer_3DDist()


def inputs(n, seed, ties=False):
    return [torch.from_numpy(a).to(DEV) for a in R.train_inputs(n, seed, ties)]


def op(depth, image, gt, combo, scale, rays_d=None):
    from lidar4d_b200.losses import lidar_main_loss
    return lidar_main_loss(depth, image, gt, 1.0, 0.01, 0.1, 0.2, depth_loss=combo[0], raydrop_loss=combo[1],
                           intensity_loss=combo[2], scale=scale, rays_d=rays_d)


def grad_tol(combo, *refs):
    """1e-6 of the largest entry; for a cos term 1e-5 (+1e-8): its gradient is the difference of two nearly equal fp32
    terms when the vectors are nearly parallel, rounded by torch in another order (tests/test_main_loss_hostsim.py)."""
    m = max(float(r.abs().max()) for r in refs)
    return 1e-5 * m + 1e-8 if "cos" in combo else 1e-6 * m


def both(n, combo, scale, seed, ties=False, chamfer=True):
    depth, image, gt, rays_d = inputs(n, seed, ties)
    d1, i1 = depth.clone().requires_grad_(True), image.clone().requires_grad_(True)
    d2, i2 = depth.clone().requires_grad_(True), image.clone().requires_grad_(True)
    loss = op(d1, i1, gt, combo, scale, rays_d if chamfer else None)
    loss.backward()
    ref = R.train_ref(d2, i2, gt, combo, scale, rays_d, cham_fn() if chamfer else None)
    ref.backward()
    return loss, ref, (d1.grad, i1.grad), (d2.grad, i2.grad)


@pytest.mark.parametrize("n,patch", SIZES)
@pytest.mark.parametrize("cname", list(R.COMBOS))
def test_train_matches_restatement(cname, n, patch):
    """Loss within 1e-6 relative (double against fp32 sums); gradients within grad_tol.  The chamfer gradient reaches
    both sides through fp32 atomics (chamfer_3DDist's backward too), so its order differs run to run on either side."""
    combo = R.COMBOS[cname]
    for scale in R.SCALES:
        loss, ref, (gd, gi), (rd, ri) = both(n, combo, scale, 11 + n)
        assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item()), (loss.item(), ref.item())
        tol = grad_tol(combo, rd, ri)
        assert float((gd - rd).abs().max()) <= tol and float((gi - ri).abs().max()) <= tol


@pytest.mark.parametrize("cname", ["defaults", "all_bce", "all_cos", "depth_huber"])
def test_ties_at_the_origin(cname):
    combo = R.COMBOS[cname]
    loss, ref, (gd, gi), (rd, ri) = both(4096, combo, 0.01, 5, ties=True)
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
    tol = grad_tol(combo, rd, ri)
    assert float((gd - rd).abs().max()) <= tol and float((gi - ri).abs().max()) <= tol


def _raw_call(n, seed, scale, crit=(0, 1, 1)):
    """l4d_main_loss through the C-ABI, returning (loss, g_depth, g_image, work)."""
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    depth, image, gt, rays_d = inputs(n, seed)
    work = torch.empty(lib.l4d_main_loss_work_bytes(n), dtype=torch.uint8, device=DEV)
    loss = torch.empty((), device=DEV)
    gd, gi = torch.empty(n, device=DEV), torch.empty(n, 2, device=DEV)
    rc = lib.l4d_main_loss(depth.data_ptr(), image.data_ptr(), gt.data_ptr(), rays_d.data_ptr(), n, *crit, 1.0, 0.01, 0.1,
                           0.2, scale, 0.2 * scale, loss.data_ptr(), gd.data_ptr(), gi.data_ptr(), work.data_ptr(),
                           work.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.l4d_last_error()
    return (depth, image, gt, rays_d), loss, gd, gi, work


@pytest.mark.parametrize("scale", R.SCALES)
def test_clouds_bit_identical_to_torch(scale):
    n = 4096
    (depth, image, gt, rays_d), *_, work = _raw_call(n, 3, scale)
    torch.cuda.synchronize()
    clouds = work[:6 * n * 4].view(torch.float32).view(2, 1, n, 3)
    m = gt[:, :, 0]
    assert torch.equal(clouds[0], rays_d * (depth * m).unsqueeze(-1) / scale)
    assert torch.equal(clouds[1], rays_d * (gt[:, :, 2] * m).unsqueeze(-1) / scale)


def test_default_gradient_bit_identical_without_chamfer():
    """The default criteria without rays_d: the gradient is the current formula, op by op."""
    depth, image, gt, _ = inputs(5000, 4)
    d, im = depth.clone().requires_grad_(True), image.clone().requires_grad_(True)
    g = 3.0
    gd, gi = torch.autograd.grad(op(d, im, gt, R.COMBOS["defaults"], 0.01) * g, (d, im))
    m = gt[:, :, 0]
    ref_d = 1.0 * torch.sign(depth * m - gt[:, :, 2] * m) * m * g
    ref_r = 0.01 * (2 * (image[:, :, 0] - m.clamp(0.2, 0.8))) * g
    ref_i = 0.1 * (2 * (image[:, :, 1] * m - gt[:, :, 1] * m)) * m * g
    assert torch.equal(gd, ref_d)
    assert torch.equal(gi, torch.stack([ref_r, ref_i], -1))


@pytest.mark.parametrize("chamfer", [False, True])
def test_repeated_calls_are_bit_identical(chamfer):
    depth, image, gt, rays_d = inputs(65536, 9)
    res = []
    for _ in range(3):
        d, im = depth.clone().requires_grad_(True), image.clone().requires_grad_(True)
        loss = op(d, im, gt, R.COMBOS["depth_cos"], 0.01, rays_d if chamfer else None)
        loss.backward()
        res.append((loss.detach().clone(), d.grad, im.grad))
    for r in res[1:]:
        assert torch.equal(r[0], res[0][0])
        if not chamfer:       # the chamfer gradient reaches depth through fp32 atomics
            assert torch.equal(r[1], res[0][1]) and torch.equal(r[2], res[0][2])


def test_launch_count_is_fixed():
    """Without the chamfer term: one launch forward, one backward, for every n.  With it: two more than the chamfer
    op's own launches at that n (l4d_chamfer_forward uses one launch per direction for small clouds, three otherwise)."""
    from lidar4d_b200 import _capi
    lib = _capi.load_library()
    for n in (1, 1024, 65536):
        depth, image, gt, rays_d = inputs(n, 1)
        for chamfer in (False, True):
            d = depth.clone().requires_grad_(True)
            c0 = lib.l4d_launch_count()
            loss = op(d, image, gt, R.COMBOS["all_bce"], 0.01, rays_d if chamfer else None)
            c1 = lib.l4d_launch_count()
            loss.backward()
            c2 = lib.l4d_launch_count()
            cham = 0
            if chamfer:
                p = torch.zeros(1, n, 3, device=DEV)
                cf = cham_fn()
                a = lib.l4d_launch_count()
                dist1, dist2, _, _ = cf(p.requires_grad_(True), torch.zeros(1, n, 3, device=DEV))
                b = lib.l4d_launch_count()
                (dist1.sum() + dist2.sum()).backward()
                cham = (b - a) + (lib.l4d_launch_count() - b)
            assert c1 - c0 == (1 if not chamfer else 2 + cham)
            assert c2 - c1 == 1


def test_no_host_sync():
    depth, image, gt, rays_d = inputs(4096, 2)
    d = depth.clone().requires_grad_(True)
    scaler_g = torch.full((), 65536.0, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = op(d, image, gt, ("huber", "bce", "cos"), 0.01, rays_d)
        (loss * scaler_g).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(d.grad).all()


def test_errors():
    from lidar4d_b200.losses import lidar_main_loss, lidar_eval_loss
    depth, image, gt, rays_d = inputs(16, 0)
    with pytest.raises(ValueError):
        lidar_main_loss(depth, image, gt, depth_loss="l2")
    with pytest.raises(ValueError):
        lidar_main_loss(depth, image, gt, rays_d=rays_d)                 # chamfer without scale
    with pytest.raises(ValueError):
        lidar_main_loss(depth, image, gt, depth_loss="huber")            # huber without scale
    with pytest.raises(RuntimeError):
        lidar_main_loss(depth.cpu(), image.cpu(), gt.cpu())
    with pytest.raises(ValueError):
        lidar_eval_loss(depth, image, gt.view(1, 4, 4, 3), raydrop_loss="x")


# ---- a training iteration of the Trainer with the op swapped in -------------------------------------------------------
class _TinyModel(torch.nn.Module):
    """render: depth and image from the ray directions through two small linear maps (enough to carry gradients)."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.wd = torch.nn.Linear(3, 1)
        self.wi = torch.nn.Linear(3, 2)
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)

    def render(self, rays_o, rays_d, t, **_):
        return {"depth_lidar": torch.sigmoid(self.wd(rays_d))[..., 0] * 0.8, "image_lidar": self.wi(rays_d)}


class FusedTrainer(MirrorTrainer):
    """train_step with runner.py:193-220 replaced by the one call of INTEGRATION.md section 5."""

    def train_step(self, data):
        from lidar4d_b200.losses import lidar_main_loss
        o = self.opt
        out = self.model.render(data["rays_o_lidar"], data["rays_d_lidar"], data["time"])
        loss = lidar_main_loss(out["depth_lidar"], out["image_lidar"], data["images_lidar"], o.alpha_d, o.alpha_r,
                               o.alpha_i, o.smooth_factor, depth_loss=o.depth_loss, raydrop_loss=o.raydrop_loss,
                               intensity_loss=o.intensity_loss, scale=o.scale, rays_d=data["rays_d_lidar"])
        return None, None, None, None, loss


def test_trainer_iteration_fp16_gradscaler():
    n = 1024
    depth, image, gt, rays_d = inputs(n, 21)
    data = {"rays_o_lidar": torch.zeros(1, n, 3, device=DEV), "rays_d_lidar": rays_d, "time": torch.zeros(1, 1, device=DEV),
            "images_lidar": gt}
    opt = default_opt(depth_loss="huber", raydrop_loss="bce", intensity_loss="mse", flow_loss=False, fp16=True)
    crit = {"depth": R.criterion("huber", opt.scale), "raydrop": R.criterion("bce", opt.scale),
            "intensity": R.criterion("mse", opt.scale)}
    res = []
    for cls in (MirrorTrainer, FusedTrainer):
        model = _TinyModel().to(DEV)
        tr = cls(opt, model, cham_fn(), criterion=crit, optimizer=lambda m: torch.optim.Adam(m.parameters(), lr=1e-3),
                 fp16=True, device=DEV)
        losses = [tr.train_iteration(data) for _ in range(3)]
        res.append((losses, [p.detach().clone() for p in model.parameters()]))
    for a, b in zip(res[0][0], res[1][0]):
        assert abs(a - b) <= 1e-5 * abs(a), (res[0][0], res[1][0])
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.allclose(a, b, rtol=0, atol=1e-5)


# ---- eval -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 66, 1030), (1, 128, 2048)])
@pytest.mark.parametrize("unet", [None, torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("cname", list(R.COMBOS))
def test_eval_matches_restatement(cname, unet, shape):
    from lidar4d_b200.losses import lidar_eval_loss
    combo = R.COMBOS[cname]
    B, H, W = shape
    depth, image, gt, r = R.eval_inputs(B, H, W, 17, unet)
    depth, image, gt = (torch.from_numpy(a).to(DEV) for a in (depth, image, gt))
    r = None if r is None else r.to(DEV)
    loss = lidar_eval_loss(depth.view(B, H * W), image.view(B, H * W, 2), gt, r, alpha_d=1.0, alpha_r=0.01, alpha_i=0.1,
                           depth_loss=combo[0], raydrop_loss=combo[1], intensity_loss=combo[2], scale=0.01)
    with torch.autocast("cuda", dtype=torch.float16):
        ref = R.eval_ref(depth, image, gt, combo, 0.01, raydrop=r)
    assert loss.dtype == torch.float32 and loss.shape == ()
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item()), (loss.item(), ref.item())
