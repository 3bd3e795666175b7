"""GPU: the ray-drop refinement stage (lidar4d_b200/refine.py, l4d_refine.cuh) against the reference's own route on CUDA:
  - box_mask against ones_like / slice assignment / multiply, bit for bit, in one launch;
  - raydrop_bce_loss against torch's CUDA BCELoss on in-range predictions only (torch's CUDA kernel asserts on anything
    else; out-of-range and NaN predictions are checked against the CPU rule instead);
  - refine_inputs against the reference's list + cat on the small LiDAR4D test model;
  - trainer_refine against tests/test_refine_oracle.py's mirror of the reference loop, within the mirror's own spread;
  - a bf16 run that learns."""
import argparse
import os

import numpy as np
import pytest
import torch

import refine_cases as RC
from parity_util import fill_state_dict

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _lib():
    from lidar4d_b200 import _capi
    return _capi.load_library()


def _reference_mask(x, boxes):
    mask = torch.ones_like(x)
    for y0, x0, h, w in boxes:
        mask[:, :, y0:y0 + h, x0:x0 + w] = 0.
    return x * mask


def _wild(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(shape, device=DEV, generator=g) * 3
    k = torch.randint(0, 20, shape, device=DEV, generator=g)
    x[k == 0] = float("inf")
    x[k == 1] = float("-inf")
    x[k == 2] = float("nan")
    x[k == 3] = 0.0
    return x


def _random_boxes(rng, H, W, n):
    out = []
    for _ in range(n):
        h, w = int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))
        out.append((int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w))
    return out


@pytest.mark.parametrize("shape", [(47, 3, 66, 1030), (2, 3, 7, 13), (1, 1, 1, 1), (3, 5, 33, 257)])
@pytest.mark.parametrize("kind", ["none", "edges", "max31", "drawn"])
def test_box_mask_bit_identical(shape, kind):
    from lidar4d_b200.refine import box_mask, draw_boxes
    B, C, H, W = shape
    rng = np.random.default_rng(H * W + len(kind))
    if kind == "none":
        boxes = []
    elif kind == "edges":
        boxes = [(0, 0, 1, W), (H - 1, 0, 1, W), (0, 0, H, 1), (0, W - 1, H, 1), (H - 1, W - 1, 1, 1), (0, 0, H, W)][:4 + (H > 2)]
    elif kind == "max31":
        boxes = _random_boxes(rng, H, W, 31)
    else:
        if H < 20 or W < 20:
            pytest.skip("draw_boxes needs int(0.1 * H) > 1")
        np.random.seed(H + W)
        boxes = []
        while not boxes:
            boxes = draw_boxes(H, W)
    x = _wild(shape, H + W)
    ref = _reference_mask(x, boxes)
    lib = _lib()
    n0 = lib.l4d_launch_count()
    out = box_mask(x, boxes)
    assert lib.l4d_launch_count() - n0 == 1
    assert torch.equal(out.view(torch.int32), ref.view(torch.int32))         # -0.0 and NaN included
    y = x.clone()
    box_mask(y, boxes, out=y)                                                 # in place
    assert torch.equal(y.view(torch.int32), ref.view(torch.int32))


def test_box_mask_32_boxes_and_bad_boxes():
    from lidar4d_b200.refine import box_mask
    x = _wild((2, 3, 66, 1030), 5)
    boxes = _random_boxes(np.random.default_rng(0), 66, 1030, 32)
    assert torch.equal(box_mask(x, boxes).view(torch.int32), _reference_mask(x, boxes).view(torch.int32))
    for bad in ([(0, 0, 1, 1)] * 33, [(-1, 0, 2, 2)], [(0, 0, 0, 2)], [(60, 0, 7, 1)], [(0, 1020, 1, 11)], [(0, 0, 1)]):
        with pytest.raises(ValueError):
            box_mask(x, bad)


def _bce_inputs(n, seed, dtype=torch.float32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.rand(n, device=DEV, generator=g)
    t = torch.rand(n, device=DEV, generator=g)
    t[: n // 2] = (t[: n // 2] > 0.5).float()
    k = min(n, 8)           # the -100 clamps, a subnormal, the last float below 1
    x[:k] = torch.tensor([0.0, 1.0, 1e-45, 1 - 2 ** -24, 2 ** -126, 0.5, 1e-3, 0.999], device=DEV)[:k]
    t[:k] = torch.tensor([1.0, 0.0, 1.0, 0.0, 0.3, 0.5, 1.0, 0.0], device=DEV)[:k]
    return x.to(dtype), t


def _ulps(a, b):
    ai, bi = a.view(torch.int32).long(), b.view(torch.int32).long()
    ai = torch.where(ai < 0, -(ai & 0x7FFFFFFF), ai)
    bi = torch.where(bi < 0, -(bi & 0x7FFFFFFF), bi)
    return (ai - bi).abs()


def _ulps16(a, b):
    ai, bi = a.view(torch.int16).int(), b.view(torch.int16).int()
    ai = torch.where(ai < 0, -(ai & 0x7FFF), ai)
    bi = torch.where(bi < 0, -(bi & 0x7FFF), bi)
    return (ai - bi).abs()


def test_bce_elements_against_torch_cuda():
    """The element expression: each element as a loss of n = 1 (the mean of one element is the element)."""
    from lidar4d_b200 import _capi
    lib = _lib()
    x, t = _bce_inputs(4096, 1)
    got = torch.empty_like(x)
    work = torch.empty(lib.l4d_bce_loss_work_bytes(), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    for i in range(x.numel()):
        rc = lib.l4d_bce_loss(x.data_ptr() + 4 * i, _capi.DTYPE_F32, t.data_ptr() + 4 * i, 1, got.data_ptr() + 4 * i,
                              work.data_ptr(), work.numel(), st)
        assert rc == 0
    ref = torch.nn.functional.binary_cross_entropy(x, t, reduction="none")
    u = _ulps(got, ref)
    print(f"[bce] element vs torch CUDA: max {int(u.max())} ulp, {int((u > 0).sum())} of {u.numel()} differ")
    assert int(u.max()) == 0                    # bit-identical on the H100 (the same logf / log1pf and contraction)
    assert got[0].item() == 100.0 and got[1].item() == 100.0


@pytest.mark.parametrize("n", [1, 1000, 4 * 66 * 1030 + 7])
def test_bce_value_and_gradient_against_torch_cuda(n):
    from lidar4d_b200.losses import raydrop_bce_loss
    x, t = _bce_inputs(n, n)
    for scale in (1.0, 65536.0):
        xa = x.clone().requires_grad_()
        loss = raydrop_bce_loss(xa, t)
        (loss * scale).backward()
        xb = x.clone().requires_grad_()
        ref = torch.nn.BCELoss()(xb, t)
        (ref * scale).backward()
        assert loss.dtype == torch.float32 and loss.dim() == 0
        assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item()), (loss.item(), ref.item())
        exact = torch.sum(torch.nn.functional.binary_cross_entropy(x.double(), t.double(), reduction="none")).item() / n
        assert abs(loss.item() - exact) <= 4 * 2 ** -23 * abs(exact) + 1e-30
        u = _ulps(xa.grad, xb.grad)
        print(f"[bce] n={n} scale={scale}: gradient max {int(u.max())} ulp, {int((u > 0).sum())} of {n} differ")
        assert int(u.max()) <= 1        # ATen's CUDA div_(numel) multiplies by the float reciprocal; here it is / n


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_bce_half_predictions(dtype):
    from lidar4d_b200.losses import raydrop_bce_loss
    x, t = _bce_inputs(66 * 1030, 3, dtype)
    xa = x.clone().requires_grad_()
    loss = raydrop_bce_loss(xa, t)
    loss.backward()
    xf = x.float().requires_grad_()
    ref = torch.nn.BCELoss()(xf, t)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
    assert xa.grad.dtype == dtype
    u = _ulps16(xa.grad, xf.grad.to(dtype))          # the float32 gradients differ by <= 1 ulp (see above)
    print(f"[bce] {dtype}: max {int(u.max())} ulp, {int((u > 0).sum())} of {u.numel()} gradients differ from torch's cast back")
    assert int(u.max()) <= 1


def test_bce_and_box_mask_do_not_synchronise():
    from lidar4d_b200.losses import raydrop_bce_loss
    from lidar4d_b200.refine import box_mask
    x, t = _bce_inputs(10000, 4)
    img = torch.rand(2, 3, 66, 1030, device=DEV)
    _lib()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        xa = x.clone().requires_grad_()
        (raydrop_bce_loss(xa, t) * 65536.0).backward()
        box_mask(img, [(1, 2, 3, 4), (10, 20, 5, 6)], out=img)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_out_of_range_predictions_give_nan():
    """torch's CUDA BCE asserts on these, so the reference here is the CPU rule: NaN loss, NaN gradient at the bad
    elements, torch's CPU gradient (BCELoss on the in-range elements with the same n) elsewhere."""
    from lidar4d_b200.losses import raydrop_bce_loss
    x, t = _bce_inputs(1000, 9)
    bad = torch.zeros(1000, dtype=torch.bool, device=DEV)
    bad[[3, 100, 500, 999]] = True
    x[3], x[100], x[500], x[999] = -1e-7, 1.0 + 1e-6, float("nan"), float("inf")
    xa = x.clone().requires_grad_()
    loss = raydrop_bce_loss(xa, t)
    loss.backward()
    assert torch.isnan(loss).item()
    assert bool(torch.isnan(xa.grad[bad]).all()) and bool(torch.isfinite(xa.grad[~bad]).all())
    xc, tc = x.cpu(), t.cpu()
    expect = (xc - tc) / torch.clamp((1 - xc) * xc, min=1e-12) / 1000
    assert torch.equal(xa.grad[~bad].cpu(), expect[~bad.cpu()])


# ---------------------------------------------------------------------------------------------------------------------
# refine_inputs on the small LiDAR4D test model
# ---------------------------------------------------------------------------------------------------------------------
class _RayLoader:
    def __init__(self, H, W, n, dtype):
        from lidar4d_b200.rays import lidar_rays
        self.items = []
        for i in range(n):
            pose = np.eye(4, dtype=np.float32)
            pose[:3, 3] = (0.1 * i, -0.05 * i, 0.02)
            ro, rd = lidar_rays(pose, H, W)
            g = np.random.default_rng(i)
            gt = np.stack([(g.uniform(0, 1, (H, W)) > 0.3), g.uniform(0, 1, (H, W)), g.uniform(0, 1, (H, W))], -1)
            self.items.append({"rays_o_lidar": torch.from_numpy(ro)[None].to(DEV), "rays_d_lidar": torch.from_numpy(rd)[None].to(DEV),
                               "time": torch.tensor([[i / max(n - 1, 1)]], device=DEV), "H_lidar": H, "W_lidar": W,
                               "images_lidar": torch.from_numpy(gt.astype(np.float32))[None].to(DEV, dtype)})

    def __len__(self):
        return len(self.items)

    def __iter__(self):
        return iter(self.items)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_refine_inputs_equal_the_reference_route(dtype):
    from oracle import lidar4d_oracle as O
    from parity_util import small_config, cuda_model_from_oracle
    from lidar4d_b200.refine import refine_inputs
    model = cuda_model_from_oracle(O.build_seeded(small_config(), 11, flow_last_std=0.02)).set_mlp_fp16(True).eval()
    loader = _RayLoader(8, 64, 3, dtype)
    opt = argparse.Namespace(num_steps=64, fp16=True)
    inputs, gt = refine_inputs(model, loader, fp16=True, opt=opt)
    ins, gts = [], []
    for data in loader:                                     # runner.py:833-863
        H, W = data["H_lidar"], data["W_lidar"]
        with torch.autocast("cuda", enabled=True), torch.no_grad():
            out = model.render(data["rays_o_lidar"], data["rays_d_lidar"], data["time"], staged=True, max_ray_batch=4096,
                               perturb=False, **vars(opt))
        img = out["image_lidar"].reshape(-1, H, W, 2)
        ins.append(torch.cat([img[..., 0], img[..., 1], out["depth_lidar"].reshape(-1, H, W)], 0).unsqueeze(0))
        gts.append(data["images_lidar"][:, :, :, 0].unsqueeze(0))
    ref_in = torch.cat(ins, 0).cuda().float().contiguous()
    ref_gt = torch.cat(gts, 0).cuda().float().contiguous()
    assert inputs.shape == (3, 3, 8, 64) and gt.shape == (3, 1, 8, 64)
    assert torch.equal(inputs, ref_in) and torch.equal(gt, ref_gt)


# ---------------------------------------------------------------------------------------------------------------------
# trainer_refine against the mirror of the reference loop
# ---------------------------------------------------------------------------------------------------------------------
ITERS = 20


def _run(fn, tmp, tag):
    from lidar4d_b200.raydrop_unet import RayDropUNet
    model = RC.StubModel(RC.frames(), fill_state_dict(RayDropUNet(3, 32, 1))).to(DEV)
    os.makedirs(os.path.join(tmp, tag))
    tr = RC.StubTrainer(model, os.path.join(tmp, tag))
    np.random.seed(RC.NP_SEED)
    torch.manual_seed(RC.TORCH_SEED)
    losses = fn(tr, RC.Loader(RC.frames(), torch.float16, DEV))
    state = np.random.get_state()
    ck = torch.load(os.path.join(tmp, tag, "lidar4d_ep0003_refine.pth"), weights_only=False)
    return np.asarray(losses, np.float64), state, ck, tr


def test_trainer_refine_against_the_mirror(tmp_path):
    from test_refine_oracle import mirror_refine
    from lidar4d_b200.refine import trainer_refine
    det = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        mirror = lambda tr, ld: mirror_refine(tr, ld, epochs=ITERS, device=DEV)[0]
        ours = lambda tr, ld: trainer_refine(tr, ld, epochs=ITERS).cpu().numpy()
        m1, s1, c1, _ = _run(mirror, str(tmp_path), "m1")
        m2, s2, c2, _ = _run(mirror, str(tmp_path), "m2")
        o, so, co, tro = _run(ours, str(tmp_path), "ours")
    finally:
        torch.backends.cudnn.deterministic = det
    for s in (s2, so):
        assert np.array_equal(s[1], s1[1]) and s[2] == s1[2]          # the same box draws, the same final state
    assert abs(o[0] - m1[0]) <= 1e-6 * abs(m1[0]), (o[0], m1[0])
    spread = np.abs(m2 - m1).max()
    diff = np.abs(o - m1).max()
    print(f"[refine] losses: mirror spread {spread:.3e}, trainer_refine vs mirror {diff:.3e}")
    assert diff <= 4 * spread + 1e-5 * np.abs(m1).max()
    w1, w2, wo = c1["model"], c2["model"], co["model"]
    assert sorted(co.keys()) == sorted(c1.keys()) == ["epoch", "model"] and co["epoch"] == c1["epoch"] == 3
    assert list(wo.keys()) == list(w1.keys())
    wspread = max((w2[k].double() - w1[k].double()).abs().max().item() for k in w1 if w1[k].is_floating_point())
    wdiff = max((wo[k].double() - w1[k].double()).abs().max().item() for k in w1 if w1[k].is_floating_point())
    wmax = max(w1[k].double().abs().max().item() for k in w1 if w1[k].is_floating_point())
    print(f"[refine] weights: mirror spread {wspread:.3e}, trainer_refine vs mirror {wdiff:.3e}")
    assert wdiff <= 4 * wspread + 1e-5 * wmax
    assert [ln for ln in tro.lines if "iter:" not in ln] == ["Preparing for Raydrop Refinemet ...", "Start UNet Optimization ..."]
    assert sum("iter:0," in ln for ln in tro.lines) == 1


def test_train_unet_does_not_synchronise_between_log_points():
    """Scoped to the whole loop body: the index copy, box_mask, the U-Net, raydrop_bce_loss, backward, torch's Adam
    and OneCycleLR."""
    from lidar4d_b200.raydrop_unet import RayDropUNet
    from lidar4d_b200.refine import train_unet
    unet = fill_state_dict(RayDropUNet(3, 32, 1)).to(DEV).train()
    inputs = torch.rand(4, 3, 32, 64, device=DEV)
    gt = (torch.rand(4, 1, 32, 64, device=DEV) > 0.5).float()
    np.random.seed(0)
    train_unet(unet, inputs, gt, epochs=2, batch_size=3)         # warm-up: cuDNN plans, Adam state
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = train_unet(unet, inputs, gt, epochs=6, batch_size=3)
        losses = train_unet(unet, inputs, gt, epochs=6)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert bool(torch.isfinite(losses).all())


def test_bf16_run_learns():
    from lidar4d_b200.raydrop_unet import RayDropUNet
    from lidar4d_b200.refine import train_unet
    torch.manual_seed(0)
    unet = RayDropUNet(3, 32, 1).to(DEV).train()
    g = torch.Generator(device=DEV).manual_seed(1)
    inputs = torch.rand(6, 3, 64, 256, device=DEV, generator=g)
    gt = (inputs[:, :1] > 0.4).float()                    # the ray drop is the first channel thresholded
    np.random.seed(1)
    losses = train_unet(unet, inputs, gt, epochs=50, autocast_dtype=torch.bfloat16).cpu().numpy()
    print(f"[refine] bf16 losses: first {losses[:3]}, last {losses[-3:]}")
    assert np.isfinite(losses).all()
    assert losses[-10:].mean() < 0.7 * losses[:10].mean()
