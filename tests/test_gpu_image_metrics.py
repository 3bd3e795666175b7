"""The depth / intensity / ray-drop meters on the GPU (lidar4d_b200.metrics: image_metrics, raydrop_metrics,
DepthMeter, IntensityMeter, RaydropMeter) against the reference's rows (tests/golden/image_metrics_ref.npz) and the
oracle (oracle/image_metrics_oracle.py) on identical CUDA tensors.

Tolerances: MedAE, accuracy and F1 bit-identical (every NaN and inf in the same slot); RMSE within 4e-6 relative and
PSNR within 2e-5 dB (NumPy's float32 mean sums in another order); SSIM within 2e-7 of skimage's powf constants and
within 1e-12 of the same expression with x*x constants (the kernels' choice; only the float64 mean's order differs)."""
import ctypes as C
import os
import warnings

import numpy as np
import pytest
import torch

import image_metrics_cases as IC
from oracle import image_metrics_oracle as IO

pytestmark = pytest.mark.gpu
FX = np.load(os.path.join(os.path.dirname(__file__), "golden", "image_metrics_ref.npz"), allow_pickle=False)
DEV = "cuda:0"


def _lib():
    from lidar4d_b200 import _capi
    return _capi.load_library()


def _same(a, b):
    a, b = np.float64(a), np.float64(b)
    return (np.isnan(a) and np.isnan(b)) or a.tobytes() == b.tobytes()


def _near(a, b, rel=0.0, abs_=0.0):
    a, b = np.float64(a), np.float64(b)
    if not (np.isfinite(a) and np.isfinite(b)):
        return _same(a, b) or (np.isnan(a) and np.isnan(b))
    return abs(a - b) <= max(rel * abs(b), abs_)


def check_image_row(row, ref, ssim_mul=None):
    """row: the kernels' (rmse, medae, lpips, ssim, psnr); ref: the reference's (powf) row."""
    assert _same(row[1], ref[1]), ("medae", row[1], ref[1])
    assert _near(row[0], ref[0], rel=4e-6), ("rmse", row[0], ref[0])
    assert _near(row[4], ref[4], abs_=2e-5), ("psnr", row[4], ref[4])
    assert _near(row[3], ref[3], abs_=2e-7), ("ssim", row[3], ref[3])
    if ssim_mul is not None:
        assert _near(row[3], ssim_mul, abs_=1e-12), ("ssim vs x*x constants", row[3], ssim_mul)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("name", IC.IMAGE_CASES)
def test_image_metrics_match_reference(name):
    from lidar4d_b200.metrics import image_metrics
    kind, p, g = IC.frame(FX, name)
    lo, hi, peak = IO.DEPTH if kind == "depth" else IO.INTENSITY
    out = image_metrics(_cuda(p[0]), _cuda(g[0]), lo, hi, peak)
    assert out.dtype == torch.float64 and out.is_cuda and out.shape == (5,)
    row = out.cpu().numpy()
    assert np.isnan(row[2])
    mul = IO.image_errors(g, p, lo, hi, peak, c_square="mul")
    check_image_row(row, FX[f"{name}_row"], ssim_mul=mul[3])


@pytest.mark.parametrize("shape", [(128, 2048), (66, 1030), (65, 1029), (7, 7), (7, 8)])
@pytest.mark.parametrize("ties", [False, True])
def test_image_metrics_random_against_oracle(shape, ties):
    """Random frames, with and without heavy ties at the median (values on a coarse grid), odd and even n."""
    from lidar4d_b200.metrics import image_metrics
    g = np.random.default_rng(shape[0] * 7 + shape[1] + ties)
    gt = g.uniform(-5, 90, shape)
    pred = gt + g.normal(0, 3, shape)
    if ties:
        gt, pred = np.round(gt / 4) * 4, np.round(pred / 4) * 4
    gt, pred = gt.astype(np.float32), pred.astype(np.float32)
    row = image_metrics(_cuda(pred), _cuda(gt), *IO.DEPTH).cpu().numpy()
    ref = IO.depth_errors(gt, pred)
    mul = IO.depth_errors(gt, pred, c_square="mul")
    check_image_row(row, ref, ssim_mul=mul[3])


def _raydrop_cases():
    return [(n, r) for n, rs in IC.RAYDROP_CASES.items() for r in rs]


@pytest.mark.parametrize("name,ratio", _raydrop_cases())
def test_raydrop_metrics_match_reference(name, ratio):
    from lidar4d_b200.metrics import raydrop_metrics
    _, p, g = IC.frame(FX, name)
    row = raydrop_metrics(_cuda(p), _cuda(g), ratio).cpu().numpy()
    ref = FX[f"{name}_r{ratio:g}_row"]
    assert _near(row[0], ref[0], rel=4e-6)
    assert _same(row[1], ref[1]) and _same(row[2], ref[2]), (row, ref)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("ratio", [0.5, 0.3, 0.7001])
def test_raydrop_low_precision_preds(dtype, ratio):
    from lidar4d_b200.metrics import raydrop_metrics
    _, p, g = IC.frame(FX, "raydrop")
    pl = _cuda(p).to(dtype)
    row = raydrop_metrics(pl, _cuda(g), ratio).cpu().numpy()
    if dtype == torch.float16:
        ref = IO.raydrop_errors(pl.cpu().numpy(), g, ratio)            # NumPy float16: ratio rounded to float16
    else:
        r16 = float(torch.tensor(ratio, dtype=torch.float64).to(torch.bfloat16))
        ref = IO.raydrop_errors(pl.float().cpu().numpy(), g, r16)
    assert _near(row[0], ref[0], rel=4e-6)
    assert _same(row[1], ref[1]) and _same(row[2], ref[2]), (row, ref)


def test_repeat_calls_are_bit_identical_and_launch_counts():
    from lidar4d_b200.metrics import image_metrics, raydrop_metrics
    lib = _lib()
    _, p, g = IC.frame(FX, "depth_a")
    P, G = _cuda(p[0]), _cuda(g[0])
    first = image_metrics(P, G, *IO.DEPTH).clone()
    torch.cuda.synchronize()
    n0 = lib.l4d_launch_count()
    for _ in range(5):
        again = image_metrics(P, G, *IO.DEPTH)
        assert torch.equal(again.view(torch.int64), first.view(torch.int64))
    assert lib.l4d_launch_count() - n0 == 5 * 4
    _, rp, rg = IC.frame(FX, "raydrop")
    a = raydrop_metrics(_cuda(rp), _cuda(rg), 0.5).clone()
    n0 = lib.l4d_launch_count()
    b = raydrop_metrics(_cuda(rp), _cuda(rg), 0.5)
    assert lib.l4d_launch_count() - n0 == 1
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))


def test_meters_stay_on_device_and_read_back_once():
    from lidar4d_b200.metrics import DepthMeter, IntensityMeter, RaydropMeter
    dm, im, rm = DepthMeter(scale=1.0), IntensityMeter(scale=1.0), RaydropMeter(ratio=0.5)
    frames = {n: IC.frame(FX, n) for n in IC.IMAGE_CASES}
    cuda = {n: (_cuda(p), _cuda(g)) for n, (_, p, g) in frames.items()}
    _, rp, rg = IC.frame(FX, "raydrop")
    rp, rg = _cuda(rp), _cuda(rg)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for n, (kind, _, _) in frames.items():
            (dm if kind == "depth" else im).update(*cuda[n])
        rm.update(rp, rg)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for m, kind in ((dm, "depth"), (im, "intensity")):
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                res = m.measure()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert sum("synchroniz" in str(x.message) for x in w) == 1
        ref = FX[f"measure_{kind}"]
        assert res.dtype == np.float64 and res.shape == (5,)
        for k in (0, 4):
            assert _near(res[k], ref[k], rel=4e-6, abs_=2e-5)
        assert _same(res[1], ref[1]) or _near(res[1], ref[1], rel=1e-15)
        assert _near(res[3], ref[3], abs_=2e-7)
        assert np.isnan(res[2])
    r = rm.measure()
    ref = FX["raydrop_r0.5_row"]
    assert _near(r[0], ref[0], rel=4e-6) and _same(r[1], ref[1]) and _same(r[2], ref[2])
    assert "Depth_error" in dm.report() and "Rdrop_error" in rm.report()
    dm.clear()
    assert dm.N == 0 and dm.V == []


def test_lpips_fn_receives_clamped_device_images():
    from lidar4d_b200.metrics import DepthMeter, IntensityMeter
    seen = []

    def fake_lpips(pred, gt, normalize=False):
        seen.append((pred.clone(), gt.clone(), normalize))
        return (pred - gt).abs().mean().reshape(1, 1, 1, 1)          # a tensor, as lpips.LPIPS returns

    _, p, g = IC.frame(FX, "depth_a")
    m = DepthMeter(scale=1.0, lpips_fn=fake_lpips)
    m.update(_cuda(p), _cuda(g))
    (sp, sg, norm), = seen
    assert norm is True and sp.is_cuda and sp.shape == (66, 1030) and sp.dtype == torch.float32
    lo, hi, _ = IO.DEPTH
    rp, rg = p[0].copy(), g[0].copy()
    for a in (rp, rg):
        a[a < lo] = lo
        a[a > hi] = hi
    assert np.array_equal(sp.cpu().numpy(), rp) and np.array_equal(sg.cpu().numpy(), rg)
    row = m.V[0].cpu().numpy()
    assert row[2] == float((sp - sg).abs().mean())
    check_image_row(row, FX["depth_a_row"])
    seen.clear()
    _, p, g = IC.frame(FX, "intensity_a")
    mi = IntensityMeter(scale=1.0, lpips_fn=lambda a, b, normalize=False: 0.25)
    mi.update(_cuda(p), _cuda(g))
    assert mi.measure()[2] == 0.25


def test_input_errors_launch_nothing():
    from lidar4d_b200.metrics import DepthMeter, RaydropMeter, image_metrics, raydrop_metrics
    lib = _lib()
    x = torch.rand(1, 16, 40, device=DEV)
    n0 = lib.l4d_launch_count()
    dm = DepthMeter(scale=1.0)
    with pytest.raises(ValueError):
        dm.update(torch.rand(2, 16, 40, device=DEV), torch.rand(2, 16, 40, device=DEV))     # B != 1
    with pytest.raises(ValueError):
        dm.update(torch.rand(1, 6, 40, device=DEV), torch.rand(1, 6, 40, device=DEV))       # H < 7
    with pytest.raises(ValueError):
        dm.update(x.cpu(), x.cpu())                                                         # host tensors
    with pytest.raises(ValueError):
        dm.update(x, torch.rand(1, 16, 41, device=DEV))
    with pytest.raises(ValueError):
        dm.update(torch.rand(1, 1, 16, 40, device=DEV), torch.rand(1, 1, 16, 40, device=DEV))
    with pytest.raises(TypeError):
        dm.update(x.double(), x.double())
    with pytest.raises(TypeError):
        dm.update(x.half(), x)
    with pytest.raises(TypeError):
        dm.update(x[0].cpu().numpy(), x[0])
    with pytest.raises(ValueError):
        image_metrics(x, x, *IO.DEPTH)                                                      # not [H, W]
    with pytest.raises(ValueError):
        image_metrics(x[0, :, :6], x[0, :, :6], *IO.DEPTH)
    rm = RaydropMeter()
    with pytest.raises(TypeError):
        rm.update(torch.ones(10, device=DEV, dtype=torch.int32), torch.ones(10, device=DEV))
    with pytest.raises(TypeError):
        rm.update(torch.ones(10, device=DEV), torch.ones(10, device=DEV, dtype=torch.float16))
    with pytest.raises(ValueError):
        rm.update(torch.ones(10, device=DEV), torch.ones(11, device=DEV))
    with pytest.raises(ValueError):
        rm.update(torch.ones(10), torch.ones(10))
    with pytest.raises(ValueError):
        raydrop_metrics(torch.ones(0, device=DEV), torch.ones(0, device=DEV))
    assert dm.N == 0 and rm.N == 0
    # the C-ABI's own checks
    V = C.c_void_p
    buf = torch.empty(lib.l4d_image_metrics_work_bytes(16, 40), dtype=torch.uint8, device=DEV)
    out = torch.empty(5, dtype=torch.float64, device=DEV)
    p, w, o = V(x.data_ptr()), V(buf.data_ptr()), V(out.data_ptr())
    st = V(torch.cuda.current_stream().cuda_stream)
    EINVAL, ESIZE = -1, -3
    assert lib.l4d_image_metrics(None, p, 16, 40, 1e-6, 80.0, 6400.0, o, w, buf.numel(), st) == EINVAL
    assert lib.l4d_image_metrics(p, p, 16, 40, 1e-6, 80.0, 6400.0, None, w, buf.numel(), st) == EINVAL
    assert lib.l4d_image_metrics(p, p, 16, 40, 1e-6, 80.0, 6400.0, o, None, buf.numel(), st) == EINVAL
    assert lib.l4d_image_metrics(p, p, 6, 40, 1e-6, 80.0, 6400.0, o, w, buf.numel(), st) == EINVAL
    assert lib.l4d_image_metrics(p, p, 16, 6, 1e-6, 80.0, 6400.0, o, w, buf.numel(), st) == EINVAL
    assert lib.l4d_image_metrics(p, p, 1 << 16, 1 << 15, 1e-6, 80.0, 6400.0, o, w, buf.numel(), st) == EINVAL
    assert lib.l4d_image_metrics(p, p, 16, 40, 1e-6, 80.0, 6400.0, o, V(buf.data_ptr() + 4), buf.numel() - 4, st) == EINVAL
    assert lib.l4d_image_metrics(p, p, 16, 40, 1e-6, 80.0, 6400.0, o, w, buf.numel() - 1, st) == ESIZE
    assert b"work buffer too small" in lib.l4d_last_error()
    assert lib.l4d_raydrop_metrics(None, p, 10, 0.5, o, st) == EINVAL
    assert lib.l4d_raydrop_metrics(p, p, 10, 0.5, None, st) == EINVAL
    assert lib.l4d_raydrop_metrics(p, p, 0, 0.5, o, st) == EINVAL
    assert lib.l4d_launch_count() == n0


def test_trainer_mirror_evaluation_end_to_end():
    """Trainer.evaluate_one_epoch's meter calls (model/runner.py:591-602) after the mirror's eval_step on the small test
    model, through the four drop-in meters, against the oracle meters on host copies of the same tensors."""
    import sys
    from trainer_mirror import MirrorTrainer, default_opt, synthetic_batch
    from parity_util import small_config, cuda_model_from_oracle
    from oracle import lidar4d_oracle as O
    from lidar4d_b200.chamfer import chamfer_3DDist
    from lidar4d_b200.metrics import RaydropMeter, IntensityMeter, DepthMeter, PointsMeter
    assert "skimage" not in sys.modules and "lpips" not in sys.modules
    dev = torch.device(DEV)
    orc = O.build_seeded(small_config(), 5, flow_last_std=0.02)
    model = cuda_model_from_oracle(orc)
    opt = default_opt(num_frames=6, num_steps=48, near_lidar=0.0105, far_lidar=0.851, fp16=False)
    _, ev, pcs, ground = synthetic_batch(64, frame=2, num_frames=6, seed=1, device=dev, H=16, W=64)
    tr = MirrorTrainer(opt, model, chamfer_3DDist(), pc_list=pcs, pc_ground_list=ground, device=dev)
    metrics = [RaydropMeter(ratio=0.5), IntensityMeter(scale=1.0), DepthMeter(scale=opt.scale)]
    assert PointsMeter.__module__ == "lidar4d_b200.metrics"           # the fourth meter of the same import line
    oracles = [IO.RaydropMeter(ratio=0.5), IO.IntensityMeter(scale=1.0), IO.DepthMeter(scale=opt.scale)]
    oracles_mul = [None, IO.IntensityMeter(scale=1.0, c_square="mul"), IO.DepthMeter(scale=opt.scale, c_square="mul")]
    for frame_seed in range(2):
        with torch.no_grad():
            pi, pd, pr, gi, gd, gr, _ = tr.eval_step(ev)
        preds_mask = torch.where(pr > 0.5, 1, 0)
        args = [(pr, gr), (pi * preds_mask, gi), (pd * preds_mask, gd)]
        for i, m in enumerate(metrics):
            m.update(*args[i])
        for i, m in enumerate(oracles):
            m.update(*args[i])
            if oracles_mul[i] is not None:
                oracles_mul[i].update(*args[i])
        ev["time"] = ev["time"] * 0.5                     # a second, different frame
    r, ref = metrics[0].measure(), oracles[0].measure()
    assert _near(r[0], ref[0], rel=4e-6) and _same(r[1], ref[1]) and _same(r[2], ref[2]), (r, ref)
    for i in (1, 2):
        row, ref, mul = metrics[i].measure(), oracles[i].measure(), oracles_mul[i].measure()
        assert np.isnan(row[2])
        assert _near(row[1], ref[1], rel=1e-15), ("medae", row, ref)
        assert _near(row[0], ref[0], rel=4e-6) and _near(row[4], ref[4], abs_=2e-5), (row, ref)
        assert _near(row[3], ref[3], abs_=2e-7) and _near(row[3], mul[3], abs_=1e-12), (row, ref, mul)
