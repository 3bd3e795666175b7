"""The reference's evaluation meters (``utils/metrics.py``) on the GPU: the point-cloud metric (``fscore`` :13-27 and
``PointsMeter`` :229-279) and the depth, intensity and ray-drop meters (``DepthMeter`` :30-98, ``IntensityMeter``
:101-169, ``RaydropMeter`` :172-226).

The reference copies every frame to the host for every meter and reduces it there with NumPy, SciPy (through skimage's
SSIM) and, for the point metric, a round trip back to the device.  Here each meter's ``update`` stays on the device and
keeps its row there; ``measure()`` reads all rows back at once.  Unlike ``utils/metrics.py`` this module needs neither
lpips nor skimage.  LPIPS is the one column it does not compute: DepthMeter / IntensityMeter leave it NaN unless the
caller passes an ``lpips_fn``.
"""
import os

import numpy as np
import torch

from . import _capi
from .chamfer import chamfer_3DDist
from .convert import pano_to_lidar


def point_metrics(pred_pano, gt_pano, lidar_K, threshold=0.05):
    """Chamfer distance and F-score between the clouds of two range images, as PointsMeter.update computes them:
    pred_pano, gt_pano [H, W] CUDA -> (cd, fscore, precision, recall), 0-dim float32 device tensors, with
    dist1 / dist2 the SQUARED nearest-neighbour distances of the predicted / ground-truth points,
    cd = mean(dist1) + mean(dist2), precision = mean(dist1 < threshold), recall = mean(dist2 < threshold) and
    fscore = 2 p r / (p + r), or 0 where that is NaN.  The threshold applies to squared distances, as in the reference.
    Raises ValueError when either image has no point (the chamfer op is undefined on an empty cloud)."""
    pred = pano_to_lidar(pred_pano, lidar_K)
    gt = pano_to_lidar(gt_pano, lidar_K)
    with torch.no_grad():
        dist1, dist2, _, _ = chamfer_3DDist()(pred[None], gt[None])
    lib = _capi.load_library()
    dev = pred.device
    out = torch.empty(5, device=dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_point_metrics(dist1.data_ptr(), dist1.shape[1], dist2.data_ptr(), dist2.shape[1], float(threshold),
                                   out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(lib, rc, "l4d_point_metrics")
    return out[0], out[1], out[2], out[3]


class PointsMeter:
    """Drop-in for utils/metrics.py:229-279.  update(preds, truths) takes [B, H, W] range images (frame 0 is measured,
    as in the reference), divides them by `scale` on the device and keeps (CD, F-score) as device tensors; measure()
    reads all frames back at once and returns their mean, a float32 numpy array [CD, F-score]."""

    def __init__(self, scale, intrinsics):
        self.V = []
        self.N = 0
        self.scale = scale
        self.intrinsics = intrinsics

    def clear(self):
        self.V = []
        self.N = 0

    def update(self, preds, truths):
        preds = preds.detach() / self.scale
        truths = truths.detach() / self.scale
        cd, fscore, _, _ = point_metrics(preds[0], truths[0], self.intrinsics, threshold=0.05)   # monoSDF threshold
        self.V.append(torch.stack([cd, fscore]))
        self.N += 1

    def measure(self):
        assert self.N == len(self.V)
        return torch.stack(self.V).cpu().numpy().mean(0)

    def write(self, writer, global_step, prefix="", suffix=""):
        writer.add_scalar(os.path.join(prefix, "CD"), self.measure()[0], global_step)

    def report(self):
        return f"Point_error (CD, F-score) = {self.measure()}"


DEPTH_RANGE = (1e-6, 80.0, 80.0 ** 2)       # (lo, hi, peak) of compute_depth_errors (utils/metrics.py:64-86)
INTENSITY_RANGE = (1e-6, 1.0, 1.0 ** 2)     # ... of compute_intensity_errors (:135-157)


def _check_image_pair(pred, gt, who):
    for name, t in (("pred", pred), ("gt", gt)):
        if not torch.is_tensor(t):
            raise TypeError(f"{who}: {name} must be a torch tensor")
        if t.dtype != torch.float32:
            raise TypeError(f"{who}: {name} must be float32, got {t.dtype}")
        if not t.is_cuda:
            raise ValueError(f"{who}: {name} must be a CUDA tensor")
    if pred.shape != gt.shape:
        raise ValueError(f"{who}: pred {tuple(pred.shape)} and gt {tuple(gt.shape)} differ in shape")
    if pred.device != gt.device:
        raise ValueError(f"{who}: pred and gt are on different devices")


def _image_metrics(pred, gt, lo, hi, peak):
    """-> (out float64 [5], work uint8): see image_metrics; `work` holds the clamped images (clamped_images)."""
    _check_image_pair(pred, gt, "image_metrics")
    if pred.dim() != 2:
        raise ValueError(f"image_metrics: pred and gt must be [H, W], got {tuple(pred.shape)}")
    H, W = pred.shape
    if H < 7 or W < 7:
        raise ValueError(f"image_metrics: SSIM's 7 x 7 window exceeds the {H} x {W} image")
    if H * W >= 1 << 31:
        raise ValueError("image_metrics: H * W must be < 2^31")
    pred, gt = pred.detach().contiguous(), gt.detach().contiguous()
    lib = _capi.load_library()
    dev = pred.device
    work = torch.empty(lib.l4d_image_metrics_work_bytes(H, W), dtype=torch.uint8, device=dev)
    out = torch.empty(5, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_image_metrics(pred.data_ptr(), gt.data_ptr(), H, W, float(lo), float(hi), float(peak),
                                   out.data_ptr(), work.data_ptr(), work.numel(), torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(lib, rc, "l4d_image_metrics")
    return out, work


def clamped_images(work, H, W):
    """The clamped (pred, gt) [H, W] float32 views of an l4d_image_metrics work buffer: pred at byte offset 0 and gt at
    byte offset L4D_IM_GT_OFFSET(H, W) = H*W*4 rounded up to a multiple of 256."""
    off = (H * W * 4 + 255) // 256 * 256
    pred = work[:H * W * 4].view(torch.float32).view(H, W)
    gt = work[off:off + H * W * 4].view(torch.float32).view(H, W)
    return pred, gt


def image_metrics(pred, gt, lo, hi, peak):
    """compute_depth_errors / compute_intensity_errors (utils/metrics.py:64-86, :135-157) on the device.

    pred, gt: float32 CUDA [H, W], 7 <= H, W.  Both are clamped to [lo, hi] in float32 (NaN stays NaN); the result is a
    float64 CUDA tensor [5] = (rmse, medae, NaN, ssim, psnr), slot 2 being the reference's LPIPS.  medae is bit for bit
    np.median; ssim is skimage's structural_similarity(pred, gt, data_range=max(gt) - min(gt)) with its C1 / C2 squared
    as x*x where skimage calls powf; rmse and psnr differ from NumPy's only by the order of the float32 mean's sum.
    `peak` is the PSNR numerator: 80**2 for depth, 1.0 for intensity.  No host synchronisation."""
    return _image_metrics(pred, gt, lo, hi, peak)[0]


def _round_ratio(ratio, dtype):
    """`preds > ratio` as NumPy compares it: ratio rounded to the preds' dtype (bfloat16, which NumPy lacks, by torch)."""
    if dtype == torch.float32:
        return float(np.float32(ratio))
    if dtype == torch.float16:
        return float(np.float16(ratio))
    return float(torch.tensor(float(ratio), dtype=torch.float64).to(torch.bfloat16).item())


def raydrop_metrics(pred, gt, ratio=0.5):
    """RaydropMeter.update (utils/metrics.py:191-216) on the device: pred (float32, float16 or bfloat16) and gt
    (float32) CUDA tensors of one shape -> float64 CUDA tensor [3] = (rmse, acc, f1), with mask = pred > ratio (ratio
    rounded to pred's dtype, as NumPy does), acc = mean(mask == gt) and f1 = 2pr/(p+r) from the counts; f1 is NaN
    where the reference's is (no predicted or no true return).  pred is cast up to float32, which is exact."""
    if not torch.is_tensor(pred) or not torch.is_tensor(gt):
        raise TypeError("raydrop_metrics: pred and gt must be torch tensors")
    if pred.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise TypeError(f"raydrop_metrics: pred must be float32, float16 or bfloat16, got {pred.dtype}")
    if gt.dtype != torch.float32:
        raise TypeError(f"raydrop_metrics: gt must be float32, got {gt.dtype}")
    if not pred.is_cuda or not gt.is_cuda:
        raise ValueError("raydrop_metrics: pred and gt must be CUDA tensors")
    if pred.shape != gt.shape or pred.device != gt.device:
        raise ValueError(f"raydrop_metrics: pred {tuple(pred.shape)} and gt {tuple(gt.shape)} differ in shape or device")
    n = pred.numel()
    if n == 0 or n >= 1 << 31:
        raise ValueError("raydrop_metrics: need 1 <= numel < 2^31")
    r = _round_ratio(ratio, pred.dtype)
    pred = pred.detach().reshape(-1).float().contiguous()
    gt = gt.detach().reshape(-1).contiguous()
    lib = _capi.load_library()
    dev = pred.device
    out = torch.empty(3, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_raydrop_metrics(pred.data_ptr(), gt.data_ptr(), n, r, out.data_ptr(),
                                     torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(lib, rc, "l4d_raydrop_metrics")
    return out


class _ImageMeter:
    lo = hi = peak = None

    def __init__(self, scale, lpips_fn=None):
        self.V = []
        self.N = 0
        self.scale = scale
        self.lpips_fn = lpips_fn

    def clear(self):
        self.V = []
        self.N = 0

    def update(self, preds, truths):
        _check_image_pair(preds, truths, type(self).__name__)
        if preds.dim() == 3:
            if preds.shape[0] != 1:
                raise ValueError(f"{type(self).__name__}: one frame at a time ([1, H, W] or [H, W]), got "
                                 f"{tuple(preds.shape)}")
        elif preds.dim() != 2:
            raise ValueError(f"{type(self).__name__}: expected [1, H, W] or [H, W], got {tuple(preds.shape)}")
        H, W = preds.shape[-2:]
        if H < 7 or W < 7:
            raise ValueError(f"{type(self).__name__}: SSIM's 7 x 7 window exceeds the {H} x {W} image")
        preds = preds.detach() / self.scale        # the reference's own torch division, so the same bits
        truths = truths.detach() / self.scale
        row, work = _image_metrics(preds.reshape(H, W), truths.reshape(H, W), self.lo, self.hi, self.peak)
        if self.lpips_fn is not None:
            p, g = clamped_images(work, H, W)
            v = self.lpips_fn(p, g, normalize=True)
            row[2] = v.detach().reshape(()) if torch.is_tensor(v) else float(v)
        self.V.append(row)
        self.N += 1

    def measure(self):
        assert self.N == len(self.V)
        return torch.stack(self.V).cpu().numpy().mean(0)


class DepthMeter(_ImageMeter):
    """Drop-in for utils/metrics.py:30-98: update(preds, truths) takes one float32 CUDA depth frame [1, H, W] or [H, W],
    divides it by `scale` on the device (the reference's torch op) and keeps the row (rmse, medae, lpips, ssim, psnr)
    as a float64 device tensor (see image_metrics, clamp range [1e-6, 80], PSNR peak 80**2); measure() reads every row
    back at once and returns their float64 mean.

    LPIPS differs on purpose: the reference ignores its `lpips_fn` argument and always builds AlexNet LPIPS (a weights
    download).  Here the slot is NaN unless `lpips_fn` is given; then it is called as the reference calls its own,
    lpips_fn(pred, gt, normalize=True), on the clamped [H, W] CUDA images, and its value fills slot 2."""
    lo, hi, peak = DEPTH_RANGE

    def write(self, writer, global_step, prefix="", suffix=""):
        writer.add_scalar(os.path.join(prefix, f"depth error{suffix}"), self.measure()[0], global_step)

    def report(self):
        return f"Depth_error = {self.measure()}"


class IntensityMeter(_ImageMeter):
    """Drop-in for utils/metrics.py:101-169: DepthMeter's contract with the clamp range [1e-6, 1] and PSNR peak 1.0."""
    lo, hi, peak = INTENSITY_RANGE

    def write(self, writer, global_step, prefix="", suffix=""):
        writer.add_scalar(os.path.join(prefix, f"intensity error{suffix}"), self.measure()[0], global_step)

    def report(self):
        return f"Inten_error = {self.measure()}"


class RaydropMeter:
    """Drop-in for utils/metrics.py:172-226: update(preds, truths) takes ray-drop probabilities (float32, float16 or
    bfloat16) and the float32 ground-truth mask, of any one shape, as CUDA tensors and keeps the row (rmse, acc, f1) as a
    float64 device tensor (see raydrop_metrics); measure() reads every row back at once and returns their float64 mean."""

    def __init__(self, ratio=0.5):
        self.V = []
        self.N = 0
        self.ratio = ratio

    def clear(self):
        self.V = []
        self.N = 0

    def update(self, preds, truths):
        self.V.append(raydrop_metrics(preds, truths, self.ratio))
        self.N += 1

    def measure(self):
        assert self.N == len(self.V)
        return torch.stack(self.V).cpu().numpy().mean(0)

    def write(self, writer, global_step, prefix="", suffix=""):
        writer.add_scalar(os.path.join(prefix, "raydrop error"), self.measure()[0], global_step)

    def report(self):
        return f"Rdrop_error (RMSE, Acc, F1) = {self.measure()}"
