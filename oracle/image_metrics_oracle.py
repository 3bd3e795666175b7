"""NumPy restatement of the reference's image meters (utils/metrics.py: DepthMeter.compute_depth_errors :64-86,
IntensityMeter.compute_intensity_errors :135-157, RaydropMeter.update :191-216) without skimage or lpips.

[skimage-ext] `structural_similarity` is scikit-image's (>= 0.19) at the reference's arguments: a 2-D float32 image,
win_size 7, uniform filter, use_sample_covariance=True, K1 = 0.01, K2 = 0.03, data_range given.  Restated here over
scipy.ndimage.uniform_filter, operation for operation in skimage's float32 order.  `c_square` selects how the constants
C1 = (K1 R)^2 and C2 = (K2 R)^2 are squared: "powf" is what skimage runs (a NumPy float32 scalar power, libm powf),
"mul" is x * x, which is what the CUDA kernels compute.

`uniform_filter_rec` restates SciPy's uniform_filter(x, 7) on float32 as its C loop runs it: axis 0 first, stored as
float32, then axis 1; mode 'reflect'; along a line a double running sum t of the extended values, started as the
left-to-right sum of the first 7 and advanced by t = t + (x[i+3] - x[i-4]), each output f32(t / 7)."""
import numpy as np
from scipy.ndimage import uniform_filter

WIN = 7
DEPTH = (1e-6, 80.0, 80 ** 2)           # (lo, hi, peak) of compute_depth_errors
INTENSITY = (1e-6, 1.0, 1.0 ** 2)       # ... of compute_intensity_errors


def _lines_rec(x):
    """uniform_filter1d(x, 7, axis=0, mode='reflect') on float32 x [n, m] -> float32: the double recurrence along axis 0,
    run for all m lines at once (each step is the same elementwise IEEE double operation for every line)."""
    n = x.shape[0]
    r = WIN // 2
    ext = np.concatenate([x[:r][::-1], x, x[n - r:][::-1]]).astype(np.float64)
    out = np.empty(x.shape, np.float32)
    t = np.zeros(x.shape[1:], np.float64)
    for k in range(WIN):
        t = t + ext[k]
    out[0] = (t / 7.0).astype(np.float32)
    for i in range(1, n):
        t = t + (ext[i + WIN - 1] - ext[i - 1])
        out[i] = (t / 7.0).astype(np.float32)
    return out


def uniform_filter_rec(x):
    """scipy.ndimage.uniform_filter(x, 7) for a 2-D float32 array, restated (see the module docstring)."""
    x = np.asarray(x, np.float32)
    return _lines_rec(_lines_rec(x).T).T


def ssim_constants(R, c_square="powf"):
    """(C1, C2) as float32: R is the float32 data range."""
    R = np.float32(R)
    k1, k2 = np.float32(0.01) * R, np.float32(0.03) * R
    if c_square == "powf":
        return k1 ** 2, k2 ** 2                          # NumPy float32 scalar power: libm powf
    if c_square == "mul":
        return k1 * k1, k2 * k2
    raise ValueError(c_square)


def ssim_map(ux, uy, uxx, uyy, uxy, C1, C2):
    """skimage's S map from the five filtered float32 maps, in its float32 order (no fused multiply-add)."""
    c = np.float32(WIN * WIN / (WIN * WIN - 1))
    vx = c * (uxx - ux * ux)
    vy = c * (uyy - uy * uy)
    vxy = c * (uxy - ux * uy)
    A1, A2, B1, B2 = (2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2)
    D = B1 * B2
    return (A1 * A2) / D


def filtered_maps(pred, gt, filt=uniform_filter):
    x, y = np.asarray(pred, np.float32), np.asarray(gt, np.float32)
    return [filt(v, size=WIN) if filt is uniform_filter else filt(v) for v in (x, y, x * x, y * y, x * y)]


def structural_similarity(im1, im2, *, data_range, c_square="powf", filt=uniform_filter):
    """[skimage-ext] skimage.metrics.structural_similarity(im1, im2, data_range=data_range) for 2-D float32 images."""
    im1, im2 = np.asarray(im1), np.asarray(im2)
    if im1.shape != im2.shape:
        raise ValueError("Input images must have the same dimensions.")
    if im1.ndim != 2 or min(im1.shape) < WIN:
        raise ValueError("win_size exceeds image extent.")
    im1, im2 = im1.astype(np.float32, copy=False), im2.astype(np.float32, copy=False)
    with np.errstate(divide="ignore", invalid="ignore"):
        C1, C2 = ssim_constants(data_range, c_square)
        S = ssim_map(*filtered_maps(im1, im2, filt), C1, C2)
    pad = (WIN - 1) // 2
    return S[pad:-pad, pad:-pad].mean(dtype=np.float64)


def image_errors(gt, pred, lo, hi, peak, lpips_value=np.nan, c_square="powf"):
    """compute_depth_errors / compute_intensity_errors on float32 arrays [1, H, W] or [H, W]: the row
    (rmse, medae, lpips, ssim, psnr) as the reference returns it (float32 scalars, the lpips slot as given)."""
    gt, pred = np.array(gt, np.float32), np.array(pred, np.float32)
    pred[pred < lo] = lo
    pred[pred > hi] = hi
    gt[gt < lo] = lo
    gt[gt > hi] = hi
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        rmse = np.sqrt(((gt - pred) ** 2).mean())
        medae = np.median(np.abs(gt - pred))
        p2, g2 = pred.reshape(pred.shape[-2:]), gt.reshape(gt.shape[-2:])
        ssim = structural_similarity(p2, g2, data_range=np.max(gt) - np.min(gt), c_square=c_square)
        psnr = 10 * np.log10(peak / np.mean((pred - gt) ** 2))
    return rmse, medae, lpips_value, ssim, psnr


def depth_errors(gt, pred, **kw):
    return image_errors(gt, pred, *DEPTH, **kw)


def intensity_errors(gt, pred, **kw):
    return image_errors(gt, pred, *INTENSITY, **kw)


def raydrop_errors(preds, truths, ratio=0.5):
    """RaydropMeter.update's row (rmse, acc, f1) on NumPy arrays of any (equal) shape."""
    preds, truths = np.asarray(preds), np.asarray(truths)
    with np.errstate(divide="ignore", invalid="ignore"):
        rmse = np.sqrt(((truths - preds) ** 2).mean())
        preds_mask = np.where(preds > ratio, 1, 0)
        acc = (preds_mask == truths).mean()
        TP = np.sum((truths == 1) & (preds_mask == 1))
        FP = np.sum((truths == 0) & (preds_mask == 1))
        FN = np.sum((truths == 1) & (preds_mask == 0))
        precision = TP / (TP + FP)
        recall = TP / (TP + FN)
        f1 = 2 * (precision * recall) / (precision + recall)
    return rmse, acc, f1


class _ImageMeter:
    """The reference meters' host path (the .cpu() copies, then the restated NumPy), with LPIPS left as NaN."""
    lo = hi = peak = None

    def __init__(self, scale, c_square="powf"):
        self.V, self.N, self.scale, self.c_square = [], 0, scale, c_square

    def clear(self):
        self.V, self.N = [], 0

    def update(self, preds, truths):
        preds = (preds / self.scale).detach().cpu().numpy()
        truths = (truths / self.scale).detach().cpu().numpy()
        self.V.append(list(image_errors(truths, preds, self.lo, self.hi, self.peak, c_square=self.c_square)))
        self.N += 1

    def measure(self):
        return np.array(self.V).mean(0)


class DepthMeter(_ImageMeter):
    lo, hi, peak = DEPTH


class IntensityMeter(_ImageMeter):
    lo, hi, peak = INTENSITY


class RaydropMeter:
    def __init__(self, ratio=0.5):
        self.V, self.N, self.ratio = [], 0, ratio

    def clear(self):
        self.V, self.N = [], 0

    def update(self, preds, truths):
        self.V.append(list(raydrop_errors(preds.detach().cpu().numpy(), truths.detach().cpu().numpy(), self.ratio)))
        self.N += 1

    def measure(self):
        return np.array(self.V).mean(0)
