"""NumPy restatement of the reference's sweep outputs: the per-frame image and point-cloud code of Simulator.render
(model/simulator.py:124-171), Trainer.test_step + Trainer.test (model/runner.py:462-469, 755-793) and the validation
panel of Trainer.evaluate_one_epoch (:611-634), written as the same NumPy expressions on the same dtypes, with cv2's
colour maps as lookup tables and its GRAY2BGR as a repeat.  torch's `x * torch.where(r > 0.5, 1, 0)` (float32 times
int64 gives float32) is `x * m.astype(float32)`.  The clouds use oracle/convert_oracle.unproject, the reference's
pano_to_lidar_with_intensities.

r is the ray drop in its own dtype (float32 or float16), intensity and depth are float32 [H, W]; luts are the
[256, 3] uint8 BGR tables of colormaps 1 (intensity) and 20 (depth)."""
import numpy as np

from . import convert_oracle


def _gray(u8):
    return np.repeat(u8[..., None], 3, axis=-1)


_QUIET = np.errstate(invalid="ignore", over="ignore")    # NaN / out-of-range casts are part of what is restated


@_QUIET
def sim(r, intensity, depth, scale, lidar_K, lut_i, lut_d):
    """-> (panel [3H, W, 3], pano = depth*m / scale, intensities = intensity*m, cloud [N, 4])."""
    m = np.where(r > 0.5, 1, 0).astype(np.float32)
    inten = intensity * m
    d = depth * m
    panel = np.concatenate([_gray((r * 255).astype(np.uint8)), lut_i[(inten * 255).astype(np.uint8)],
                            lut_d[(d * 255).astype(np.uint8)]], axis=0)
    pano = d / scale
    return panel, pano, inten, convert_oracle.unproject(pano, inten, lidar_K)


@_QUIET
def test(r, intensity, depth, scale, alpha_r, lidar_K, lut_i, lut_d):
    """-> (raydrop [H, W], intensity [H, W, 3], depth [H, W, 3], pano = depth' / scale, points [N, 3])."""
    if alpha_r > 0:
        m = np.where(r > 0.5, 1, 0).astype(np.float32)
        intensity = intensity * m
        depth = depth * m
    raydrop = (np.where(r > 0.5, 1.0, 0.0) * 255).astype(np.uint8)
    pano = depth / scale
    return (raydrop, lut_i[(intensity * 255).astype(np.uint8)], lut_d[(depth * 255).astype(np.uint8)], pano,
            convert_oracle.unproject(pano, None, lidar_K))


@_QUIET
def evaluate(r, intensity, depth, lut_i, lut_d):
    """-> the validation panel [6H, W, 3]; rows 5-6 are float32 * int64 mask, i.e. float64, as NumPy promotes them."""
    m = np.where(r > 0.5, 1, 0)
    return np.concatenate([_gray((r * 255).astype(np.uint8)), lut_i[(intensity * 255).astype(np.uint8)],
                           lut_d[(depth * 255).astype(np.uint8)], _gray((m * 255).astype(np.uint8)),
                           lut_i[(intensity * m * 255).astype(np.uint8)], lut_d[(depth * m * 255).astype(np.uint8)]],
                          axis=0)
