"""Frames for tests/golden/image_metrics_ref.npz, rebuilt from seeds instead of stored (the fixture holds results, not
images).  Test infrastructure, used by tests/golden/make_image_metrics_golden.py and by the tests that read its outputs.

Depth frames are 66 x 1030 range images in metres, ray-cast with ground_cases' scene (a ground plane, two walls, box
"cars") along the sensor model's directions: ray drops are zeros, ranges past 80 m are kept (the meters clamp them),
and the prediction is a noisy copy multiplied by its own drop mask, as Trainer.evaluate_one_epoch passes it.  Values
are quantised to 1/256 m (intensities to 1/4096) in float64 before the cast, so the frames do not depend on the
platform's transcendental functions; the fixture stores the SHA-256 of every rebuilt frame and `frame` refuses one
that does not match."""
import hashlib

import numpy as np

import ground_cases as GC


def _q(v, step):
    return (np.round(np.asarray(v, np.float64) / step) * step).astype(np.float32)


def _depth_pair(seed, H, W):
    rng = np.random.default_rng(seed)
    t = GC.ranges(GC.directions(H, W), rng).reshape(H, W)
    t = np.where(np.isfinite(t) & (t < 120.0), t, 0.0)                       # no return: 0 (ray drop)
    gt = _q(t, 1 / 256)
    noise = rng.uniform(-0.4, 0.4, (H, W)) * (1 + t / 20)
    keep = rng.random((H, W)) > 0.08                                         # the prediction's own drop mask
    pred = _q(np.where(keep, np.maximum(t + noise, 0.0), 0.0), 1 / 256)
    return pred, gt


def _intensity_pair(seed, H, W):
    rng = np.random.default_rng(seed)
    gt = _q(rng.uniform(-0.1, 1.2, (H, W)), 1 / 4096)
    pred = _q(np.asarray(gt, np.float64) + rng.uniform(-0.15, 0.15, (H, W)), 1 / 4096)
    pred[rng.random((H, W)) < 0.05] = 0.0
    return pred, gt


def _build(name):
    """-> (kind, pred [1, H, W] float32, gt [1, H, W] float32) for an image case, or ("raydrop", pred, gt)."""
    if name == "depth_a":
        p, g = _depth_pair(201, 66, 1030)
    elif name == "depth_b":
        p, g = _depth_pair(202, 66, 1030)
    elif name.startswith("depth_"):                                          # depth_<H>x<W>
        H, W = (int(v) for v in name[6:].split("x"))
        p, g = _depth_pair(203 + H + W, H, W)
    elif name == "intensity_a":
        p, g = _intensity_pair(301, 66, 1030)
    elif name == "intensity_8x9":
        p, g = _intensity_pair(302, 8, 9)
    elif name == "const_gt":                                                 # R = 0
        p, g = _depth_pair(401, 16, 40)
        g[:] = np.float32(12.5)
    elif name == "identical":                                                # mse 0: PSNR inf
        p, g = _depth_pair(402, 16, 40)
        p = g.copy()
    elif name == "nan_pixel":
        p, g = _depth_pair(403, 16, 40)
        p[5, 17] = np.nan
    elif name.startswith("raydrop"):
        rng = np.random.default_rng(500 + len(name))
        g = (rng.random((66, 1030)) > 0.2).astype(np.float32)
        p = _q(np.clip(0.75 * g + rng.uniform(-0.4, 0.45, g.shape), 0, 1), 1 / 1024)
        p[rng.random(g.shape) < 0.05] = np.float32(0.5)                      # exact ratio values
        if name == "raydrop_all_dropped":
            p[:] = 0.0                                                       # no predicted return: F1 NaN
        return "raydrop", p[None], g[None]
    else:
        raise KeyError(name)
    kind = "intensity" if name.startswith("intensity") else "depth"
    return kind, np.asarray(p, np.float32)[None], np.asarray(g, np.float32)[None]


IMAGE_CASES = ["depth_a", "depth_b", "depth_7x7", "depth_7x1030", "depth_8x9", "depth_65x1029", "intensity_a",
               "intensity_8x9", "const_gt", "identical", "nan_pixel"]
RAYDROP_CASES = {"raydrop": (0.5, 0.3), "raydrop_all_dropped": (0.5,)}      # case -> the ratios it is measured at


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def frame(f, name):
    """(kind, pred, gt) of case `name`, checked against the SHA-256 stored in fixture f (an opened npz), if given."""
    kind, p, g = _build(name)
    if f is not None and digest(p, g) != str(f[f"{name}_sha256"]):
        raise RuntimeError(f"the rebuilt {name} frames differ from the ones the reference outputs were computed on")
    return kind, p, g
