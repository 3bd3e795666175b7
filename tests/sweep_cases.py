"""Frames for tests/golden/sweep_ref.npz, rebuilt from seeds instead of stored.  Test infrastructure, used by
tests/golden/make_sweep_golden.py and by the tests that read its outputs.

A frame is what the render and the U-Net hand to the reference's image code: depth [H, W] and image [H, W, 2] (ray drop,
intensity) float32 and a refined ray drop [H, W] in float32 or float16.  The values are chosen where the 8-bit images
are decided: exactly k/255 and one ulp either side (as float32), ray drops at 0.5 and one ulp either side (in their own
dtype), depths past 256/255 (the cast wraps), negative values (-1 -> 255), and one NaN in each plane.  They are built
from integers and float64 -> float32 casts only, so they do not depend on the platform's maths library; the fixture
stores the SHA-256 of every rebuilt frame and `frames` refuses one that does not match."""
import hashlib

import numpy as np

# case -> (H, W, frames, dtype of the refined ray drop, seed)
CASES = {
    "66x1030": (66, 1030, 2, np.float32, 11),
    "32x1024": (32, 1024, 2, np.float32, 12),
    "8x16": (8, 16, 2, np.float32, 13),
    "66x1030_f16": (66, 1030, 1, np.float16, 14),
    "8x16_f16": (8, 16, 2, np.float16, 15),
}


def _near_k(rng, shape, dtype=np.float32):
    """k/255 for random k in 0..255, moved by -1, 0 or +1 ulp of `dtype`."""
    x = (rng.integers(0, 256, shape) / 255.0).astype(dtype)
    off = rng.integers(-1, 2, shape)
    return np.where(off > 0, np.nextafter(x, dtype(np.inf)), np.where(off < 0, np.nextafter(x, dtype(-np.inf)), x))


def _pick(rng, *options):
    sel = rng.integers(0, len(options), options[0].shape)
    out = options[0].copy()
    for k in range(1, len(options)):
        out[sel == k] = options[k][sel == k]
    return out


def _raydrop(rng, shape, dtype):
    half = dtype(0.5)
    at = np.full(shape, half)
    either = np.where(rng.random(shape) < 0.5, np.nextafter(at, dtype(0)), np.nextafter(at, dtype(1)))
    x = _pick(rng, rng.random(shape).astype(dtype), _near_k(rng, shape, dtype), at, either)
    x.flat[0] = dtype(np.nan)
    x.flat[1] = dtype(-1 / 255)
    return x


def _frame(rng, H, W, dtype):
    s = (H, W)
    inten = _pick(rng, _near_k(rng, s), rng.uniform(-0.05, 1.1, s).astype(np.float32))
    depth = _pick(rng, _near_k(rng, s), rng.uniform(0, 1.6, s).astype(np.float32),
                  rng.uniform(1.0, 300.0, s).astype(np.float32))
    inten.flat[2] = np.nan
    depth.flat[3] = np.nan
    depth.flat[4] = np.float32(-1 / 255)
    image = np.stack([_raydrop(rng, s, np.float32), inten], -1)
    return {"depth": depth, "image": image, "unet": _raydrop(rng, s, dtype)}


def _build(name):
    H, W, n, dtype, seed = CASES[name]
    rng = np.random.default_rng(seed)
    return [_frame(rng, H, W, dtype) for _ in range(n)]


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def frames_digest(fr):
    return digest(*[f[k] for f in fr for k in ("depth", "image", "unet")])


def frames(f, name):
    """The frames of case `name`, checked against the SHA-256 stored in fixture f (an opened npz), if given."""
    fr = _build(name)
    if f is not None and frames_digest(fr) != str(f[f"{name}_sha256"]):
        raise RuntimeError(f"the rebuilt {name} frames differ from the ones the reference outputs were computed on")
    return fr


def poses(n, seed):
    """n seeded lidar2world poses [n, 4, 4] float64 along a curving path (metres): the stand-in KITTI-360 poses."""
    rng = np.random.default_rng(seed)
    out = np.tile(np.eye(4), (n, 1, 1))
    yaw = 0.3 + 0.05 * np.arange(n) + rng.uniform(-0.01, 0.01, n)
    c, s = np.cos(yaw), np.sin(yaw)
    out[:, 0, 0], out[:, 0, 1], out[:, 1, 0], out[:, 1, 1] = c, -s, s, c
    out[:, :3, 3] = np.array([1385.2, 3870.4, 115.9]) + np.cumsum(rng.uniform(0.5, 1.5, (n, 3)) * [1, 0.6, 0.02], 0)
    return out


# what tests/golden/make_sweep_golden.py ran on each case
SCALE = 0.01
# case -> (refine, fov_lidar)
SIM = {"66x1030": (True, (2.0, 26.9)), "32x1024": (False, (10.0, 40.0)), "8x16": (True, (2.0, 26.9))}
# case -> (alpha_r, refine, write_video)
TEST = {"66x1030_f16": (0.01, True, False), "32x1024": (0.0, False, True), "8x16_f16": (0.01, True, False)}
EVAL = ("66x1030_f16", "8x16")


def same(fx, key, a):
    """True when array `a` is, byte for byte (shape and dtype included), what the fixture holds under `key`: the array
    itself for small cases, its SHA-256 for the others."""
    stored = fx[key]
    a = np.ascontiguousarray(a)
    if stored.dtype.kind == "U":
        return digest(a) == str(stored)
    return stored.shape == a.shape and stored.dtype == a.dtype and stored.tobytes() == a.tobytes()


def raydrop_of(frame, refine):
    return frame["unet"] if refine else frame["image"][..., 0]
