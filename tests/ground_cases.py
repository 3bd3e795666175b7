"""Synthetic KITTI-like LiDAR sweeps for tests/golden/ground_ref.npz, rebuilt from seeds instead of stored (a 66 x 1030
sweep's float32 coordinates would be 0.8 MB each).  Test infrastructure, used by tests/golden/make_ground_golden.py and by
the tests that read its outputs.

The scene, ray-cast in float64 along the sensor model's directions (rays.lidar_rays, fov_up 2, fov 26.9): a ground plane
near z = -1.73 m with a tilt and 2 cm noise, two long walls, box "cars", hits inside the ego box, sparse outliers,
misses (no return), ranges far beyond 50 m, and clusters of exact duplicates (some of more than 64 points, whose mean
neighbour distance is 0).  Coordinates are quantised to a 1/256 m grid in float64, so the float32 cloud does not depend
on the platform's transcendental functions; the fixture stores the SHA-256 of every rebuilt cloud and `cloud` refuses
one that does not match."""
import hashlib

import numpy as np

K = (2.0, 26.9)


def _q(v):
    return (np.round(np.asarray(v, np.float64) * 256.0) / 256.0).astype(np.float32)


def directions(H, W):
    i, j = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64), indexing="xy")
    az = (-(i - W / 2) / W * 2 * np.pi).reshape(-1)
    el = ((K[0] - j / H * K[1]) / 180 * np.pi).reshape(-1)
    return np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1)


def _boxes(rng, m):
    c = np.stack([rng.uniform(-35, 35, m), rng.uniform(-7, 7, m), np.full(m, -1.73)], 1)
    c = c[(np.abs(c[:, 0]) > 5) | (np.abs(c[:, 1]) > 3)]
    half = np.stack([rng.uniform(1.8, 2.4, len(c)), rng.uniform(0.8, 1.0, len(c)), rng.uniform(0.7, 0.9, len(c))], 1)
    lo, hi = c - half, c + half
    lo[:, 2] = -1.73
    hi[:, 2] = -1.73 + 2 * half[:, 2]
    return lo, hi


def ranges(d, rng, tilt=(0.004, -0.006)):
    """Ray-cast ranges along unit directions d [N, 3] (inf = no return)."""
    n = len(d)
    t = np.full(n, np.inf)
    gz = -1.73
    denom = d[:, 2] - tilt[0] * d[:, 0] - tilt[1] * d[:, 1]        # z = gz + tx x + ty y
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = np.where(denom < -1e-9, gz / denom, np.inf)
        t = np.minimum(t, tg)
        for y0 in (9.0, -11.0):                                      # walls y = y0, |x| < 45, z < 5
            tw = y0 / d[:, 1]
            ok = (tw > 0) & (np.abs(tw * d[:, 0]) < 45) & (tw * d[:, 2] < 5)
            t = np.where(ok & (tw < t), tw, t)
        lo, hi = _boxes(rng, 24)
        for a, b in zip(lo, hi):                                     # slab test
            t1, t2 = (a[None] - 0) / d, (b[None] - 0) / d
            tmin = np.max(np.minimum(t1, t2), 1)
            tmax = np.min(np.maximum(t1, t2), 1)
            ok = (tmax >= tmin) & (tmin > 0)
            t = np.where(ok & (tmin < t), tmin, t)
    t = t + rng.normal(0, 0.02, n)
    return t


def sweep(seed, H=66, W=1030, tilt=(0.004, -0.006)):
    """-> float32 [M, 3]: one sensor sweep (returns only), with ego-box hits, outliers, far points and duplicates."""
    rng = np.random.default_rng(seed)
    d = directions(H, W)
    t = ranges(d, rng, tilt)
    n = len(t)
    ego = rng.choice(n, 300, replace=False)
    t[ego] = rng.uniform(0.3, 1.6, 300)                              # inside |x| < 2, |y| < 1, |z| < 2 mostly
    out = rng.choice(n, 400, replace=False)
    t[out] = rng.uniform(1, 50, 400)                                 # sparse outliers
    far = rng.choice(n, 300, replace=False)
    t[far] = rng.uniform(50, 200, 300)
    miss = rng.random(n) < 0.03
    t[miss] = np.inf
    keep = np.isfinite(t) & (t < 250)
    pts = _q(d[keep] * t[keep, None])
    for size in (70, 90, 12, 5):                                     # exact duplicate clusters
        src = rng.integers(0, len(pts))
        at = np.sort(rng.integers(0, len(pts), size))
        pts = np.insert(pts, at, pts[src], axis=0)
    return pts


def digest(points):
    return hashlib.sha256(np.ascontiguousarray(points, np.float32).tobytes()).hexdigest()


SWEEPS = {"sweep_a": (11, (0.004, -0.006)), "sweep_b": (12, (-0.01, 0.008))}


def cloud(f, name):
    """The sweep `name` of fixture f (an opened ground_ref.npz), checked against its stored SHA-256."""
    seed, tilt = SWEEPS[name]
    pts = sweep(seed, tilt=tilt)
    if digest(pts) != str(f[f"{name}_sha256"]):
        raise RuntimeError(f"the rebuilt {name} cloud differs from the one the reference outputs were computed on")
    return pts


def small_clouds(rng):
    """Edge clouds, stored in the fixture: 70 and 200 points with a ground plane spanning more than 3 m in y, and one
    with a 66-point duplicate cluster."""
    out = {}
    for name, n in (("small70", 70), ("small200", 200)):
        g = np.stack([rng.uniform(-20, 20, n), rng.uniform(-15, 15, n), -1.7 + rng.normal(0, 0.03, n)], 1)
        k = n // 4
        g[:k, 2] = rng.uniform(-1.0, 3.0, k)
        out[name] = _q(g)
    dup = np.stack([rng.uniform(-20, 20, 150), rng.uniform(-15, 15, 150), -1.7 + rng.normal(0, 0.03, 150)], 1)
    dup = _q(dup)
    dup = np.insert(dup, 40, np.repeat(dup[7:8], 65, 0), axis=0)
    out["dup"] = dup
    return out


def pack(indices, n):
    """Sorted indices into a cloud of n points -> uint8 [8 + ceil(n / 8)]: n as 8 little-endian bytes, then the bit mask."""
    m = np.zeros(n, bool)
    m[np.asarray(indices, np.int64)] = True
    return np.concatenate([np.frombuffer(np.int64(n).tobytes(), np.uint8), np.packbits(m)])


def unpack(bits):
    n = int(np.frombuffer(bits[:8].tobytes(), np.int64)[0])
    return np.flatnonzero(np.unpackbits(bits[8:], count=n))
