"""The 123,708-point `mixed` cloud of tests/golden/convert_ref.npz, rebuilt from its seed instead of stored (its float32
coordinates alone would be 1.5 MB).  Test infrastructure, used by tests/golden/make_convert_golden.py (which stores the
reference's outputs on it) and by the tests that read those outputs.

Everything drawn from the seed is computed in float64 and quantised to a 1/256 m grid, so the float32 coordinates
do not depend on the platform's float32 transcendental functions; a float64 rounding difference could only matter at an
exact grid midpoint.  The fixture stores the SHA-256 of the rebuilt cloud, and `mixed_cloud` refuses a cloud that does
not match it.  The few points built bit by bit - zero-distance points with underflowing coordinates, and points within 2
ulps of a .5 rounding boundary - come from the fixture itself (`special`)."""
import hashlib

import numpy as np

H, W, K = 66, 1030, (2.0, 26.9)
SEED = 2024
SPECIAL = ("z0", "z1", "z2", "halves")


def _q(v):
    return (np.round(np.asarray(v, np.float64) * 256.0) / 256.0).astype(np.float32)


def _points(rng, az, el, r):
    xyz = np.stack([np.cos(el) * np.cos(az) * r, np.cos(el) * np.sin(az) * r, np.sin(el) * r], 1)
    inten = (rng.integers(0, 256, len(r)) / 256).astype(np.float32)
    return np.concatenate([_q(xyz), inten[:, None]], 1)


def sweep_directions():
    """(azimuth, elevation) of every pixel of the sensor model (rays.lidar_rays), row-major, in float64."""
    i, j = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64), indexing="xy")
    return (-(i - W / 2) / W * 2 * np.pi).reshape(-1), ((K[0] - j / H * K[1]) / 180 * np.pi).reshape(-1)


def digest(points):
    return hashlib.sha256(np.ascontiguousarray(points, np.float32).tobytes()).hexdigest()


def build(special, seed=SEED):
    """-> (cloud [N, 4] float32, slice of the sweep within it).  special: the SPECIAL float32 arrays.
    Layout: zero-distance group z0, a full 66 x 1030 sensor sweep with ranges in [1, 90], zero-distance group z1, then
    in seeded random order: jittered directions (many pixels hit several times), exact duplicates of sweep and jitter
    points with other intensities (ties: the earlier point wins), points above fov_up / below fov_down / far past
    max_depth, points with x < 0 and y <= 0 just below the -x axis (beta just under 2 pi: c == W, dropped, or W - 1),
    the near-.5 points; finally zero-distance group z2."""
    rng = np.random.default_rng(seed)
    az, el = sweep_directions()
    sweep = _points(rng, az, el, rng.uniform(1, 90, H * W))
    nj = 45000
    jit = _points(rng, rng.uniform(-np.pi, np.pi, nj) + rng.uniform(-0.6, 0.6, nj) * 2 * np.pi / W,
                  np.deg2rad(rng.uniform(K[0] - K[1], K[0], nj)), rng.uniform(1, 90, nj))
    dup = sweep[rng.integers(0, H * W, 6000)].copy()
    dup[:, 3] = (rng.integers(0, 256, 6000) / 256).astype(np.float32)
    dup_j = jit[rng.integers(0, nj, 2000)].copy()
    dup_j[:, 3] = (rng.integers(0, 256, 2000) / 256).astype(np.float32)
    nf = 2000
    above = rng.random(nf) < 0.5
    elf = np.deg2rad(np.where(above, rng.uniform(K[0] + 0.6, 40, nf), rng.uniform(-60, K[0] - K[1] - 0.6, nf)))
    rf = np.where(rng.random(nf) < 0.8, rng.uniform(1, 50, nf), rng.uniform(80, 1000, nf))
    fov_out = _points(rng, rng.uniform(-np.pi, np.pi, nf), elf, rf)
    nw = 600
    xw = -rng.uniform(2, 40, nw)
    yw = xw * rng.uniform(0, 0.006, nw)                 # <= 0; below 1/512 in size it quantises to -0.0 (atan2 = -pi)
    zw = -xw * np.tan(np.deg2rad(rng.uniform(-20, 0, nw)))
    cw = np.concatenate([_q(np.stack([xw, yw, zw], 1)), (rng.integers(0, 256, (nw, 1)) / 256).astype(np.float32)], 1)
    rest = np.concatenate([jit, dup, fov_out, cw, np.asarray(special["halves"], np.float32), dup_j])
    rest = rest[rng.permutation(len(rest))]
    z0, z1, z2 = (np.asarray(special[k], np.float32) for k in ("z0", "z1", "z2"))
    cloud = np.concatenate([z0, sweep, z1, rest, z2])
    return cloud, slice(len(z0), len(z0) + H * W)


def mixed_cloud(f):
    """The mixed cloud of fixture f (an opened convert_ref.npz) and the slice of its sweep, checked against the stored
    SHA-256."""
    cloud, sweep = build({k: f[f"mixed_{k}"] for k in SPECIAL}, int(f["mixed_seed"]))
    if digest(cloud) != str(f["mixed_sha256"]):
        raise RuntimeError("the rebuilt mixed cloud differs from the one the reference outputs were computed on")
    return cloud, sweep


# The range images of the mixed and sweep cases are stored losslessly but compactly: a depth is the float32 distance
# np.linalg.norm(xyz) of one of the cloud's points, so the image is stored as that point's index relative to the pixel's
# own sweep point (mostly 0), and the intensities, all multiples of 1/256 below 1, as bytes.  The generator checks
# that decoding gives back the reference's arrays bit for bit.
EMPTY = np.int32(-(1 << 31))


def encode_pano(pano, points, base):
    flat = np.asarray(pano, np.float32).reshape(-1)
    dist = np.linalg.norm(points[:, :3], axis=1)
    order = np.argsort(dist, kind="stable")
    nz = np.flatnonzero(flat != 0)
    idx = order[np.minimum(np.searchsorted(dist[order], flat[nz]), len(order) - 1)]
    if not np.array_equal(dist[idx], flat[nz]):
        raise ValueError("a depth of the range image is no point's distance")
    code = np.full(flat.size, EMPTY, np.int32)
    code[nz] = idx - (base + nz)
    return code


def decode_pano(code, points, base, shape):
    dist = np.linalg.norm(points[:, :3], axis=1)
    pano = np.zeros(code.size, np.float32)
    nz = np.flatnonzero(code != EMPTY)
    pano[nz] = dist[code[nz].astype(np.int64) + base + nz]
    return pano.reshape(shape)


def encode_intensities(inten):
    k = np.round(np.asarray(inten, np.float64) * 256)
    if not (np.array_equal(decode_intensities(k.astype(np.uint8)), inten) and k.max() <= 255):
        raise ValueError("intensities are not multiples of 1/256 in [0, 1)")
    return k.astype(np.uint8)


def decode_intensities(k):
    return k.astype(np.float32) / np.float32(256)
