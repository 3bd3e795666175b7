"""Vectorised numpy restatement of the reference's ``utils/convert.py`` -- TEST INFRASTRUCTURE ONLY (imported by tests/
and scripts/convert_probe.py; the product never imports it).  Pinned bit for bit to the reference's own outputs in
tests/golden/convert_ref.npz (tests/golden/make_convert_golden.py) by tests/test_convert_oracle.py.

``project`` restates lidar_to_pano_with_intensities (convert.py:4-65).  The reference loops over NumPy float32 scalars,
so under NEP 50 every step is float32, with the Python-float constants rounded once to float32:
  dist  = np.linalg.norm(xyz)              = sqrt((x*x + y*y) + z*z)
  beta  = fl(pi) - arctan2(y, x)
  alpha = arctan2(z, sqrt(x**2 + y**2)) + fl(fov_down/180*pi),  fov_down = fov - fov_up in double
  c = round(beta / fl(2*pi/W)),  r = round(H - alpha / fl(fov/180*pi/H))     (half to even)
One scalar detail has no array equivalent: ``np.float32 ** 2`` is libm ``powf``, which is 1 ulp off ``x*x`` for some
inputs, while the array ``x**2`` takes NumPy's square fast path.  ``_spow2`` therefore applies the scalar operator
element by element.  The sequential z-buffer (``if pano == 0: set; elif pano > dist: set``) becomes: a zero-distance
point empties its pixel and keeps its own intensity; among the points after the last such point of a pixel the smallest
distance wins, the earliest on ties (np.maximum.at / np.minimum.at).

``unproject`` restates pano_to_lidar_with_intensities (convert.py:99-138), which is already array code.
"""
import numpy as np


def _spow2(v):
    """[x**2 for x in v] with NumPy float32 scalars (libm powf), as the reference's loop computes it."""
    return np.fromiter((s ** 2 for s in v), dtype=np.float32, count=v.shape[0])


def pre_round(points, lidar_H, lidar_W, lidar_K):
    """The float32 values the reference rounds, per point: (dist, c_pre, r_pre, atan2(y, x), atan2(z, rho))."""
    p = np.asarray(points, dtype=np.float32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    fov_up, fov = lidar_K
    fov_down = fov - fov_up
    with np.errstate(invalid="ignore", over="ignore"):
        dist = np.linalg.norm(p[:, :3], axis=1)
        a_xy = np.arctan2(y, x)
        beta = np.float32(np.pi) - a_xy
        a_z = np.arctan2(z, np.sqrt(_spow2(x) + _spow2(y)))
        alpha = a_z + np.float32(fov_down / 180 * np.pi)
        c_pre = beta / np.float32(2 * np.pi / lidar_W)
        r_pre = np.float32(lidar_H) - alpha / np.float32(fov / 180 * np.pi / lidar_H)
    return dist, c_pre, r_pre, a_xy, a_z


def project(points, lidar_H, lidar_W, lidar_K, max_depth=80, return_pixels=False):
    """points [N, 3 | 4] float32 -> (pano [H, W], intensities [H, W]) float32; with return_pixels also the flat pixel of
    every point (-1 = skipped).  Points at a NaN distance are skipped (the reference raises on them)."""
    p = np.asarray(points, dtype=np.float32)
    n = p.shape[0]
    inten = p[:, 3] if p.shape[1] > 3 else np.zeros(n, np.float32)
    dist, c_pre, r_pre, _, _ = pre_round(p, lidar_H, lidar_W, lidar_K)
    with np.errstate(invalid="ignore"):
        c = np.rint(c_pre).astype(np.float64)
        r = np.rint(r_pre).astype(np.float64)
        ok = (dist < np.float32(max_depth)) & (c >= 0) & (c < lidar_W) & (r >= 0) & (r < lidar_H)
    pix = np.full(n, -1, np.int64)
    pix[ok] = r[ok].astype(np.int64) * lidar_W + c[ok].astype(np.int64)
    pano, out_i = zbuffer(pix, dist, inten, lidar_H, lidar_W)
    return (pano, out_i, pix) if return_pixels else (pano, out_i)


def zbuffer(pix, dist, inten, lidar_H, lidar_W):
    """The reference's sequential z-buffer over points already placed on flat pixels (pix = -1: skipped)."""
    n = pix.shape[0]
    hw = lidar_H * lidar_W
    ok = pix >= 0
    idx = np.arange(n, dtype=np.int64)
    zero = ok & (dist == 0)
    zlast = np.full(hw, -1, np.int64)
    np.maximum.at(zlast, pix[zero], idx[zero])
    cand = ok & (dist > 0)
    cand[cand] = idx[cand] > zlast[pix[cand]]
    best = np.full(hw, np.inf, np.float64)
    np.minimum.at(best, pix[cand], dist[cand].astype(np.float64))
    win_pts = cand.copy()
    win_pts[cand] = dist[cand].astype(np.float64) == best[pix[cand]]
    winner = np.full(hw, n, np.int64)
    np.minimum.at(winner, pix[win_pts], idx[win_pts])
    pano = np.zeros(hw, np.float32)
    out_i = np.zeros(hw, np.float32)
    hit = winner < n
    pano[hit] = dist[winner[hit]]
    out_i[hit] = inten[winner[hit]]
    reset = ~hit & (zlast >= 0)
    out_i[reset] = inten[zlast[reset]]
    return pano.reshape(lidar_H, lidar_W), out_i.reshape(lidar_H, lidar_W)


def unproject(pano, intensities, lidar_K):
    """pano [H, W], intensities [H, W] (or None) float32 -> [N, 4] (or [N, 3]) float32 rows of the pixels with
    pano != 0, in row-major order."""
    fov_up, fov = lidar_K
    pano = np.asarray(pano, dtype=np.float32)
    H, W = pano.shape
    i, j = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing="xy")
    beta = -(i - W / 2) / W * 2 * np.pi
    alpha = (fov_up - j / H * fov) / 180 * np.pi
    dirs = np.stack([np.cos(alpha) * np.cos(beta), np.cos(alpha) * np.sin(beta), np.sin(alpha)], -1)
    pts = dirs * pano.reshape(H, W, 1)
    if intensities is not None:
        pts = np.concatenate([pts, np.asarray(intensities, np.float32).reshape(H, W, 1)], axis=2)
    return pts[np.where(pano != 0.0)]
