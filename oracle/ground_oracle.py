"""NumPy restatement of the flow loss's point-cloud preparation (the reference's utils/misc.py point_removal with Open3D's
statistical outlier removal), stage by stage, for the tests of lidar4d_b200.misc.

Every stage also reports the points whose decision lies within a few ulps of its threshold (`*_near`): there a
different but equally valid evaluation order (BLAS, a parallel reduction) may decide the other way, so the GPU tests
accept a differing decision on exactly those points.

Open3D's PointCloud::RemoveStatisticalOutliers(nb_neighbors, std_ratio), from its public source [open3d-ext]:
  * k = min(nb_neighbors, n) nearest points of each point, the point itself included; squared distances in nanoflann's
    L2_Adaptor order ((dx*dx) + dy*dy) + dz*dz;
  * avg_i = (sum of sqrt(d2) over those neighbours, ascending, from 0.0) / k;
  * n_valid counts the points whose search returned neighbours: all n;
  * mean = (sum over avg_i > 0, in index order, from 0.0) / n_valid;
    std = sqrt((sum over avg_i > 0 of (avg_i - mean) * (avg_i - mean), in index order) / (n_valid - 1));
  * keep i iff avg_i > 0 and avg_i < mean + std_ratio * std, in index order.
Neighbour identity comes from scipy's cKDTree; the distances are then recomputed in the order above, so the oracle
does not depend on the tree's own arithmetic (two neighbours at equal distance give the same sum whichever is kept)."""
import random

import numpy as np
from scipy.spatial import cKDTree

NEAR_ULPS = 4


def _near(values, thr, ulps=NEAR_ULPS):
    thr = np.asarray(thr, np.float64)
    return np.abs(np.asarray(values, np.float64) - thr) <= ulps * np.spacing(np.abs(thr))


# --- range filter ---------------------------------------------------------------------------------------------------
def range_filter_mask(pc, dist_min=1, dist_max=50, z_limit=(-2.5, 4)):
    """misc.py:116-125 on float32 points [N, >=3] -> (keep mask, near mask).  float32 throughout: the array square is
    x*x and the row sum runs left to right."""
    p = np.asarray(pc, np.float32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    d = np.sqrt((x * x + y * y) + z * z)
    ego = (x > -2) & (x < 2) & (y > -1) & (y < 1) & (z > -2) & (z < 2)
    keep = (d >= np.float32(dist_min)) & (d <= np.float32(dist_max)) & (z > np.float32(z_limit[0])) & (z < np.float32(z_limit[1])) & ~ego
    near = np.zeros(len(p), bool)
    for v, t in ((d, dist_min), (d, dist_max), (z, z_limit[0]), (z, z_limit[1])):
        t32 = np.float32(t)
        near |= np.abs(v.astype(np.float64) - np.float64(t32)) <= NEAR_ULPS * np.float64(np.spacing(np.abs(t32)))
    return keep, near


# --- statistical outlier removal ------------------------------------------------------------------------------------
def knn_mean_dist(points, k=64):
    """avg_i of Open3D's rule for float64 points [n, 3]."""
    p = np.ascontiguousarray(points, np.float64)
    n = len(p)
    kk = min(k, n)
    _, idx = cKDTree(p).query(p, k=kk)
    idx = idx.reshape(n, kk)
    d = p[idx] - p[:, None, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    d2.sort(axis=1)
    s = np.zeros(n)
    for j in range(kk):                                  # sequential, ascending
        s = s + np.sqrt(d2[:, j])
    return s / kk


def outlier_stats(avg, std_ratio=3.0):
    """-> (threshold, mean, std) in Open3D's sequential order."""
    n = len(avg)
    pos = [float(a) for a in avg if a > 0]
    s = 0.0
    for a in pos:
        s += a
    mean = s / n
    q = 0.0
    for a in pos:
        q += (a - mean) * (a - mean)
    std = float(np.sqrt(q / (n - 1))) if n > 1 else float("nan")
    return mean + std_ratio * std, mean, std


def statistical_outlier_removal(points, nb_neighbors=64, std_ratio=3.0):
    """-> (kept indices, near mask, avg, threshold).  An empty cloud stays empty."""
    if len(points) == 0:
        return np.zeros(0, np.int64), np.zeros(0, bool), np.zeros(0), float("nan")
    avg = knn_mean_dist(points, nb_neighbors)
    thr = outlier_stats(avg, std_ratio)[0]
    keep = (avg > 0) & (avg < thr)
    return np.flatnonzero(keep), _near(avg, thr), avg, thr


# --- RANSAC ---------------------------------------------------------------------------------------------------------
def estimate_plane(xyz):
    """misc.py:18-57 with normalize=False, on a float64 [3, 3] array: NumPy float64 scalar arithmetic."""
    u = xyz[1, :] - xyz[0, :]
    v = xyz[2, :] - xyz[0, :]
    if not np.all(u):
        return None
    q = v / u
    if q[0] == q[1] and q[2] == q[1]:
        return None
    a = (u[1] * v[2]) - (u[2] * v[1])
    b = (u[2] * v[0]) - (u[0] * v[2])
    c = (u[0] * v[1]) - (u[1] * v[0])
    d = -(a * xyz[0, 0] + b * xyz[0, 1] + c * xyz[0, 2])
    return np.array([a, b, c, d])


def plane_distances(points, coeffs, r):
    """|((a x + b y) + c z) + d| / r, every operation rounded on its own."""
    p = np.asarray(points, np.float64)
    a, b, c, d = (np.float64(v) for v in coeffs)
    return np.abs(((a * p[:, 0] + b * p[:, 1]) + c * p[:, 2]) + d) / np.float64(r)


def my_ransac(data, distance_threshold=0.3, P=0.99, sample_size=3, max_iterations=1000):
    """misc.py:60-113 on the global `random`: -> (inlier indices of the best hypothesis, its coefficients, per-hypothesis
    counts, per-hypothesis near counts)."""
    L = len(data)
    best, best_count, i, K = None, -999, 0, 10
    counts, nears = [], []
    population = range(L)
    while i < K:
        s = random.sample(population, sample_size)
        if abs(data[s[0], 1] - data[s[1], 1]) < 3:
            continue
        co = estimate_plane(data[s, :])
        if co is None:
            continue
        r = np.sqrt(co[0] ** 2 + co[1] ** 2 + co[2] ** 2)
        dist = plane_distances(data, co[:3].tolist() + [co[3]], r)
        inl = dist < distance_threshold
        cnt = np.int64(inl.sum())
        counts.append(int(cnt))
        nears.append(int(_near(dist, distance_threshold).sum()))
        if cnt > best_count:
            best_count, best = cnt, (co, inl)
            w = cnt / L
            K = np.log(1 - P) / np.log(1.0 - np.power(w, 3))
        i += 1
        if i > max_iterations:
            break
    return np.flatnonzero(best[1]), best[0], counts, nears


# --- the whole of point_removal -------------------------------------------------------------------------------------
def point_removal(pc_raw, n_ransac=6, ground_z=-1):
    """misc.py:128-154 on float32 points -> dict of every stage's indices, decisions and near-threshold flags.  Consumes
    the global `random` exactly as the reference does."""
    pc_raw = np.asarray(pc_raw, np.float32)
    out = {}
    keep, near = range_filter_mask(pc_raw)
    out["rf_keep"], out["rf_near"] = np.flatnonzero(keep), np.flatnonzero(near)
    pc = pc_raw[keep][:, :3].astype(np.float64)
    ind, near, avg, thr = statistical_outlier_removal(pc)
    out["sor1_keep"], out["sor1_near"], out["sor1_avg"], out["sor1_thr"] = ind, np.flatnonzero(near), avg, thr
    pc = pc[ind]
    union = np.zeros(len(pc), bool)
    out["ransac_counts"], out["ransac_near"] = [], []
    for _ in range(n_ransac):
        inl, _, counts, nears = my_ransac(pc, distance_threshold=0.15)
        union[inl] = True
        out["ransac_counts"].append(counts)
        out["ransac_near"].append(nears)
    ground = union & (pc[:, 2] < ground_z)
    out["ground"] = np.flatnonzero(ground)
    rest = pc[~ground]
    ind, near, avg, thr = statistical_outlier_removal(rest)
    out["sor2_keep"], out["sor2_near"], out["sor2_avg"], out["sor2_thr"] = ind, np.flatnonzero(near), avg, thr
    out["points"], out["ground_points"] = rest[ind], pc[ground]
    return out
