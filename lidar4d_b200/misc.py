"""The flow loss's point-cloud preparation on the GPU: the reference's ``utils/misc.py`` (``range_filter``,
``estimate_plane``, ``my_ransac``, ``point_removal``) without Open3D, and ``Trainer.process_pointcloud`` of
``model/runner.py`` as a function.  Backed by the ``l4d_range_filter`` / ``l4d_knn_mean_dist`` / ``l4d_outlier_select`` /
``l4d_plane_scores`` / ``l4d_plane_mask`` / ``l4d_ground_split`` / ``l4d_pose_transform`` entry points of the C-ABI.

Point clouds are CUDA tensors; results are CUDA tensors written on torch's current stream, float32 out of
``range_filter`` and float64 from the first outlier removal on, as Open3D yields.  Each compaction reads its row count
back to the host once (a synchronisation), as ``pano_to_lidar`` does.

RANSAC.  ``my_ransac`` draws its samples from the *global* ``random`` with exactly the reference's sequence of
``random.sample`` calls, so that ``random.getstate()`` afterwards equals the reference's.  The rejection tests and the
plane coefficients are the reference's NumPy scalar expressions on a float64 host copy of the cloud (they touch three
points each).  Hypotheses are drawn ahead in batches, with the RNG state kept after every accepted draw; one launch
scores a batch, the adaptive loop is replayed on the counts, and the state is restored to just after the last draw the
reference would have consumed.  Deliberate differences from the reference:
  * where every draw is rejected the reference loops forever; this raises ``RuntimeError`` after
    ``MAX_CONSECUTIVE_REJECTIONS`` rejected draws in a row;
  * fewer than ``sample_size`` points raise ``ValueError`` (``random.sample`` does too, but only after the reference's
    loop has started);
  * the point-to-plane distances are evaluated term by term, ((a x + b y) + c z) + d, where NumPy's ``matmul`` may use
    BLAS; a point can only be decided differently within a few ulps of the threshold.
"""
import random

import numpy as np
import torch

from . import _capi
from .convert import pano_to_lidar

RANSAC_BATCH = 256
MAX_CONSECUTIVE_REJECTIONS = 10 ** 6


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _cuda(x, name, dtype):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (lidar4d_b200.misc has no CPU path)")
    if x.dim() != 2 or x.shape[1] < 3:
        raise ValueError(f"{name}: expected [N, >=3], got {tuple(x.shape)}")
    return x.detach().to(dtype).contiguous()


def _xyz64(x, name):
    return _cuda(x, name, torch.float64)[:, :3].contiguous()


def _work(nbytes, dev):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def range_filter(pcd, dist_min=1, dist_max=50, z_limit=[-2.5, 4]):
    """misc.py:116-125.  pcd [N, C >= 3] -> the rows with dist_min <= |xyz| <= dist_max, z_limit[0] < z < z_limit[1],
    outside the ego box |x| < 2, |y| < 1, |z| < 2, in order; float32 arithmetic as NumPy's on a float32 cloud."""
    pts = _cuda(pcd, "pcd", torch.float32)
    n, stride = pts.shape
    out = torch.empty_like(pts)
    if n == 0:
        return out
    lib = _capi.load_library()
    dev = pts.device
    count = torch.empty(1, dtype=torch.int32, device=dev)
    nwork = lib.l4d_range_filter_work_bytes(n)
    work = _work(nwork, dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_range_filter(pts.data_ptr(), n, stride, float(dist_min), float(dist_max), float(z_limit[0]),
                                  float(z_limit[1]), out.data_ptr(), count.data_ptr(), work.data_ptr(), nwork, _stream(dev))
    _capi.check(lib, rc, "l4d_range_filter")
    return out[:int(count.item())]


def knn_mean_dist(points, k=64):
    """Mean distance from every point to its min(k, n) nearest points (itself included), float64, exact (k <= 64)."""
    pts = _xyz64(points, "points")
    lib = _capi.load_library()
    avg = torch.empty(len(pts), dtype=torch.float64, device=pts.device)
    with torch.cuda.device(pts.device):
        rc = lib.l4d_knn_mean_dist(pts.data_ptr(), len(pts), int(k), avg.data_ptr(), _stream(pts.device))
    _capi.check(lib, rc, "l4d_knn_mean_dist")
    return avg


def _select(pts, avg, std_ratio, stats=None):
    lib = _capi.load_library()
    n, dev = len(pts), pts.device
    out = torch.empty(n, 3, dtype=torch.float64, device=dev)
    ind = torch.empty(n, dtype=torch.int32, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    nwork = lib.l4d_outlier_select_work_bytes(n)
    work = _work(nwork, dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_outlier_select(pts.data_ptr(), n, avg.data_ptr(), float(std_ratio), out.data_ptr(), ind.data_ptr(),
                                    count.data_ptr(), stats.data_ptr() if stats is not None else None, work.data_ptr(),
                                    nwork, _stream(dev))
    _capi.check(lib, rc, "l4d_outlier_select")
    m = int(count.item())
    return out[:m], ind[:m].long()


def statistical_outlier_removal(points, nb_neighbors, std_ratio):
    """Open3D's ``PointCloud.remove_statistical_outlier(nb_neighbors, std_ratio)`` -> (points [M, 3] float64, ind [M]
    int64).  avg_i = mean distance to the min(nb_neighbors, n) nearest points (the point itself included); keep
    avg_i > 0 and avg_i < mean + std_ratio * std over the points with avg_i > 0, mean and std dividing by n and n - 1
    as Open3D does.  1 <= nb_neighbors <= 64."""
    pts = _xyz64(points, "points")
    if not 1 <= int(nb_neighbors) <= 64:
        raise ValueError("nb_neighbors must be in [1, 64]")
    if len(pts) == 0:
        return pts, torch.empty(0, dtype=torch.int64, device=pts.device)
    return _select(pts, knn_mean_dist(pts, nb_neighbors), std_ratio)


def estimate_plane(xyz, normalize=True):
    """misc.py:18-57.  xyz: 3 x 3 points (rows) -> np.array([a, b, c, d]), or None when p1 - p0 has a zero component or
    the two edge vectors are exactly proportional.  NumPy float64 scalar arithmetic on the host, as the reference."""
    if torch.is_tensor(xyz):
        xyz = xyz.detach().cpu().numpy()
    xyz = np.asarray(xyz, np.float64)
    e1, e2 = xyz[1, :] - xyz[0, :], xyz[2, :] - xyz[0, :]
    if not np.all(e1):
        return None
    ratio = e2 / e1
    if ratio[0] == ratio[1] and ratio[2] == ratio[1]:
        return None
    a = (e1[1] * e2[2]) - (e1[2] * e2[1])
    b = (e1[2] * e2[0]) - (e1[0] * e2[2])
    c = (e1[0] * e2[1]) - (e1[1] * e2[0])
    if normalize:
        norm = np.sqrt(a ** 2 + b ** 2 + c ** 2)
        a, b, c = a / norm, b / norm, c / norm
    d = -(a * xyz[0, 0] + b * xyz[0, 1] + c * xyz[0, 2])
    return np.array([a, b, c, d])


def ransac_drive(host, score, distance_threshold=0.3, P=0.99, sample_size=3, max_iterations=1000, batch=RANSAC_BATCH):
    """The host half of ``my_ransac``: host = float64 numpy [L, 3]; score(hyp) maps float64 [m, 5] hypotheses
    (a, b, c, d, r) to their m inlier counts.  -> (coefficients [4], r, per-hypothesis counts) of the reference's loop,
    leaving the global ``random`` where the reference leaves it."""
    L = len(host)
    if L < sample_size or sample_size < 3:
        raise ValueError(f"my_ransac needs sample_size >= 3 and at least sample_size points (got {L}, {sample_size})")
    population = range(L)
    best, best_count, i, K = None, -999, 0, 10
    counts_all = []
    rejected = 0
    while True:
        want = max_iterations + 1 - i
        if np.isfinite(K):
            want = min(want, max(int(np.ceil(K)) - i, 1))
        want = min(want, batch)
        hyps, coeffs, states = [], [], []
        exhausted = False
        while len(hyps) < want:
            s = random.sample(population, sample_size)
            co = None
            if not abs(host[s[0], 1] - host[s[1], 1]) < 3:
                co = estimate_plane(host[s, :], normalize=False)
            if co is None:
                rejected += 1
                if rejected >= MAX_CONSECUTIVE_REJECTIONS:
                    exhausted = True
                    break
                continue
            rejected = 0
            hyps.append((co[0], co[1], co[2], co[3], np.sqrt(co[0] ** 2 + co[1] ** 2 + co[2] ** 2)))
            coeffs.append(co)
            states.append(random.getstate())
        counts = [int(c) for c in score(np.array(hyps, np.float64).reshape(-1, 5))] if hyps else []
        for j, c in enumerate(counts):
            counts_all.append(c)
            near = np.int64(c)
            if near > best_count:
                best_count, best = near, (coeffs[j], hyps[j][4])
                w = near / L
                K = np.log(1 - P) / np.log(1.0 - np.power(w, 3))
            i += 1
            if i > max_iterations or not i < K:
                random.setstate(states[j])
                return best[0], best[1], counts_all
        if exhausted:
            raise RuntimeError(f"my_ransac: {MAX_CONSECUTIVE_REJECTIONS} draws in a row were rejected (no three points "
                               "span 3 m in y and a plane); the reference would loop forever")


def _plane_scorer(pts, distance_threshold):
    lib = _capi.load_library()
    dev = pts.device

    def score(hyp):
        h = torch.from_numpy(np.ascontiguousarray(hyp)).to(dev)
        counts = torch.empty(len(hyp), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            rc = lib.l4d_plane_scores(pts.data_ptr(), len(pts), h.data_ptr(), len(hyp), float(distance_threshold),
                                      counts.data_ptr(), _stream(dev))
        _capi.check(lib, rc, "l4d_plane_scores")
        return counts.cpu().numpy()
    return score


def _mark_plane(pts, coeffs, r, distance_threshold, mask):
    lib = _capi.load_library()
    with torch.cuda.device(pts.device):
        rc = lib.l4d_plane_mask(pts.data_ptr(), len(pts), *(float(v) for v in coeffs), float(r), float(distance_threshold),
                                mask.data_ptr(), _stream(pts.device))
    _capi.check(lib, rc, "l4d_plane_mask")


def _ransac_into(pts, host, mask, distance_threshold, P=0.99, sample_size=3, max_iterations=1000):
    coeffs, r, counts = ransac_drive(host, _plane_scorer(pts, distance_threshold), distance_threshold, P, sample_size,
                                     max_iterations)
    _mark_plane(pts, coeffs, r, distance_threshold, mask)
    return coeffs, counts


def my_ransac(data, distance_threshold=0.3, P=0.99, sample_size=3, max_iterations=1000):
    """misc.py:60-113.  data [L, >=3] -> (indices of the best plane's inliers, int64 CUDA tensor; its unnormalised
    coefficients [a, b, c, d] as a NumPy array).  See the module docstring for the RNG contract and the differences."""
    pts = _xyz64(data, "data")
    host = pts.cpu().numpy()
    mask = torch.zeros(len(pts), dtype=torch.uint8, device=pts.device)
    coeffs, _ = _ransac_into(pts, host, mask, distance_threshold, P, sample_size, max_iterations)
    return torch.nonzero(mask).view(-1), coeffs


def _split(pts, mask, z_max):
    lib = _capi.load_library()
    n, dev = len(pts), pts.device
    ground = torch.empty(n, 3, dtype=torch.float64, device=dev)
    rest = torch.empty(n, 3, dtype=torch.float64, device=dev)
    gi = torch.empty(n, dtype=torch.int32, device=dev)
    ri = torch.empty(n, dtype=torch.int32, device=dev)
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    nwork = lib.l4d_ground_split_work_bytes(n)
    work = _work(nwork, dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_ground_split(pts.data_ptr(), n, mask.data_ptr(), float(z_max), ground.data_ptr(), gi.data_ptr(),
                                  rest.data_ptr(), ri.data_ptr(), counts.data_ptr(), work.data_ptr(), nwork, _stream(dev))
    _capi.check(lib, rc, "l4d_ground_split")
    ng, nr = counts.cpu().tolist()
    return ground[:ng], gi[:ng].long(), rest[:nr], ri[:nr].long()


def point_removal_stages(pc_raw):
    """point_removal with every stage's kept indices: a dict with `points`, `ground` (as point_removal returns) and
    `rf_keep` (into pc_raw), `sor1_keep` (into the range-filtered cloud), `ransac_counts` (six lists), `ground_index`
    (into the cloud after the first outlier removal), `sor2_keep` (into the non-ground rest)."""
    pc = _cuda(pc_raw, "pc_raw", torch.float32)
    dev = pc.device
    out = {}
    # range filter with the row index carried along in a fourth column (exact in float32 below 2^24 rows; beyond that
    # the mask is recomputed from the kept rows instead)
    if len(pc) < (1 << 24):
        tagged = torch.cat([pc[:, :3], torch.arange(len(pc), device=dev, dtype=torch.float32)[:, None]], 1)
        kept = range_filter(tagged)
        out["rf_keep"], pts = kept[:, 3].long(), kept[:, :3].double().contiguous()
    else:
        pts = range_filter(pc[:, :3]).double().contiguous()
        out["rf_keep"] = None
    if len(pts) == 0:
        raise ValueError("point_removal: no point survives the range filter")
    pts, out["sor1_keep"] = statistical_outlier_removal(pts, 64, 3.0)
    if len(pts) == 0:
        raise ValueError("point_removal: no point survives the outlier removal")
    host = pts.cpu().numpy()
    mask = torch.zeros(len(pts), dtype=torch.uint8, device=dev)
    out["ransac_counts"] = [_ransac_into(pts, host, mask, 0.15)[1] for _ in range(6)]
    out["ground"], out["ground_index"], rest, _ = _split(pts, mask, -1.0)
    out["points"], out["sor2_keep"] = statistical_outlier_removal(rest, 64, 3.0)
    return out


def point_removal(pc_raw):
    """misc.py:128-154.  pc_raw [N, >=3] CUDA -> (points [M, 3], ground [G, 3]), float64 CUDA tensors: the range
    filter, Open3D's statistical outlier removal (64, 3.0), the union of six my_ransac(distance_threshold=0.15) inlier
    sets below z = -1 as the ground, and a second outlier removal of the rest.  Consumes the global ``random`` as the
    reference does.  A NumPy array (the reference Trainer's call, runner.py:938-941) is moved to the current CUDA
    device and the results come back as float64 NumPy arrays, as the reference returns them."""
    if isinstance(pc_raw, np.ndarray):
        st = point_removal_stages(torch.from_numpy(np.ascontiguousarray(pc_raw)).cuda())
        return st["points"].cpu().numpy(), st["ground"].cpu().numpy()
    st = point_removal_stages(pc_raw)
    return st["points"], st["ground"]


def _transform(pts, pose, scale):
    lib = _capi.load_library()
    out = torch.empty_like(pts)
    if len(pts) == 0:
        return out
    pose = np.ascontiguousarray(pose, np.float32).reshape(4, 4)
    with torch.cuda.device(pts.device):
        rc = lib.l4d_pose_transform(pts.data_ptr(), len(pts), float(scale), pose.ctypes.data, out.data_ptr(),
                                    _stream(pts.device))
    _capi.check(lib, rc, "l4d_pose_transform")
    return out


def pano_depth(images_lidar, scale):
    """runner.py:933-937: gt_depth = images[..., 2] * images[..., 0], divided by scale in the images' dtype as NumPy 2
    divides a float16 / float32 array by a Python float (the scalar is rounded to the array's dtype first)."""
    gt_depth = images_lidar[:, :, :, 2] * images_lidar[:, :, :, 0]
    s = torch.tensor(float(scale), dtype=gt_depth.dtype, device=gt_depth.device)
    return gt_depth.squeeze(0) / s


def process_pointcloud(loader, scale, num_frames, lidar_K):
    """Trainer.process_pointcloud (runner.py:924-951) -> (pc_list, pc_ground_list): for every batch of `loader`
    (dicts with images_lidar [1, H, W, C], poses_lidar [1, 4, 4], time [1, 1]), the frame's range image unprojected,
    point_removal, scaled back and moved by the pose; stored as float64 NumPy arrays [M, 3] under
    str(int(time * (num_frames - 1))), as the reference stores them.  The unprojection is lidar4d_b200.convert's, whose
    device cosf / sinf may differ from NumPy's float32 ones by an ulp; everything after it is the reference's
    arithmetic (see process_frame)."""
    pc_list, pc_ground_list = {}, {}
    for data in loader:
        images = data["images_lidar"]
        dev = images.device if images.is_cuda else torch.device("cuda", torch.cuda.current_device())
        pano = pano_depth(images.to(dev), scale)
        frame_idx = int(data["time"] * (num_frames - 1))
        pc_list[f"{frame_idx}"], pc_ground_list[f"{frame_idx}"] = process_frame(pano_to_lidar(pano, lidar_K),
                                                                                data["poses_lidar"], scale)
    return pc_list, pc_ground_list


def process_frame(pc_raw, pose, scale):
    """The part of process_pointcloud after the unprojection: point_removal, then both clouds scaled by `scale` and
    moved by the float32 4 x 4 pose -> (points, ground) as float64 NumPy arrays."""
    points, ground = point_removal(pc_raw)
    pose = pose.squeeze(0).detach().cpu().numpy() if torch.is_tensor(pose) else np.asarray(pose)
    return _transform(points, pose, scale).cpu().numpy(), _transform(ground, pose, scale).cpu().numpy()
