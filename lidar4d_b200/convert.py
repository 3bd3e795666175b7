"""Range image <-> point cloud conversions of the reference's ``utils/convert.py`` on the GPU, same names and argument
order, backed by ``l4d_pano_project`` / ``l4d_pano_unproject`` of the C-ABI library.

Inputs are CUDA tensors; outputs are CUDA float32 tensors written on torch's current stream.  There is no CPU path:
host inputs raise.  lidar_K = (fov_up, fov) in degrees.  Differences from the reference:
  * the reference returns float64 range images filled with float32 values; these are float32 with the same values;
  * points are read as float32 (the reference's float32 path, the one its callers take);
  * a point at a NaN distance is skipped (the reference raises on it inside ``round``);
  * ``lidar_to_pano`` works: the reference's passes ``max_dpeth=`` to a function whose parameter is ``max_depth`` and
    raises ``TypeError`` on every call.
"""
import torch

from . import _capi


def _device_tensor(x, name):
    if not torch.is_tensor(x) or not x.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (lidar4d_b200.convert has no CPU path)")
    return x.detach().contiguous().float()


def _project(points, H, W, lidar_K, max_depth, with_intensities):
    lib = _capi.load_library()
    dev = points.device
    fov_up, fov = float(lidar_K[0]), float(lidar_K[1])
    H, W = int(H), int(W)
    n, stride = points.shape[0], points.shape[1]
    pano = torch.empty(H, W, device=dev)
    inten = torch.empty(H, W, device=dev) if with_intensities else None
    nwork = lib.l4d_pano_project_work_bytes(H, W)
    work = torch.empty(max(nwork, 1), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_pano_project(points.data_ptr() if n else None, n, stride, fov_up, fov, H, W, float(max_depth),
                                  pano.data_ptr(), inten.data_ptr() if inten is not None else None, work.data_ptr(), nwork,
                                  torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(lib, rc, "l4d_pano_project")
    return pano, inten


def lidar_to_pano_with_intensities(local_points_with_intensities, lidar_H, lidar_W, lidar_K, max_depth=80):
    """convert.py:4-65.  local_points_with_intensities [N, 4] (x, y, z, intensity) in the lidar frame ->
    (pano [H, W], intensities [H, W]): per pixel the nearest distance below max_depth (0 = empty) and its intensity."""
    pts = _device_tensor(local_points_with_intensities, "local_points_with_intensities")
    if pts.dim() != 2 or pts.shape[1] != 4:
        raise ValueError(f"local_points_with_intensities: expected [N, 4], got {tuple(pts.shape)}")
    return _project(pts, lidar_H, lidar_W, lidar_K, max_depth, True)


def lidar_to_pano(local_points, lidar_H, lidar_W, lidar_K, max_depth=80):
    """convert.py:68-96.  local_points [N, 3] -> pano [H, W].  The reference's version raises TypeError on every call
    (it passes ``max_dpeth=`` on); this one returns the range image its docstring describes."""
    pts = _device_tensor(local_points, "local_points")
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"local_points: expected [N, 3], got {tuple(pts.shape)}")
    return _project(pts, lidar_H, lidar_W, lidar_K, max_depth, False)[0]


def _unproject(pano, intensities, lidar_K):
    out, count = _unproject_device(pano, intensities, lidar_K)
    # the one device-to-host read: the exact row count (<= H*W < 2^31) is needed to size the result, and it
    # synchronises with the stream
    return out[:int(count.item())]


def _unproject_device(pano, intensities, lidar_K):
    """-> (out [H*W, 3 or 4], count [1] int32), both on the device: the first count rows are the cloud.  No host read."""
    lib = _capi.load_library()
    if pano.dim() != 2:
        raise ValueError(f"pano: expected [H, W], got {tuple(pano.shape)}")
    H, W = pano.shape
    dev = pano.device
    fov_up, fov = float(lidar_K[0]), float(lidar_K[1])
    out = torch.empty(H * W, 3 if intensities is None else 4, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    nwork = lib.l4d_pano_unproject_work_bytes(H, W)
    work = torch.empty(max(nwork, 1), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = lib.l4d_pano_unproject(pano.data_ptr(), intensities.data_ptr() if intensities is not None else None, H, W,
                                    fov_up, fov, out.data_ptr(), count.data_ptr(), work.data_ptr(), nwork,
                                    torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(lib, rc, "l4d_pano_unproject")
    return out, count


def pano_to_lidar_with_intensities(pano, intensities, lidar_K):
    """convert.py:99-138.  pano [H, W], intensities [H, W] -> [N, 4]: one row (x, y, z, intensity) per pixel with
    pano != 0 (NaN included), in row-major pixel order.  Reads the row count back to the host once (a synchronisation);
    the result is a view of an [H*W, 4] buffer."""
    pano = _device_tensor(pano, "pano")
    intensities = _device_tensor(intensities, "intensities")
    if intensities.shape != pano.shape:
        raise ValueError(f"intensities {tuple(intensities.shape)} and pano {tuple(pano.shape)} differ in shape")
    return _unproject(pano, intensities, lidar_K)


def pano_to_lidar(pano, lidar_K):
    """convert.py:141-155.  pano [H, W] -> points [N, 3] (as pano_to_lidar_with_intensities, without the intensity
    column; one 4-byte device-to-host read)."""
    return _unproject(_device_tensor(pano, "pano"), None, lidar_K)
