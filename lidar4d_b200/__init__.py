"""lidar4d_b200 - H100-native (sm_90a) implementation of the LiDAR4D per-ray
volume-rendering hot path behind the reference's LiDAR4D nn.Module API.

`from lidar4d_b200 import LiDAR4D` gives the drop-in module; it loads
csrc/liblidar4d_b200.so through the C-ABI in include/lidar4d_b200.h and raises
if the library or a CUDA device is missing (there is no CPU fallback).
"""
from .geometry import FieldConfig, make_frame  # noqa: F401


_CONVERT = ("lidar_to_pano_with_intensities", "lidar_to_pano", "pano_to_lidar_with_intensities", "pano_to_lidar")


def __getattr__(name):
    if name in ("LiDAR4D", "LiDAR_Renderer"):
        from . import model
        return getattr(model, name)
    if name in _CONVERT:
        from . import convert
        return getattr(convert, name)
    if name in ("point_metrics", "PointsMeter", "image_metrics", "raydrop_metrics", "DepthMeter", "IntensityMeter",
                "RaydropMeter"):
        from . import metrics
        return getattr(metrics, name)
    raise AttributeError(name)
