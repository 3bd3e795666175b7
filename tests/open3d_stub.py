"""Test infrastructure: the few Open3D names the reference's utils/misc.py uses (geometry.PointCloud with
remove_statistical_outlier, utility.Vector3dVector), with the outlier rule of oracle/ground_oracle.py, so that the
reference's own point_removal runs without Open3D.  `calls` records the kept indices of every
remove_statistical_outlier call."""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import ground_oracle as GO  # noqa: E402

calls = []


def Vector3dVector(a):
    return np.array(a, dtype=np.float64).reshape(-1, 3)


class PointCloud:
    def __init__(self):
        self.points = np.zeros((0, 3))

    def remove_statistical_outlier(self, nb_neighbors, std_ratio):
        pts = np.asarray(self.points, np.float64)
        if len(pts) == 0:
            ind = np.zeros(0, np.int64)
        else:
            ind = GO.statistical_outlier_removal(pts, nb_neighbors, std_ratio)[0]
        calls.append(ind)
        out = PointCloud()
        out.points = Vector3dVector(pts[ind])
        return out, [int(i) for i in ind]


def install():
    o3d = types.ModuleType("open3d")
    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud)
    o3d.utility = types.SimpleNamespace(Vector3dVector=Vector3dVector)
    sys.modules["open3d"] = o3d
    return o3d
