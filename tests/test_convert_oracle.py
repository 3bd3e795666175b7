"""CPU: oracle/convert_oracle.py reproduces the reference's utils/convert.py bit for bit on every case of
tests/golden/convert_ref.npz (written by tests/golden/make_convert_golden.py from the reference's own functions), and
the reference's lidar_to_pano really cannot be called (the reason lidar4d_b200.convert.lidar_to_pano differs from it)."""
import os
import sys

import numpy as np
import pytest

import convert_cases
from oracle import convert_oracle as CO

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "convert_ref.npz")
REF = os.environ.get("LIDAR4D_REFERENCE", "/root/reference")


def load_case(f, name):
    """(points, H, W, lidar_K, pano, intensities) of one projection case of the fixture."""
    h, w = (int(v) for v in f[f"{name}_hw"])
    k = tuple(float(v) for v in f[f"{name}_K"])
    if name in ("mixed", "sweep"):
        cloud, sweep = convert_cases.mixed_cloud(f)
        pts, base = (cloud, sweep.start) if name == "mixed" else (cloud[sweep], 0)
        pano = convert_cases.decode_pano(f[f"{name}_pano_code"], pts, base, (h, w))
        return pts, h, w, k, pano, convert_cases.decode_intensities(f[f"{name}_intensities_u8"])
    return f[f"{name}_points"], h, w, k, f[f"{name}_pano"], f[f"{name}_intensities"]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", ["mixed", "sweep", "half", "pixel"])
def test_oracle_projection_equals_reference_fixture(name):
    f = np.load(GOLDEN)
    pts, h, w, k, pano, inten = load_case(f, name)
    p, i = CO.project(pts, h, w, k, 80)
    assert np.array_equal(bits(p), bits(pano))
    assert np.array_equal(bits(i), bits(inten))
    if name == "mixed":
        assert len(pts) >= 120_000
        d = np.linalg.norm(pts[:, :3], axis=1)
        assert (d == 0).sum() >= 100 and (d >= 80).any() and ((d > 70) & (d < 80)).any()


def test_oracle_unprojection_equals_reference_fixture():
    f = np.load(GOLDEN)
    pano, inten = f["unproj_pano"], f["unproj_intensities"]
    assert np.isnan(pano).any() and (pano < 0).any() and (pano == 0).any()
    ref = f["unproj_points"]
    assert np.array_equal(bits(CO.unproject(pano, inten, (2.0, 26.9))), bits(ref))
    assert np.array_equal(bits(CO.unproject(pano, None, (2.0, 26.9))), bits(ref[:, :3]))


def test_fixture_covers_the_z_buffer_rules():
    """The mixed cloud has pixels emptied by a zero-distance point with no refill (depth 0, intensity kept), pixels
    refilled after such a point, exact ties, and points that round to c == W."""
    f = np.load(GOLDEN)
    pts, h, w, k, pano, inten = load_case(f, "mixed")
    _, _, pix = CO.project(pts, h, w, k, 80, return_pixels=True)
    d = np.linalg.norm(pts[:, :3], axis=1)
    zero_pix = np.unique(pix[(d == 0) & (pix >= 0)])
    flat_p, flat_i = pano.reshape(-1), inten.reshape(-1)
    assert ((flat_p[zero_pix] == 0) & (flat_i[zero_pix] != 0)).any()
    assert (flat_p[zero_pix] > 0).any()
    _, c_pre, _, _, _ = CO.pre_round(pts, h, w, k)
    assert (np.rint(c_pre) == w).sum() > 10
    key = pix.astype(np.int64) * (1 << 32) + d.view(np.uint32)
    _, counts = np.unique(key[pix >= 0], return_counts=True)
    assert (counts > 1).sum() > 100


def test_reference_lidar_to_pano_raises_type_error():
    """utils/convert.py:89-95 passes max_dpeth= to lidar_to_pano_with_intensities, whose parameter is max_depth."""
    if not os.path.exists(os.path.join(REF, "utils", "convert.py")):
        pytest.skip("the reference checkout is not present")
    sys.path.insert(0, REF)
    try:
        conv = pytest.importorskip("utils.convert")
    finally:
        sys.path.remove(REF)
    assert callable(conv.lidar_to_pano)
    with pytest.raises(TypeError, match="max_dpeth"):
        conv.lidar_to_pano(np.ones((4, 3), np.float32), 66, 1030, [2.0, 26.9])
