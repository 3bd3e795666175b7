"""CPU: argument checking of the range-image / point-cloud entry points (l4d_pano_project, l4d_pano_unproject,
l4d_point_metrics) through ctypes.  Every bad argument is an error code, before any launch; none needs a GPU."""
import pytest

from lidar4d_b200 import _capi

FAKE = 256              # a device pointer that is never dereferenced: the argument check returns first
BIG = 1 << 40


def _project(lib, n=10, stride=4, H=66, W=1030, pts=FAKE, pano=FAKE, work=FAKE, nwork=BIG):
    return lib.l4d_pano_project(pts, n, stride, 2.0, 26.9, H, W, 80.0, pano, None, work, nwork, None)


def _unproject(lib, H=66, W=1030, pano=FAKE, out=FAKE, count=FAKE, work=FAKE, nwork=BIG):
    return lib.l4d_pano_unproject(pano, None, H, W, 2.0, 26.9, out, count, work, nwork, None)


def test_work_sizes():
    lib = _capi.load_library()
    assert lib.l4d_pano_project_work_bytes(66, 1030) == 66 * 1030 * 12
    assert lib.l4d_pano_unproject_work_bytes(66, 1030) == (66 * 1030 + 1023) // 1024 * 4
    assert lib.l4d_pano_unproject_work_bytes(1, 1) == 4


@pytest.mark.parametrize("H,W", [(0, 1030), (66, 0), (0, 0), (1 << 16, (1 << 15) + 1), (1 << 31, 2), (65536, 65536)])
def test_bad_image_sizes(H, W):
    lib = _capi.load_library()
    assert _project(lib, H=H, W=W) == -1
    assert b"H*W <= 2^31" in lib.l4d_last_error()
    assert _unproject(lib, H=H, W=W) == -1
    assert b"H*W <= 2^31" in lib.l4d_last_error()


def test_largest_image_passes_the_size_check():
    """H*W = 2^31 is allowed: with a too-small work buffer the next check (not the size check) fails."""
    lib = _capi.load_library()
    assert _project(lib, H=1 << 16, W=1 << 15, nwork=0) == -3
    assert _unproject(lib, H=1 << 16, W=1 << 15, nwork=0) == -3


@pytest.mark.parametrize("stride", [0, 2, 5, 16])
def test_bad_stride(stride):
    lib = _capi.load_library()
    assert _project(lib, stride=stride) == -1
    assert b"stride must be 3 or 4" in lib.l4d_last_error()


def test_null_pointers():
    lib = _capi.load_library()
    assert _project(lib, pts=None) == -1
    assert _project(lib, pano=None) == -1
    assert _unproject(lib, pano=None) == -1
    assert _unproject(lib, out=None) == -1
    assert _unproject(lib, count=None) == -1
    for args in ((None, 3, FAKE, 4), (FAKE, 3, None, 4), (FAKE, 3, FAKE, 4, None)):
        d1, n, d2, m, *out = args
        assert lib.l4d_point_metrics(d1, n, d2, m, 0.05, out[0] if out else FAKE, None) == -1
    assert b"null pointer" in lib.l4d_last_error()


def test_too_small_work():
    lib = _capi.load_library()
    need = lib.l4d_pano_project_work_bytes(66, 1030)
    assert _project(lib, nwork=need - 1) == -3
    assert b"work buffer too small" in lib.l4d_last_error()
    assert _project(lib, work=None) == -3
    need = lib.l4d_pano_unproject_work_bytes(66, 1030)
    assert _unproject(lib, nwork=need - 1) == -3
    assert _unproject(lib, work=None) == -3


def test_empty_clouds():
    """n = 0 points is a valid projection (points may then be NULL; its argument check passes, as a too-small work
    buffer behind it shows); an empty cloud is an error for the metric."""
    lib = _capi.load_library()
    assert _project(lib, n=0, pts=None, nwork=0) == -3
    assert lib.l4d_point_metrics(FAKE, 0, FAKE, 4, 0.05, FAKE, None) == -1
    assert b"empty point cloud" in lib.l4d_last_error()
    assert lib.l4d_point_metrics(FAKE, 4, FAKE, 0, 0.05, FAKE, None) == -1
