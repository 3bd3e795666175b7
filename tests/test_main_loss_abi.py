"""CPU: argument checking of l4d_main_loss, l4d_main_loss_backward, l4d_main_eval_loss and the re-based l4d_lidar_loss
through ctypes.  Every bad argument is an error code, returned before any launch; none needs a GPU."""
import pytest

from lidar4d_b200 import _capi

FAKE = 256              # a device pointer that is never dereferenced: the argument check returns first
EINVAL, ESIZE = -1, -3


def train(lib, depth=FAKE, image=FAKE, gt=FAKE, rays_d=FAKE, n=1024, crit=(0, 1, 1), scale=0.01, loss=FAKE, gd=FAKE,
          gi=FAKE, work=FAKE, work_bytes=None):
    if work_bytes is None:
        work_bytes = lib.l4d_main_loss_work_bytes(n)
    return lib.l4d_main_loss(depth, image, gt, rays_d, n, *crit, 1.0, 0.01, 0.1, 0.2, scale, 0.2 * scale, loss, gd, gi,
                             work, work_bytes, None)


def evaluate(lib, depth=FAKE, image=FAKE, gt=FAKE, raydrop=None, dtype=0, B=1, H=66, W=1030, crit=(0, 1, 1), loss=FAKE):
    return lib.l4d_main_eval_loss(depth, image, gt, raydrop, dtype, B, H, W, *crit, 1.0, 0.01, 0.1, 0.002, loss, None)


@pytest.mark.parametrize("name", ["depth", "image", "gt", "loss", "gd", "gi", "work"])
def test_train_null_pointers(name):
    lib = _capi.load_library()
    assert train(lib, **{name: None}) == EINVAL
    assert (b"null" in lib.l4d_last_error())


def test_train_sizes_and_codes():
    lib = _capi.load_library()
    assert train(lib, n=0) == EINVAL
    assert train(lib, n=1 << 31) == EINVAL
    for crit in ((5, 1, 1), (0, 5, 1), (0, 1, 99)):
        assert train(lib, crit=crit) == EINVAL
        assert b"unknown criterion" in lib.l4d_last_error()
    assert train(lib, work_bytes=lib.l4d_main_loss_work_bytes(1024) - 1) == ESIZE
    assert train(lib, scale=0.0) == EINVAL                 # the chamfer term divides by scale
    assert train(lib, scale=float("nan")) == EINVAL


def test_work_bytes_grow_with_n():
    lib = _capi.load_library()
    a, b = lib.l4d_main_loss_work_bytes(1), lib.l4d_main_loss_work_bytes(1024)
    assert 0 < a < b and b >= 1024 * (18 * 4 + 16)


def test_backward_checks():
    lib = _capi.load_library()
    f = lib.l4d_main_loss_backward
    assert f(FAKE, FAKE, 0, FAKE, FAKE, FAKE, None) == EINVAL
    for i in range(5):
        args = [FAKE] * 5
        args[i] = None
        assert f(args[0], args[1], 16, *args[2:], None) == EINVAL


def test_eval_checks():
    lib = _capi.load_library()
    for name in ("depth", "image", "gt", "loss"):
        assert evaluate(lib, **{name: None}) == EINVAL
    assert evaluate(lib, B=0) == EINVAL
    assert evaluate(lib, H=1 << 16, W=1 << 15) == EINVAL
    assert evaluate(lib, crit=(0, 6, 1)) == EINVAL
    assert evaluate(lib, raydrop=FAKE, dtype=3) == EINVAL


def test_lidar_loss_keeps_its_contract():
    """n = 0 adds nothing and launches nothing; null pointers are still rejected."""
    lib = _capi.load_library()
    before = lib.l4d_launch_count()
    assert lib.l4d_lidar_loss(FAKE, FAKE, FAKE, 0, 1.0, 0.01, 0.1, 0.2, FAKE, FAKE, FAKE, None) == 0
    assert lib.l4d_launch_count() == before
    assert lib.l4d_lidar_loss(None, FAKE, FAKE, 16, 1.0, 0.01, 0.1, 0.2, FAKE, FAKE, FAKE, None) == EINVAL
