"""CPU: the element math of the refinement loop's ops compiled for the host (tests/hostsim/refinesim.cu over
lidar4d_b200/csrc/l4d_refine.cuh, contraction off) against what the reference runs on the CPU:
  - the box mask against torch's ones_like / slice assignment / multiply (runner.py:888-898), bit for bit, on values with
    negatives, +-inf and NaN;
  - the BCE element against torch's CPU binary_cross_entropy(reduction='none') to 1 ulp (torch's CPU log differs from
    the C library's in the last bit for a few per cent of elements), and the clamp at -100 exactly;
  - the gradient against torch's CPU BCELoss gradient, bit for bit, for upstream gradients 1 and 65,536;
  - a prediction outside [0, 1] or NaN gives a NaN element and gradient (torch refuses such input).
And the C-ABI's argument checks, which return before any launch and need no GPU."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from lidar4d_b200 import _capi

SO_PATH = os.path.join(os.path.dirname(__file__), "hostsim", "_refinesim.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(SO_PATH):
        pytest.fail(f"{SO_PATH} missing: run __graft_entry__.build()")
    h = C.CDLL(SO_PATH)
    P, N, U = C.c_void_p, C.c_size_t, C.c_uint32
    h.rfs_box_mask.argtypes = [P, P, U, U, U, P, U]
    h.rfs_bce.argtypes = [P, P, N, P]
    h.rfs_bce_grad.argtypes = [P, P, N, C.c_float, P]
    return h


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _wild(rng, shape):
    x = rng.standard_normal(shape).astype(np.float32) * 3
    k = rng.integers(0, 20, shape)
    x[k == 0] = np.inf
    x[k == 1] = -np.inf
    x[k == 2] = np.nan
    x[k == 3] = 0.0
    return x


def _reference_mask(x, boxes):
    t = torch.from_numpy(x)
    mask = torch.ones_like(t)
    for y0, x0, h, w in boxes:
        mask[:, :, y0:y0 + h, x0:x0 + w] = 0.
    return (t * mask).numpy()


def _boxes(rng, H, W, n):
    out = []
    for _ in range(n):
        h, w = int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))
        out.append((int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w))
    return out


@pytest.mark.parametrize("shape,n", [((2, 3, 12, 40), 0), ((2, 3, 12, 40), 31), ((1, 1, 1, 1), 1), ((3, 2, 7, 13), 32),
                                     ((1, 3, 66, 103), 5)])
def test_box_mask_bit_exact(lib, shape, n):
    rng = np.random.default_rng(sum(shape) + n)
    x = _wild(rng, shape)
    B, Ch, H, W = shape
    boxes = _boxes(rng, H, W, n)
    if n >= 2:      # boxes on every edge and corner
        boxes[0] = (0, 0, 1, W)
        boxes[1] = (H - 1, W - 1, 1, 1)
    out = np.empty_like(x)
    arr = np.array(boxes, np.int32).reshape(-1, 4)
    lib.rfs_box_mask(_p(x), _p(out), B * Ch, H, W, _p(arr), len(boxes))
    ref = _reference_mask(x, boxes)
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))        # -0.0 and NaN payloads included


def _inputs(rng, n):
    x = rng.uniform(0, 1, n).astype(np.float32)
    x[:6] = [0.0, 1.0, 1e-45, 1 - 2 ** -24, 2 ** -126, 0.5]        # the clamps, subnormal and the last float below 1
    t = rng.uniform(0, 1, n).astype(np.float32)
    t[: n // 3] = np.round(t[: n // 3])                               # binary targets, as the ray-drop mask
    t[:6] = [1.0, 0.0, 1.0, 0.0, 0.3, 0.5]
    return x, t


def _ulps(a, b):
    ai, bi = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7FFFFFFF), ai)
    bi = np.where(bi < 0, -(bi & 0x7FFFFFFF), bi)
    return np.abs(ai - bi)


def test_bce_element_against_torch_cpu(lib):
    x, t = _inputs(np.random.default_rng(1), 200_000)
    got = np.empty_like(x)
    lib.rfs_bce(_p(x), _p(t), x.size, _p(got))
    ref = torch.nn.functional.binary_cross_entropy(torch.from_numpy(x), torch.from_numpy(t), reduction="none").numpy()
    u = _ulps(got, ref)
    assert u.max() <= 1, u.max()
    assert got[0] == 100.0 and got[1] == 100.0       # log(0) and log1p(-1) clamped at -100
    print(f"BCE element vs torch CPU: {np.mean(u > 0) * 100:.2f} % of elements 1 ulp off")


@pytest.mark.parametrize("g", [1.0, 65536.0])
def test_bce_gradient_bit_exact_against_torch_cpu(lib, g):
    x, t = _inputs(np.random.default_rng(2), 100_003)
    got = np.empty_like(x)
    lib.rfs_bce_grad(_p(x), _p(t), x.size, g, _p(got))
    xt = torch.from_numpy(x).requires_grad_()
    (torch.nn.BCELoss()(xt, torch.from_numpy(t)) * g).backward()
    assert np.array_equal(got.view(np.uint32), xt.grad.numpy().view(np.uint32))


def test_out_of_range_predictions_are_nan(lib):
    x = np.array([-1e-8, 1.0000001, -np.inf, np.inf, np.nan, 2.0, 0.25], np.float32)
    t = np.full_like(x, 0.5)
    loss, grad = np.empty_like(x), np.empty_like(x)
    lib.rfs_bce(_p(x), _p(t), x.size, _p(loss))
    lib.rfs_bce_grad(_p(x), _p(t), x.size, 1.0, _p(grad))
    assert np.isnan(loss[:6]).all() and np.isnan(grad[:6]).all()
    assert np.isfinite(loss[6]) and np.isfinite(grad[6])


# ---------------------------------------------------------------------------------------------------------------------
# C-ABI argument checks (the real library; every call returns before touching a pointer or the device)
# ---------------------------------------------------------------------------------------------------------------------
FAKE = 256


def _boxes_arg(boxes):
    return (C.c_int32 * (4 * len(boxes)))(*[v for b in boxes for v in b]) if boxes else None


@pytest.mark.parametrize("boxes,text", [
    ([(-1, 0, 1, 1)], b"outside"), ([(0, -1, 1, 1)], b"outside"), ([(0, 0, 0, 1)], b"outside"),
    ([(0, 0, 1, 0)], b"outside"), ([(60, 0, 7, 1)], b"outside"), ([(0, 1000, 1, 31)], b"outside"),
    ([(0, 0, 1, 1)] * 33, b"more than 32"), ([(0, 2 ** 31 - 1, 1, 2)], b"outside")])
def test_box_mask_rejects_bad_boxes(boxes, text):
    lib = _capi.load_library()
    assert lib.l4d_box_mask(FAKE, FAKE, 2, 3, 66, 1030, _boxes_arg(boxes), len(boxes), None) == _capi.EINVAL
    assert text in lib.l4d_last_error()


def test_box_mask_rejects_bad_shapes_and_pointers():
    lib = _capi.load_library()
    for args in ((None, FAKE, 1, 1, 4, 4), (FAKE, None, 1, 1, 4, 4), (FAKE, FAKE, 0, 1, 4, 4), (FAKE, FAKE, 1, 1, 4, 0),
                 (FAKE, FAKE, 1 << 16, 1 << 15, 1, 1)):
        assert lib.l4d_box_mask(*args, None, 0, None) == _capi.EINVAL
    assert lib.l4d_box_mask(FAKE, FAKE, 1, 1, 4, 4, None, 3, None) == _capi.EINVAL
    assert b"null boxes" in lib.l4d_last_error()


def test_bce_rejects_bad_arguments():
    lib = _capi.load_library()
    wb = lib.l4d_bce_loss_work_bytes()
    assert wb >= 8 * 1024
    assert lib.l4d_bce_loss(FAKE, 3, FAKE, 10, FAKE, FAKE, wb, None) == _capi.EINVAL
    assert b"dtype" in lib.l4d_last_error()
    assert lib.l4d_bce_loss(FAKE, 0, FAKE, 0, FAKE, FAKE, wb, None) == _capi.EINVAL
    assert lib.l4d_bce_loss(FAKE, 0, FAKE, 1 << 31, FAKE, FAKE, wb, None) == _capi.EINVAL
    assert lib.l4d_bce_loss(None, 0, FAKE, 10, FAKE, FAKE, wb, None) == _capi.EINVAL
    assert lib.l4d_bce_loss(FAKE, 0, FAKE, 10, None, FAKE, wb, None) == _capi.EINVAL
    assert lib.l4d_bce_loss(FAKE, 0, FAKE, 10, FAKE, FAKE, wb - 1, None) == -3          # L4D_ESIZE
    assert lib.l4d_bce_loss_backward(FAKE, 7, FAKE, 10, FAKE, FAKE, None) == _capi.EINVAL
    assert lib.l4d_bce_loss_backward(FAKE, 2, FAKE, 10, None, FAKE, None) == _capi.EINVAL
    assert lib.l4d_bce_loss_backward(FAKE, 2, FAKE, 10, FAKE, None, None) == _capi.EINVAL
