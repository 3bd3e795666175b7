"""CPU: argument checking of l4d_encoder_forward / _backward and l4d_mlp_forward / _backward through ctypes.  Every bad
argument is an error code returned before any launch, and n = 0 returns before one; none needs a GPU."""
import ctypes as C

import pytest

from lidar4d_b200 import _capi
from lidar4d_b200.geometry import make_time_query
from parity_util import small_config

FAKE = 256              # a device pointer that is never dereferenced: the argument check returns first
EINVAL, ESIZE = -1, -3


@pytest.fixture(scope="module")
def env():
    lib = _capi.load_library()
    cfg = _capi.make_config(small_config(), True)
    q = _capi.make_time_query(make_time_query(0.4, 8))
    g = _capi.L4DMasterGrads()
    _capi.fill_pointer_table(g, small_config(), lambda n: FAKE)
    return lib, cfg, q, g


def enc_fwd(env, module=0, q=True, slice_=0, x=FAKE, n=100, out=FAKE, staged=FAKE):
    lib, cfg, qq, _ = env
    return lib.l4d_encoder_forward(C.byref(cfg), staged, module, C.byref(qq) if q else None, slice_, x, n, out, None)


def enc_bwd(env, module=0, x=FAKE, n=100, g_out=FAKE, g_x=None, grads=True, work=FAKE, work_bytes=None, slice_=0):
    lib, cfg, q, g = env
    if work_bytes is None:
        work_bytes = lib.l4d_grad_work_bytes(C.byref(cfg))
    return lib.l4d_encoder_backward(C.byref(cfg), FAKE, module, C.byref(q), slice_, x, n, g_out, g_x,
                                    C.byref(g) if grads else None, work, work_bytes, None)


def mlp_fwd(env, net=0, inp=FAKE, n=100, out=FAKE):
    lib, cfg, _, _ = env
    return lib.l4d_mlp_forward(C.byref(cfg), FAKE, net, inp, n, out, None)


def mlp_bwd(env, net=0, inp=FAKE, n=100, g_out=FAKE, g_in=None, grads=True, work=FAKE, work_bytes=None):
    lib, cfg, _, g = env
    if work_bytes is None:
        work_bytes = lib.l4d_grad_work_bytes(C.byref(cfg))
    return lib.l4d_mlp_backward(C.byref(cfg), FAKE, net, inp, n, g_out, g_in, C.byref(g) if grads else None, work,
                                work_bytes, None)


def test_zero_points_is_a_no_op(env):
    for m in range(13):
        assert enc_fwd(env, module=m, n=0) == 0
    for m in range(12):
        assert enc_bwd(env, module=m, n=0) == 0
    for net in range(3):
        assert mlp_fwd(env, net=net, n=0) == 0 and mlp_bwd(env, net=net, n=0) == 0


def test_null_and_misaligned_pointers(env):
    lib = env[0]
    assert enc_fwd(env, x=None) == EINVAL and b"null" in lib.l4d_last_error()
    assert enc_fwd(env, out=None) == EINVAL
    assert enc_fwd(env, staged=None) == EINVAL
    assert enc_fwd(env, x=FAKE + 2) == EINVAL and b"misaligned" in lib.l4d_last_error()
    assert enc_fwd(env, out=FAKE + 1) == EINVAL
    assert enc_bwd(env, g_out=None) == EINVAL
    assert enc_bwd(env, grads=False) == EINVAL
    assert enc_bwd(env, work=None) == EINVAL
    assert enc_bwd(env, module=8, g_x=FAKE + 2) == EINVAL
    assert mlp_fwd(env, inp=None) == EINVAL and mlp_fwd(env, out=None) == EINVAL
    assert mlp_fwd(env, inp=FAKE + 2) == EINVAL
    assert mlp_bwd(env, g_out=None) == EINVAL and mlp_bwd(env, grads=False) == EINVAL
    assert mlp_bwd(env, g_in=FAKE + 3) == EINVAL


def test_ids_sizes_and_rules(env):
    lib, cfg, _, _ = env
    assert enc_fwd(env, module=13) == EINVAL and b"module" in lib.l4d_last_error()
    assert enc_bwd(env, module=99) == EINVAL
    assert mlp_fwd(env, net=3) == EINVAL and mlp_bwd(env, net=7) == EINVAL
    assert enc_fwd(env, n=(1 << 31) + 1) == EINVAL and mlp_fwd(env, n=0xFFFFFFFF) == EINVAL
    assert enc_fwd(env, module=1, q=False) == EINVAL and b"query" in lib.l4d_last_error()
    assert enc_fwd(env, module=4, q=False) == EINVAL
    assert enc_fwd(env, module=5, slice_=8) == EINVAL            # time_resolution 8
    assert enc_bwd(env, module=12) == EINVAL                      # the frequency encoding has no parameters
    assert enc_bwd(env, module=0, g_x=FAKE) == EINVAL             # only the planes give an input gradient
    assert enc_bwd(env, work_bytes=lib.l4d_grad_work_bytes(C.byref(cfg)) - 4) == ESIZE
    assert mlp_bwd(env, work_bytes=16) == ESIZE
