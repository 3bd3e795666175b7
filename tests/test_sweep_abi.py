"""CPU: argument checking of l4d_sweep_images through ctypes.  Every bad argument is an error code, before any launch;
none needs a GPU."""
import pytest

from lidar4d_b200 import _capi

FAKE = 256              # a device pointer that is never dereferenced: the argument check returns first


def _call(lib, depth=FAKE, image=FAKE, raydrop=None, dtype=0, H=66, W=1030, layout=0, lut_i=FAKE, lut_d=FAKE,
          panel=FAKE, pano=FAKE, inten=FAKE):
    return lib.l4d_sweep_images(depth, image, raydrop, dtype, H, W, layout, 0.01, 1, lut_i, lut_d, panel, pano, inten,
                                None)


def _fails(lib, text, **kw):
    assert _call(lib, **kw) == -1
    assert text in lib.l4d_last_error()


@pytest.mark.parametrize("layout", [_capi.SWEEP_SIM, _capi.SWEEP_TEST, _capi.SWEEP_EVAL])
def test_null_pointers(layout):
    lib = _capi.load_library()
    for name in ("depth", "image", "panel"):
        _fails(lib, b"null pointer", layout=layout, **{name: None})
    for name in ("lut_i", "lut_d"):
        _fails(lib, b"null colour table", layout=layout, **{name: None})
    if layout != _capi.SWEEP_EVAL:
        _fails(lib, b"null pano", layout=layout, pano=None)
    if layout == _capi.SWEEP_SIM:
        _fails(lib, b"null intensities", layout=layout, inten=None)


@pytest.mark.parametrize("H,W", [(0, 1030), (66, 0), (1 << 16, 1 << 15), (65536, 65536), (1 << 31, 2)])
def test_bad_sizes(H, W):
    lib = _capi.load_library()
    _fails(lib, b"H*W < 2^31", H=H, W=W)


def test_unknown_layout_and_dtype():
    lib = _capi.load_library()
    _fails(lib, b"unknown layout", layout=3)
    _fails(lib, b"dtype", raydrop=FAKE, dtype=2)
    _fails(lib, b"dtype", raydrop=None, dtype=_capi.SWEEP_F16)
    _fails(lib, b"dtype", raydrop=None, dtype=7)
