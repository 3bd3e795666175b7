"""Test helper: build and load tests/hostsim/_points_hostsim.so, the host mirrors of the explicit-point kernels
(lidar4d_b200/csrc/l4d_points.cuh) compiled for the CPU.  Staging and unstaging come from the host-sim library
(hostsim_util).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

from lidar4d_b200 import _capi

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostsim", "points_hostsim.cu")
SO = os.path.join(HERE, "hostsim", "_points_hostsim.so")
_LIB = None


def build(force=False):
    deps = [SRC] + [os.path.join(HERE, "..", "lidar4d_b200", "csrc", f) for f in ("l4d_core.cuh", "l4d_bwd.cuh", "l4d_host.h")]
    if not force and os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    cmd = ["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC,-ffp-contract=off",
           "-gencode", "arch=compute_90a,code=sm_90a", "-o", SO, SRC]
    subprocess.run(cmd, check=True)
    return SO


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(SO)
        P, V, U32 = C.POINTER, C.c_void_p, C.c_uint32
        L.hs_points_last_error.restype = C.c_char_p
        L.hs_points_last_error.argtypes = []
        L.hs_density_saved_bytes.restype = C.c_size_t
        L.hs_density_saved_bytes.argtypes = [P(_capi.L4DConfig), U32]
        L.hs_density_forward_ex.argtypes = [P(_capi.L4DConfig), V, P(_capi.L4DFrame), V, U32, V, V, V, V, V]
        L.hs_density_backward.argtypes = [P(_capi.L4DConfig), V, P(_capi.L4DFrame), V, U32, V, V, V,
                                          P(_capi.L4DMasterGrads), V]
        L.hs_attribute_backward.argtypes = [P(_capi.L4DConfig), V, V, V, V, U32, V, V, P(_capi.L4DMasterGrads), V]
        for n in ("hs_density_forward_ex", "hs_density_backward", "hs_attribute_backward"):
            getattr(L, n).restype = C.c_int
        _LIB = L
    return _LIB
