"""ORACLE support (test infrastructure, NOT product code): compile the reference's OWN chamfer extension
(/root/reference/utils/chamfer3D/chamfer3D.cu + chamfer_cuda.cpp, a self-contained torch cpp-extension) for sm_90a
from the sources where they lie, into oracle/_ref/ (git-ignored, travels to the GPU box with the snapshot).

    python oracle/build_ref.py            # build container only: needs /root/reference (read-only) and nvcc

It is used (a) as the TRUE oracle of tests/test_chamfer.py - distances and indices of the CUDA kernel must equal the
reference kernel's bit for bit - and (b) as the same-box performance bar of the chamfer op (bench.py / profiles).
Nothing is copied: the two source files are compiled in place by torch.utils.cpp_extension (ninja + nvcc), the
reference's own setup.py / JIT loader (dist_chamfer_3D.py:8-28) is not run.  The rest of the reference's hot path
needs tiny-cuda-nn (absent, CUDA-only, un-vendored) and is not buildable here; see DESIGN.md.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/utils/chamfer3D"
OUT = os.path.join(ROOT, "oracle", "_ref")
NAME = "chamfer_3D_ref"


def so_path():
    return os.path.join(OUT, NAME + ".so")


def build(force: bool = False) -> str:
    """Returns the path of the built extension, or '' when the reference sources are not available here."""
    out = so_path()
    srcs = [os.path.join(REF, "chamfer_cuda.cpp"), os.path.join(REF, "chamfer3D.cu")]
    if not all(os.path.exists(s) for s in srcs):
        return out if os.path.exists(out) else ""
    if os.path.exists(out) and not force and all(os.path.getmtime(s) < os.path.getmtime(out) for s in srcs):
        return out
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    from torch.utils import cpp_extension
    cpp_extension.load(name=NAME, sources=srcs, build_directory=OUT, verbose=True, is_python_module=False,
                       extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo"])
    return out


def load():
    """Import the prebuilt reference extension (raises if it was never built)."""
    import importlib.util
    import torch  # noqa: F401  (the extension links against libtorch)
    p = so_path()
    if not os.path.exists(p):
        raise FileNotFoundError(p + " - run `python oracle/build_ref.py` in the build container")
    spec = importlib.util.spec_from_file_location(NAME, p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    p = build(force="--force" in sys.argv)
    print("built:" if p else "reference sources not available:", p)
