"""Generate tests/golden/image_metrics_ref.npz: the rows and measure() of the reference's own, unmodified DepthMeter,
IntensityMeter and RaydropMeter (utils/metrics.py) on the frames of tests/image_metrics_cases.py, for
tests/test_image_metrics_oracle.py (CPU) and tests/test_gpu_image_metrics.py (the CUDA ops against the reference).

Run where the reference checkout exists (CPU only, seconds):
    python tests/golden/make_image_metrics_golden.py [OUT.npz]      # the checkout tests/ref_stubs.py points at

skimage and lpips are replaced by tests/skimage_stub.py: structural_similarity by oracle/image_metrics_oracle.py's
restatement (neither package is a dependency of this project), LPIPS by a sentinel.  DepthMeter runs at scale 1.0, so
that no division enters the comparison.  What is recorded, per case:
  <case>_sha256              the SHA-256 of the rebuilt (pred, gt) frames;
  <case>_row                 the meter's row (rmse, medae, lpips, ssim, psnr) of an image case, float64;
  <case>_r<ratio>_row        the row (rmse, acc, f1) of a ray-drop case at each of its ratios, float64;
  measure_depth / measure_intensity / measure_raydrop_r<ratio>  measure() over all cases of that meter, in list order."""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)

import image_metrics_cases as IC  # noqa: E402
import skimage_stub  # noqa: E402


def raydrop_key(name, ratio):
    return f"{name}_r{ratio:g}"


def main(out_path):
    import scipy
    M = skimage_stub.reference_metrics()
    fx = {"numpy_version": np.array(np.__version__), "scipy_version": np.array(scipy.__version__),
          "lpips_sentinel": np.array(skimage_stub.SENTINEL)}
    meters = {"depth": M.DepthMeter(scale=1.0), "intensity": M.IntensityMeter(scale=1.0)}
    warnings.simplefilter("ignore", RuntimeWarning)
    for name in IC.IMAGE_CASES:
        kind, p, g = IC.frame(None, name)
        fx[f"{name}_sha256"] = np.array(IC.digest(p, g))
        m = meters[kind]
        m.update(torch.from_numpy(p.copy()), torch.from_numpy(g.copy()))
        fx[f"{name}_row"] = np.array(m.V[-1], np.float64)
        print(name, kind, fx[f"{name}_row"])
    for kind, m in meters.items():
        fx[f"measure_{kind}"] = np.asarray(m.measure(), np.float64)
    ratios = sorted({r for rs in IC.RAYDROP_CASES.values() for r in rs})
    for ratio in ratios:
        m = M.RaydropMeter(ratio=ratio)
        for name, rs in IC.RAYDROP_CASES.items():
            if ratio not in rs:
                continue
            _, p, g = IC.frame(None, name)
            fx[f"{name}_sha256"] = np.array(IC.digest(p, g))
            m.update(torch.from_numpy(p.copy()), torch.from_numpy(g.copy()))
            fx[f"{raydrop_key(name, ratio)}_row"] = np.array(m.V[-1], np.float64)
            print(raydrop_key(name, ratio), fx[f"{raydrop_key(name, ratio)}_row"])
        fx[f"measure_raydrop_r{ratio:g}"] = np.asarray(m.measure(), np.float64)
    np.savez_compressed(out_path, **fx)
    print(f"wrote {out_path} ({os.path.getsize(out_path)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "image_metrics_ref.npz"))
