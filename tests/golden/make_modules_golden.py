"""Generate tests/golden/modules_ref.npz by calling the submodules of the UNMODIFIED reference LiDAR4D
(/root/reference/model/{lidar4d,hash_field,planes_field,flow_field}.py) on top of oracle/tcnn_shim.py: hash grids,
HashGridT at the times of modules_golden_util.times, raw time slices, hex-planes, the flow field and its grid, the
frequency encoding and the three networks.  Outputs, parameter-gradient fingerprints and the input gradients (planes,
networks) of a seeded scalar loss, at the small test configuration and at the default L = 8.

Run in the build container only (needs /root/reference, read-only):
    python tests/golden/make_modules_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True
REF = "/root/reference"

from oracle import tcnn_shim  # noqa: E402
import modules_golden_util as U  # noqa: E402


def reference_model(name):
    tcnn_shim.install()
    sys.path.insert(0, REF)
    import model.hash_field as hf
    import model.flow_field as ff
    import model.lidar4d as l4d
    cfg = U.config(name)
    if name == "small":
        # the reference's dynamic-hash and flow-grid sizes are constructor defaults (hash_field.py:100,
        # flow_field.py:50-54): reach them through the constructors' keyword arguments
        class SmallHash(hf.HashGrid4D):
            def __init__(self, **kw):
                super().__init__(hash_size_dynamic=list(cfg.hash_size_dynamic), **kw)

        class SmallFlow(ff.FlowField):
            def __init__(self, **kw):
                super().__init__(base_resolution=cfg.flow_base_resolution, max_resolution=cfg.flow_max_resolution,
                                 log2_hashmap_size=cfg.flow_log2_hashmap_size, **kw)
        l4d.HashGrid4D, l4d.FlowField = SmallHash, SmallFlow
    else:
        l4d.HashGrid4D, l4d.FlowField = hf.HashGrid4D, ff.FlowField
    kw = {k: v for k, v in U.CONFIGS[name][0].items()
          if k not in ("hash_size_dynamic", "flow_base_resolution", "flow_max_resolution", "flow_log2_hashmap_size")}
    ref = l4d.LiDAR4D(**kw)
    res = ref.load_state_dict(U.oracle(name).ref_state_dict(), strict=False)
    assert not [k for k in res.missing_keys if not k.startswith("unet.")], res
    return ref


def main():
    out = {}
    for name in U.CONFIGS:
        cfg = U.config(name)
        ref = reference_model(name)
        params = dict(ref.named_parameters())
        inp = U.inputs(cfg)
        for k, v in inp.items():
            out[f"{name}/in/{k}"] = v.numpy()
        for ci, (key, fn, names, xkey) in enumerate(U.calls(cfg)):
            ref.zero_grad(set_to_none=True)
            i = dict(inp)
            if xkey:
                i[xkey] = inp[xkey].clone().requires_grad_(True)
            outs = fn(ref, i)
            gs = U.upstream(outs, 100 + ci)
            loss = sum((o.float() * g).sum() for o, g in zip(outs, gs))
            if loss.requires_grad:                  # the frequency encoding has no parameters
                loss.backward()
            for j, o in enumerate(outs):
                out[f"{name}/{key}/out{j}"] = o.detach().float().numpy()
            if names:          # one row per parameter of `names`
                out[f"{name}/{key}/fp"] = np.stack([U.fingerprint(params[n].grad if params[n].grad is not None
                                                                  else torch.zeros_like(params[n])) for n in names])
            if xkey:
                out[f"{name}/{key}/gx"] = i[xkey].grad.numpy()
            print(f"[{name}] {key}: " + ", ".join(str(tuple(o.shape)) for o in outs))
    path = os.path.join(ROOT, "tests", "golden", U.GOLDEN)
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
