"""CPU: the oracle's restatement of LiDAR4D's submodules reproduces tests/golden/modules_ref.npz, which the unmodified
reference modules (hash_field.py, planes_field.py, flow_field.py, the tcnn encodings and networks on the shim) produced:
outputs, parameter-gradient fingerprints and input gradients, at the small configuration and at L = 8."""
import os

import numpy as np
import pytest
import torch

import modules_golden_util as U
from parity_util import rel_err

TOL = 1e-5
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", U.GOLDEN))


@pytest.mark.parametrize("name", list(U.CONFIGS))
def test_oracle_reproduces_reference_modules(name):
    cfg = U.config(name)
    orc = U.oracle(name)
    om = U.OracleModules(orc)
    inp = U.inputs(cfg)
    for k, v in inp.items():
        assert np.array_equal(v.numpy(), GOLDEN[f"{name}/in/{k}"]), k
    bad = []
    for ci, (key, _, names, xkey) in enumerate(U.calls(cfg)):
        orc.zero_grad(set_to_none=True)
        i = dict(inp)
        if xkey:
            i[xkey] = inp[xkey].clone().requires_grad_(True)
        outs = om.call(key, i)
        loss = sum((o * g).sum() for o, g in zip(outs, U.upstream(outs, 100 + ci)))
        if loss.requires_grad:
            loss.backward()
        for j, o in enumerate(outs):
            e = rel_err(o, torch.from_numpy(GOLDEN[f"{name}/{key}/out{j}"]))
            if not e < TOL:
                bad.append((key, f"out{j}", e))
        for r, n in enumerate(names):
            p = orc.p(n)
            fp = U.fingerprint(p.grad if p.grad is not None else torch.zeros_like(p))
            if not U.fp_close(fp, GOLDEN[f"{name}/{key}/fp"][r], TOL):
                bad.append((key, n, fp, GOLDEN[f"{name}/{key}/fp"][r]))
        if xkey:
            e = rel_err(i[xkey].grad, torch.from_numpy(GOLDEN[f"{name}/{key}/gx"]))
            if not e < TOL:
                bad.append((key, "gx", e))
    assert not bad, bad
