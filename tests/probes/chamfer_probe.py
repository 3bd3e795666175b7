"""Chamfer op timing on the GPU (CUDA events) next to the CPU oracle on a bounded sample; one JSON line."""
import json, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from lidar4d_b200.chamfer import chamfer_3DDist

dev = torch.device("cuda:0")
f = chamfer_3DDist()
out = {}
# the reference's own kernel, compiled in place by oracle/build_ref.py (same-box bar; chamfer3D.cu:141-142 launches it on the
# default stream, so time it with device-wide events)
try:
    from oracle import build_ref
    ref_ext = build_ref.load()
except Exception as e:      # noqa: BLE001
    ref_ext = None
    print(f"[chamfer] reference extension not available: {e}")
for (n, m) in ((1024, 1024), (30000, 30000), (100000, 100000)):
    g = torch.Generator().manual_seed(0)
    a = (torch.rand(1, n, 3, generator=g) * 2 - 1).to(dev).requires_grad_(True)
    b = (torch.rand(1, m, 3, generator=g) * 2 - 1).to(dev).requires_grad_(True)
    for _ in range(3):
        d1, d2, _, _ = f(a, b)
        (d1.sum() + d2.sum()).backward()
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    reps = 10
    e[0].record()
    for _ in range(reps):
        d1, d2, _, _ = f(a, b)
    e[1].record()
    for _ in range(reps):
        d1, d2, _, _ = f(a, b)
        (d1.sum() + d2.sum()).backward()
    e[2].record()
    torch.cuda.synchronize()
    fwd = e[0].elapsed_time(e[1]) / reps
    both = e[1].elapsed_time(e[2]) / reps
    pairs = 2.0 * n * m
    # FP32 pipe: 6 lane-operations per pair (3 subtractions, 1 multiply, 2 fma) at 128 lanes per clock per SM:
    # 132 SMs x 128 x 1.98 GHz / 6
    peak_pairs = 132 * 128 * 1.98e9 / 6
    out[f"{n}x{m}"] = {"fwd_ms": fwd, "fwd_bwd_ms": both, "pairs_per_s": pairs / (fwd * 1e-3),
                       "frac_of_fp32_pipe_peak": pairs / (fwd * 1e-3) / peak_pairs}
    if ref_ext is not None:
        r1, r2 = torch.zeros(1, n, device=dev), torch.zeros(1, m, device=dev)
        j1, j2 = torch.zeros(1, n, dtype=torch.int32, device=dev), torch.zeros(1, m, dtype=torch.int32, device=dev)
        ad, bd = a.detach(), b.detach()
        ref_ext.forward(ad, bd, r1, r2, j1, j2)
        torch.cuda.synchronize()
        rr = 3 if n >= 30000 else 10
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(rr):
            ref_ext.forward(ad, bd, r1, r2, j1, j2)
        e1.record()
        torch.cuda.synchronize()
        ref_ms = e0.elapsed_time(e1) / rr
        out[f"{n}x{m}"].update(reference_fwd_ms=ref_ms, speedup_vs_reference_kernel=ref_ms / fwd)
        print(f"[chamfer] {n} x {m}: reference kernel fwd {ref_ms:.3f} ms -> {ref_ms / fwd:.1f}x", flush=True)
    print(f"[chamfer] {n} x {m}: fwd {fwd:.3f} ms ({pairs / fwd / 1e6:.1f} G pairs/s, {100 * out[f'{n}x{m}']['frac_of_fp32_pipe_peak']:.0f}% of the FP32 pipe peak), fwd+bwd {both:.3f} ms", flush=True)
# CPU oracle on a bounded sample
from oracle import chamfer_oracle as CO
rng = np.random.default_rng(0)
x1 = rng.uniform(-1, 1, (1, 4096, 3)).astype(np.float32); x2 = rng.uniform(-1, 1, (1, 30000, 3)).astype(np.float32)
t0 = time.perf_counter(); CO.nn_distance(x1[0], x2[0]); dt = time.perf_counter() - t0
out["cpu_oracle"] = {"sample": "4096 x 30000 one direction, numpy", "pairs_per_s": 4096 * 30000 / dt}
print(f"[chamfer] cpu oracle: {4096 * 30000 / dt / 1e6:.1f} M pairs/s", flush=True)
print(json.dumps({"op": "chamfer", "results": out}))
