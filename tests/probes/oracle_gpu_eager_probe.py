"""SURVEY.md 8(d)(ii): the reference-equivalent PyTorch path in GPU eager mode, timed next to the CUDA path.

The true reference (PyTorch + tiny-cuda-nn) cannot run in this environment; its closest stand-in on a GPU is the
oracle (the reference's op graph restated in plain torch on the tcnn spec) executed eagerly on the same GPU.
Test infrastructure (lives under tests/, imports oracle/); prints one JSON line."""
import json, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench
from lidar4d_b200.rays import synthetic_sweep

dev = torch.device("cuda:0")
L = int(sys.argv[1]) if len(sys.argv) > 1 else 16
N = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
orc, _ = bench.build_oracle(L)
orc = orc.to(dev)
opt = torch.optim.Adam(orc.parameters(), lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
ro, rd, t = synthetic_sweep(7, bench.N_FRAMES, bench.H_SWEEP, bench.W_SWEEP)
sel = np.linspace(0, ro.shape[0] - 1, N).astype(np.int64)
ro_t, rd_t = torch.from_numpy(ro[sel]).to(dev), torch.from_numpy(rd[sel]).to(dev)


def step(seed):
    opt.zero_grad()
    out = orc.render(ro_t, rd_t, float(t), num_steps=bench.S_STEPS, perturb=True, seed=seed)
    loss = (out["depth_lidar"] - 0.3).abs().mean() + ((out["image_lidar"] - 0.5) ** 2).mean()
    loss.backward()
    opt.step()


for i in range(2):
    step(i)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 3
e0.record()
for i in range(reps):
    step(10 + i)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
print(json.dumps({"probe": "oracle (plain torch restatement of the reference graph) in GPU eager mode", "n_levels_hash": L,
                  "rays": N, "samples": bench.S_STEPS, "ms_per_step": ms, "rays_per_s": N / (ms * 1e-3),
                  "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9,
                  "note": "fwd + bwd + Adam, fp32, CUDA events, 2 warm-ups; includes the per-call fp16 table rounding the reference's tcnn modules also do"}))
