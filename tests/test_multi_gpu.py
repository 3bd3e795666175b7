"""GPU, >= 2 devices (gpurun --gpus 2): ray-sharded data parallelism over NCCL.  Each rank renders its contiguous
ray range with the global ray offset, losses are normalised by the global ray count, ONE all-reduce of the flat
gradient arena follows; the result must equal the single-GPU gradient of the whole batch (SURVEY.md 8(e))."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
from oracle import lidar4d_oracle as O
from parity_util import small_config, cuda_model_from_oracle, rel_err, test_rays
from lidar4d_b200.parallel import RayShardedDP
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
orc = O.build_seeded(small_config(), 21, flow_last_std=0.02)
ro, rd = test_rays(4, 9)
N, S, t = ro.shape[0], 200, 0.4
ro_t, rd_t = torch.from_numpy(ro)[None].cuda(), torch.from_numpy(rd)[None].cuda()
def grads(model, dp, overlapped=False):
    model.zero_grad(set_to_none=True)
    model._jitter_calls = 0
    out = dp.render(ro_t, rd_t, torch.tensor([[t]]), num_steps=S, perturb=True) if dp else \
          model.render(ro_t, rd_t, torch.tensor([[t]]), num_steps=S, perturb=True)
    loss = ((out["depth_lidar"] - 0.3).abs().sum() + ((out["image_lidar"] - 0.5) ** 2).sum()) / N
    if dp and overlapped: dp.final_backward(loss)      # hash-table bucket reduced on a side stream behind the kernels' event
    else: loss.backward()
    if dp: dp.allreduce_grads()
    return {{k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}}
for fp16 in (False, True):
    m = cuda_model_from_oracle(orc, device=f"cuda:{{rank}}").set_mlp_fp16(fp16)
    g_dp = grads(m, RayShardedDP(m, world_size=world, rank=rank))
    g_1 = grads(m, None)                      # every rank also computes the whole batch alone
    worst = max(rel_err(g_dp[k], g_1[k]) for k in g_1)
    assert worst < 1e-4, (fp16, worst)
    g_ov = grads(m, RayShardedDP(m, world_size=world, rank=rank), overlapped=True)
    worst_ov = max(rel_err(g_ov[k], g_1[k]) for k in g_1)
    assert worst_ov < 1e-4, ("overlapped", fp16, worst_ov)
    if rank == 0: print(f"mlp_fp16={{fp16}} sharded-vs-single worst rel err {{worst:.2e}}", flush=True)
dist.barrier(); dist.destroy_process_group()
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_gradients_equal_single_gpu(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29571", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert "sharded-vs-single" in r.stdout
