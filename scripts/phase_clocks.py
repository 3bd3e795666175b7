"""Debug: per-phase clock breakdown of k_bwd_dense_tc (needs a -DL4D_PHASE_CLOCKS build at L4D_LIB_PATH)."""
import ctypes, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from lidar4d_b200 import LiDAR4D, _capi
from lidar4d_b200.rays import synthetic_sweep

dev = torch.device("cuda:0")
L, N = int(sys.argv[1]) if len(sys.argv) > 1 else 16, 4096
torch.manual_seed(0)
m = LiDAR4D(**bench.model_kwargs(L)).to(dev)
bench.randomize(m, 0)
m.materialize_weights = False
m.set_mlp_fp16(True)
ro, rd, t = synthetic_sweep(7)
sel = np.linspace(0, 65535, N).astype(np.int64)
ro_t, rd_t = torch.from_numpy(ro[sel])[None].to(dev), torch.from_numpy(rd[sel])[None].to(dev)
lib = _capi.load_library()
buf = (ctypes.c_ulonglong * 32)()
names = {0: "ray prologue", 1: "per-row values (k_bwd_composite)", 2: "load_x #1", 3: "P1 mma+epilogues", 4: "P2 heads fwd, dw3/dW2, dH1",
         6: "P2 dW1g, dG", 7: "P3", 8: "load_x #2", 9: "P4 dW1 (mma + flush)", 11: "P4 dX (-> dfeat)", 12: "ray epilogue"}
for it in range(3):
    m.zero_grad(set_to_none=True)
    out = m.render(ro_t, rd_t, float(t), num_steps=768, perturb=True)
    lib.l4d_debug_phase_clocks(buf)
    (out["depth_lidar"].sum() + out["image_lidar"].sum()).backward()
    torch.cuda.synchronize()
lib.l4d_debug_phase_clocks(buf)
v = np.array(list(buf), dtype=np.float64)
tot = v.sum()
n_tiles = N * 6
print(f"[clk] total {tot/132/1.98e6:.2f} ms per CTA; {tot/n_tiles:.0f} cycles per tile")
for i in range(13):
    if v[i] > 0:
        print(f"[clk] {i:2d} {names.get(i,''):34s} {100*v[i]/tot:6.2f}%  {v[i]/n_tiles:9.0f} cyc/tile")
