"""Gradient updates per sample that the backward's hash-grid scatters send to L2, on the benchmark's own rays (host only).

For the static hash and the dynamic hash (contracted path: one float per entry), both scattered by k_bwd_encoders, per level
and in total, under three reductions of a warp of 32 consecutive samples of one ray:
  per-lane    every sample updates each of its corners (8 in 3D, 4 in 2D);
  cell-run    runs of consecutive samples in the same cell update each corner once (the former static-hash path used it at the
              levels up to res 1200, bench.STATIC_AGG_RES, and per-lane updates above);
  vertex-run  one update per distinct grid vertex of the warp (l4d_vertex_sum in lidar4d_b200/csrc/l4d_bwd.cuh).
Positions are those of bench.py::red_counts: the unjittered z grid of S = 768 samples, x01 = (o + d z + bound) / (2 bound), for
--rays rays spread evenly over one synthetic sweep.
The counts are of updated values; the dynamic hash packs two x-neighbour updates that fall in one aligned quad of entries
into one 16-byte reduction, which this does not model.

  python scripts/red_count.py [--levels 16] [--frame 0] [--rays 512]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def warp_counts(cell):
    """cell: int64 [rays, S, D] cells at one level, S a multiple of 32 -> (per-lane, cell-run, vertex-run) updates per sample"""
    R, S, D = cell.shape
    K = 1 << D
    w = cell.reshape(R, S // 32, 32, D)
    same = np.all(w[:, :, 1:] == w[:, :, :-1], axis=-1)
    runs = 1 + (~same).sum(-1)                                         # runs of equal cells per warp
    offs = np.array([[(s >> a) & 1 for a in range(D)] for s in range(K)], np.int64)
    vert = w[:, :, :, None, :] + offs[None, None, None]                # [R, W, 32, K, D]
    vert = vert.reshape(R, S // 32, 32 * K, D)
    # distinct vertices per warp: lexicographic sort of the warp's 32 K vertices, count changes
    key = vert[..., 0]
    for a in range(1, D):
        key = key * (1 << 21) + vert[..., a]
    key = np.sort(key, axis=-1)
    distinct = 1 + (key[..., 1:] != key[..., :-1]).sum(-1)
    n = float(R * S)
    return float(K), float(K * runs.sum()) / n, float(distinct.sum()) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, default=16)
    ap.add_argument("--frame", type=int, default=0)
    ap.add_argument("--rays", type=int, default=512)
    args = ap.parse_args()
    import bench
    from lidar4d_b200.geometry import FieldConfig
    from lidar4d_b200.rays import synthetic_sweep
    cfg = FieldConfig(**bench.model_kwargs(args.levels))
    ro, rd, _ = synthetic_sweep(args.frame, bench.N_FRAMES, bench.H_SWEEP, bench.W_SWEEP)
    sel = np.linspace(0, len(ro) - 1, args.rays).astype(np.int64)
    ro, rd = np.asarray(ro, np.float32)[sel], np.asarray(rd, np.float32)[sel]
    z = np.linspace(np.float32(cfg.near_lidar), np.float32(cfg.far_lidar), bench.S_STEPS, dtype=np.float32)
    x01 = (ro[:, None, :] + rd[:, None, :] * z[None, :, None] + np.float32(cfg.bound)) / np.float32(2 * cfg.bound)
    L = args.levels

    def cells(g, l, coords):
        return np.floor(coords * g.scale[l] + np.float32(0.5)).astype(np.int64)

    print(f"updates per sample, {args.rays} rays of frame {args.frame}, S = {bench.S_STEPS}, L = {L}")
    print("static hash            per-lane  cell-run  vertex-run")
    gs = cfg.static_grid()
    tot = np.zeros(3)
    former = 0.0
    for l in range(L):
        c = warp_counts(cells(gs, l, x01))
        tot += c
        former += c[1] if int(gs.resolution[l]) <= bench.STATIC_AGG_RES else c[0]
        print(f"  level {l:2d} res {int(gs.resolution[l]):5d}  {c[0]:7.2f}  {c[1]:8.2f}  {c[2]:10.2f}")
    print(f"  total                {tot[0]:7.1f}  {tot[1]:8.1f}  {tot[2]:10.1f}")
    print(f"  former path (cell runs up to res {bench.STATIC_AGG_RES}): {former:.1f}")
    print("dynamic hash (x,t) query, one value per corner")
    tot_d = np.zeros(3)
    for p in range(3):
        gd = cfg.dynamic_grid(p)
        ca = x01[..., 1] if p == 2 else x01[..., 0]                       # planes (x,y) (x,z) (y,z), as l4d_bw_dynhash_slice
        cb = x01[..., 1] if p == 0 else x01[..., 2]
        xy = np.stack([ca, cb], -1)
        for l in range(L):
            c = warp_counts(cells(gd, l, xy))
            tot_d += c
            print(f"  plane {p} level {l:2d} res {int(gd.resolution[l]):5d}  {c[0]:5.2f}  {c[1]:6.2f}  {c[2]:6.2f}")
    print(f"  total                {tot_d[0]:7.1f}  {tot_d[1]:8.1f}  {tot_d[2]:10.1f}")


if __name__ == "__main__":
    main()
