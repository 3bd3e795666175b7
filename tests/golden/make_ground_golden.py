"""Generate tests/golden/ground_ref.npz: every stage of the reference's own, unmodified utils/misc.py point_removal
(range_filter, Open3D's remove_statistical_outlier, six my_ransac calls, the ground split, the second outlier removal)
and of Trainer.process_pointcloud (model/runner.py), for tests/test_ground_oracle.py (CPU) and
tests/test_gpu_ground.py (the CUDA ops against the reference).

Run where the reference checkout exists (CPU only, about a minute):
    python tests/golden/make_ground_golden.py [OUT.npz]          # LIDAR4D_REFERENCE = checkout (default /root/reference)

Open3D is replaced by tests/open3d_stub.py, whose outlier rule is oracle/ground_oracle.py's statement of Open3D's
(Open3D is not a dependency of this project).  The global `random` is seeded per case.  What is recorded, per case:
  rf_keep            rows of the cloud range_filter keeps (the cloud is passed with its row index as a fourth column,
                     which range_filter carries along);
  sor1_keep/sor2_keep  the kept indices of the two outlier removals, as the stub returned them to the reference;
  ransac_counts_<j>  the inlier count of every hypothesis my_ransac call j scored, read from its own np.sum;
  ground             indices (into the cloud after the first outlier removal) of the points returned as ground;
  rng_state          random.getstate()[1] after point_removal.
Index sets are stored as packed bit masks over their parent cloud (ground_cases.pack).  The reference's outputs themselves are checked against those indices before anything is written.  Cases: two 66 x 1030
sweeps rebuilt from seeds (tests/ground_cases.py, stored as SHA-256) and three small stored clouds; `chain_*`: one
process_pointcloud run on a 16 x 256 range image with a pose, for the float32 and the float16 images, with the
unprojected cloud point_removal received (`chain_*_pc_raw`)."""
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)
REF = os.environ.get("LIDAR4D_REFERENCE", "/root/reference")

import ground_cases as GC  # noqa: E402
import open3d_stub  # noqa: E402

CASE_SEEDS = {"sweep_a": 101, "sweep_b": 102, "small70": 103, "small200": 104, "dup": 105}
CHAIN = dict(H=16, W=256, scale=0.01, num_frames=51, time=0.46, seed=106)


class _CountingNumpy(types.ModuleType):
    """NumPy as misc.py sees it, with np.sum over boolean arrays (my_ransac's inlier count, misc.py:93) recorded."""

    def __init__(self, log):
        super().__init__("numpy")
        self._log = log

    def __getattr__(self, name):
        return getattr(np, name)

    def sum(self, a, *args, **kw):
        r = np.sum(a, *args, **kw)
        if isinstance(a, np.ndarray) and a.dtype == bool:
            self._log.append(int(r))
        return r


def reference_misc():
    """The reference's utils/misc.py with the Open3D stub (also when another test imported it with a bare stub)."""
    o3d = open3d_stub.install()
    if REF not in sys.path:
        sys.path.insert(0, REF)
    sys.dont_write_bytecode = True
    import utils.misc as misc
    misc.o3d = o3d
    return misc


def run_reference(misc, pc, seed):
    """point_removal on float32 pc [N, 3] -> dict of recorded stages (see the module docstring)."""
    random.seed(seed)
    open3d_stub.calls.clear()
    counts, inliers = [], []
    np_proxy = _CountingNumpy(counts)
    orig_np, orig_ransac = misc.np, misc.my_ransac

    def ransac(*a, **k):
        start = len(counts)
        out = orig_ransac(*a, **k)
        inliers.append(out[0])
        ransac_counts.append(counts[start:])
        return out
    ransac_counts = []
    tagged = np.concatenate([pc, np.arange(len(pc), dtype=np.float32)[:, None]], 1)
    rf = misc.range_filter(tagged)
    rf_keep = rf[:, 3].astype(np.int64)
    assert np.array_equal(rf[:, :3], pc[rf_keep])
    misc.np, misc.my_ransac = np_proxy, ransac
    try:
        points, ground = misc.point_removal(pc)
    finally:
        misc.np, misc.my_ransac = orig_np, orig_ransac
    state = random.getstate()
    assert len(open3d_stub.calls) == 2 and len(inliers) == 6
    sor1, sor2 = open3d_stub.calls
    pc1 = pc[rf_keep].astype(np.float64)[sor1]
    union = np.unique(np.concatenate(inliers))
    g = union[pc1[union, 2] < -1]
    assert np.array_equal(ground, pc1[g])
    rest = np.delete(pc1, g, axis=0)
    assert np.array_equal(points, rest[sor2])
    return {"rf_keep": rf_keep, "sor1_keep": sor1, "ground": g, "sor2_keep": sor2, "ransac_counts": ransac_counts,
            "rng_state": np.array(state[1], np.uint32), "points": points, "ground_points": ground}


def chain_inputs():
    """A 16 x 256 range image of the same scene, with ray drops, its pose and time: images_lidar [1, H, W, 3] float32
    (raydrop mask, intensity, depth * scale), poses_lidar [1, 4, 4] float32, time [1, 1] float32."""
    H, W, s = CHAIN["H"], CHAIN["W"], CHAIN["scale"]
    rng = np.random.default_rng(CHAIN["seed"])
    t = GC.ranges(GC.directions(H, W), rng)
    t = np.where(np.isfinite(t) & (t < 80), t, 0.0).reshape(H, W)
    drop = (rng.random((H, W)) < 0.1) | (t == 0)
    img = np.stack([(~drop).astype(np.float32), rng.random((H, W)).astype(np.float32), (t * s).astype(np.float32)], -1)
    a = 0.3
    pose = np.array([[np.cos(a), -np.sin(a), 0, 12.5], [np.sin(a), np.cos(a), 0, -3.25], [0, 0, 1, 0.8], [0, 0, 0, 1]],
                    np.float32)
    return img[None], pose[None], np.array([[CHAIN["time"]]], np.float32)


def run_chain(misc, dtype):
    """Trainer.process_pointcloud of the reference, unbound, on one frame."""
    import torch
    from ref_stubs import install_reference_stubs
    install_reference_stubs()
    reference_misc()
    import model.runner as runner
    seen = []

    def point_removal(pc):
        seen.append(np.array(pc))
        return misc.point_removal(pc)
    runner.point_removal = point_removal
    img, pose, tm = chain_inputs()
    images = torch.from_numpy(img).to(dtype)
    data = {"images_lidar": images, "poses_lidar": torch.from_numpy(pose), "time": torch.from_numpy(tm)}

    class Loader(list):
        _data = types.SimpleNamespace(intrinsics_lidar=list(GC.K))      # a list of Python floats, as the dataset's
    me = types.SimpleNamespace(opt=types.SimpleNamespace(scale=CHAIN["scale"], num_frames=CHAIN["num_frames"]),
                               log=lambda *a: None)
    random.seed(CHAIN["seed"])
    runner.Trainer.process_pointcloud(me, Loader([data]))
    runner.point_removal = misc.point_removal
    (key, pts), = me.pc_list.items()
    return key, pts, me.pc_ground_list[key], seen[0]


def main(out_path):
    import scipy
    misc = reference_misc()
    fx = {"numpy_version": np.array(np.__version__), "scipy_version": np.array(scipy.__version__)}
    clouds = {name: GC.sweep(seed, tilt=tilt) for name, (seed, tilt) in GC.SWEEPS.items()}
    for name, pts in clouds.items():
        fx[f"{name}_sha256"] = np.array(GC.digest(pts))
    for name, pts in GC.small_clouds(np.random.default_rng(2025)).items():
        clouds[name] = pts
        fx[f"{name}_points"] = pts
    for name, pts in clouds.items():
        seed = CASE_SEEDS[name]
        r = run_reference(misc, pts, seed)
        fx[f"{name}_seed"] = np.array(seed, np.int64)
        sizes = {"rf_keep": len(pts), "sor1_keep": len(r["rf_keep"]), "ground": len(r["sor1_keep"]),
                 "sor2_keep": len(r["sor1_keep"]) - len(r["ground"])}
        for k, n in sizes.items():
            fx[f"{name}_{k}"] = GC.pack(r[k], n)
            assert np.array_equal(GC.unpack(fx[f"{name}_{k}"]), r[k])
        for j, c in enumerate(r["ransac_counts"]):
            fx[f"{name}_ransac_counts_{j}"] = np.asarray(c, np.int32)
        fx[f"{name}_rng_state"] = r["rng_state"]
        print(f"{name}: {len(pts)} points, range filter {len(r['rf_keep'])}, outliers 1 {len(r['sor1_keep'])}, ground "
              f"{len(r['ground'])}, outliers 2 {len(r['sor2_keep'])}, hypotheses {[len(c) for c in r['ransac_counts']]}")
    import torch
    for tag, dtype in (("f32", torch.float32), ("f16", torch.float16)):
        key, pts, ground, pc_raw = run_chain(misc, dtype)
        fx[f"chain_{tag}_pc_raw"] = pc_raw
        fx[f"chain_{tag}_key"] = np.array(key)
        fx[f"chain_{tag}_points"] = pts
        fx[f"chain_{tag}_ground"] = ground
        fx[f"chain_{tag}_rng_state"] = np.array(random.getstate()[1], np.uint32)
        assert pts.dtype == np.float64 and ground.dtype == np.float64
        print(f"chain {tag}: key {key}, {len(pts)} points, {len(ground)} ground")
    np.savez_compressed(out_path, **fx)
    print(f"wrote {out_path} ({os.path.getsize(out_path)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ground_ref.npz"))
