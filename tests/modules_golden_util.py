"""Shared by tests/golden/make_modules_golden.py, tests/test_modules_golden.py and tests/test_gpu_modules.py (test
infrastructure): the submodule calls of LiDAR4D whose reference results tests/golden/modules_ref.npz holds, their
inputs, and the oracle's restatement of each call.

Every call is written against the reference's module API (model.hash_encoder(x, t), model.planes_encoder(xt), ...), so
one function runs on the reference model on the tcnn shim, on the CUDA LiDAR4D, and - through `oracle_fn` - on the
oracle.  The loss of a call is sum_i <output_i, G_i> with seeded G_i; gradients of big tables are stored as fingerprints
(a projection and the L1 norm, float64)."""
import numpy as np
import torch

from oracle import lidar4d_oracle as O
from lidar4d_b200.geometry import FieldConfig, lagrange_basis, make_time_query

GOLDEN = "modules_ref.npz"
N = 16

SMALL = dict(min_resolution=8, base_resolution=16, max_resolution=512, time_resolution=8,
             n_levels_hash=4, log2_hashmap_size=12, num_frames=6, near_lidar=0.0105, far_lidar=0.851,
             hash_size_dynamic=(9, 8, 8), flow_base_resolution=8, flow_max_resolution=256,
             flow_log2_hashmap_size=10)
L8 = dict(n_levels_hash=8, num_frames=51, near_lidar=0.0105, far_lidar=0.851)     # the reference's defaults otherwise
CONFIGS = {"small": (SMALL, 31), "L8": (L8, 32)}


def config(name) -> FieldConfig:
    return FieldConfig(**CONFIGS[name][0])


def oracle(name) -> O.OracleLiDAR4D:
    """seeded parameters; MLP masters fp16-representable, so the fp32 reference and the fp16 working copies agree"""
    kw, seed = CONFIGS[name]
    return O.snap_mlp_weights_fp16(O.build_seeded(config(name), seed, flow_last_std=0.02))


def times(cfg: FieldConfig):
    """0 and 1 (single slice), a slice node, between nodes, and the neighbour times (k +- 1) / F of t = 0.4"""
    F = cfg.num_frames
    k = int(np.float32(np.float32(0.4) * np.float32(F - 1)))
    return [0.0, 1.0, 3 / 7, 0.4, (k + 1) / F, (k - 1) / F]


def inputs(cfg: FieldConfig, seed: int = 7):
    g = torch.Generator().manual_seed(seed)
    x3 = torch.rand(N, 3, generator=g)
    e = float(np.float32(1.0) - np.finfo(np.float32).eps)
    x3[0], x3[1], x3[2], x3[3], x3[4] = 0.0, 1.0, e, -0.03, 1.04          # edges and points outside [0, 1]
    x3[5] = torch.tensor([1.2, -0.2, 0.5])
    xt = torch.cat([x3, torch.rand(N, 1, generator=g)], -1)              # rows with their own times
    xt[0, 3], xt[1, 3], xt[2, 3], xt[3, 3] = 0.0, 1.0, e, 1.05
    return {
        "x3": x3, "x2": x3[:, :2].clone(), "xt": xt, "d01": torch.rand(N, 3, generator=g),
        "feat": torch.randn(N, cfg.sigma_in_dim, generator=g) * 0.5,
        "attr": torch.randn(N, cfg.attr_in_dim, generator=g) * 0.5,
    }


def flow_xt(inp, t):
    """flow_net input: row 0 carries t, the other rows other times (flow_field.py:122 takes row 0's for all)"""
    xt = inp["xt"].clone()
    xt[0, 3] = float(np.float32(t))
    return xt


def _tt(t):
    return torch.tensor(t, dtype=torch.float32)


def dyn_names(cfg, planes=(0, 1, 2)):
    return [f"hash_encoder.hash_dynamic.{p}.hash_t.{s}.params" for p in planes for s in range(cfg.time_resolution)]


def plane_names(cfg, cis=range(6)):
    return [f"planes_encoder.planes.{s}.{c}" for s in range(cfg.n_levels_plane) for c in cis]


FLOW_NAMES = ["flow_net.grid_enc.params", "flow_net.mlp.0.weight", "flow_net.mlp.2.weight", "flow_net.mlp.4.weight"]


def calls(cfg: FieldConfig):
    """(key, fn(model, inputs) -> list of outputs, parameter names, differentiable input or None).  t-dependent calls
    appear once per time of times(cfg)."""
    T = cfg.time_resolution
    out = [
        ("hash_static", lambda m, i: [m.hash_encoder.hash_static(i["x3"])], ["hash_encoder.hash_static.params"], None),
        ("hash_slice0", lambda m, i: [m.hash_encoder.hash_dynamic[0].hash_t[0](i["x2"])],
         ["hash_encoder.hash_dynamic.0.hash_t.0.params"], None),
        (f"hash_slice{T - 1}", lambda m, i: [m.hash_encoder.hash_dynamic[2].hash_t[T - 1](i["x2"])],
         [f"hash_encoder.hash_dynamic.2.hash_t.{T - 1}.params"], None),
        ("planes", lambda m, i: list(m.planes_encoder(i["xt"])), plane_names(cfg), "xt"),
        ("flow_grid", lambda m, i: [m.flow_net.grid_enc(i["x3"])], ["flow_net.grid_enc.params"], None),
        ("view", lambda m, i: [m.view_encoder(i["d01"])], [], None),
        ("sigma_net", lambda m, i: [m.sigma_net(i["feat"])], ["sigma_net.params"], "feat"),
        ("intensity_net", lambda m, i: [m.intensity_net(i["attr"])], ["intensity_net.params"], "attr"),
        ("raydrop_net", lambda m, i: [m.raydrop_net(i["attr"])], ["raydrop_net.params"], "attr"),
    ]
    for j, t in enumerate(times(cfg)):
        out += [
            (f"hash_encoder_t{j}", lambda m, i, t=t: list(m.hash_encoder(i["x3"], _tt(t))),
             ["hash_encoder.hash_static.params"] + dyn_names(cfg), None),
            (f"hash_dynamic1_t{j}", lambda m, i, t=t: [m.hash_encoder.hash_dynamic[1](i["x3"][:, [0, 2]], _tt(t))],
             dyn_names(cfg, (1,)), None),
            (f"flow_net_t{j}", lambda m, i, t=t: [m.flow_net(flow_xt(i, t))], FLOW_NAMES, None),
        ]
    return out


class OracleModules:
    """The reference's module API on the oracle's functions (the restatement the golden file pins)."""

    def __init__(self, orc: O.OracleLiDAR4D):
        self.o = orc

    def call(self, key, i):
        o, c = self.o, self.o.cfg
        L = c.n_levels_hash
        tq = lambda t: make_time_query(np.float32(t), c.time_resolution)
        if key == "hash_static":
            return [o.hash_static(i["x3"])]
        if key.startswith("hash_slice"):
            k = int(key[len("hash_slice"):])
            p = 0 if k == 0 else 2
            return [O.hash_encode(i["x2"], o.p(f"hash_encoder.hash_dynamic.{p}.hash_t.{k}.params"), o.g_dynamic[p])]
        if key == "planes":
            return [o.planes(i["xt"], "static"), o.planes(i["xt"], "dynamic")]
        if key == "flow_grid":
            return [O.hash_encode(i["x3"], o.p("flow_net.grid_enc.params"), o.g_flow)]
        if key == "view":
            return [O.frequency_encode(i["d01"], c.view_degree)]
        if key == "sigma_net":
            return [O.fused_mlp(i["feat"], o.p("sigma_net.params"), c.sigma_in_dim, 16, 64, 1, o.mlp_dtype)]
        if key in ("intensity_net", "raydrop_net"):
            return [O.fused_mlp(i["attr"], o.p(f"{key}.params"), c.attr_in_dim, 1, 64, 2, o.mlp_dtype)]
        t = times(c)[int(key.rsplit("_t", 1)[1])]
        if key.startswith("hash_encoder"):
            return [o.hash_static(i["x3"]), o.hash_dynamic(i["x3"], tq(t))]
        if key.startswith("hash_dynamic1"):
            return [o.hash_dynamic(i["x3"], tq(t))[:, L:2 * L]]
        if key.startswith("flow_net"):
            xt = flow_xt(i, t)
            return [o.flow_field(xt[:, :3], lagrange_basis(np.float32(xt[0, 3])))]
        raise KeyError(key)


def upstream(outs, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(o.shape, generator=g) for o in outs]


def fingerprint(g: torch.Tensor) -> np.ndarray:
    v = g.detach().double().reshape(-1).cpu().numpy()
    return np.array([float(v @ O.projection_vector(v.size)), float(np.abs(v).sum())])


def fp_close(a, b, tol) -> bool:
    """fingerprints agree: the projections within tol of the L1 norm, the L1 norms relatively"""
    scale = max(abs(b[1]), 1e-30)
    return abs(a[0] - b[0]) <= tol * scale and abs(a[1] - b[1]) <= tol * scale
