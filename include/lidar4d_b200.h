/*
 * lidar4d_b200.h - C-ABI of the H100 (sm_90a) LiDAR4D hot-path library
 * (liblidar4d_b200.so).  Plain C: pointers, sizes, POD structs; no torch / ATen
 * types cross this boundary.
 *
 * What it replaces (paths relative to the reference checkout):
 *   - the tiny-cuda-nn plugin surface used by the hot path
 *       tcnn.Encoding(HashGrid)   model/hash_field.py:47-57, :107-117; model/flow_field.py:67-77
 *       tcnn.Encoding(Frequency)  model/lidar4d.py:68-74
 *       tcnn.Network(FullyFusedMLP) model/lidar4d.py:83-117
 *   - the PyTorch op graph around it
 *       LiDAR_Renderer.run        model/renderer.py:44-140   (sampling, compositing)
 *       LiDAR4D.density/attribute model/lidar4d.py:139-223
 *       LiDAR4D.flow              model/lidar4d.py:124-137
 *       Planes4D / F.grid_sample  model/planes_field.py:56-141
 *       HashGrid4D / HashGridT    model/hash_field.py:65-88, :141-172
 *       FlowField                 model/flow_field.py:102-130
 *   - error convention: unlike the reference's chamfer plugin (utils/chamfer3D/chamfer3D.cu:144-150,
 *     printf + ignored return), every entry point returns 0 on success and a negative L4D_E* code
 *     on failure; l4d_last_error() gives the message; nothing throws or aborts across the ABI.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless named host_*; the caller owns every buffer
 *     (inputs, outputs, workspaces, gradients); the library allocates nothing on the hot path.
 *   - all work is enqueued on the caller's stream (`stream` = cudaStream_t cast to void*); no
 *     device synchronisation inside; re-entrant (no global state except the thread-local error string).
 *   - host-side decisions (frame index, first/last-frame branches, time-slice indices, Lagrange
 *     bases) arrive pre-computed in L4DFrame so that no device->host sync is needed
 *     (the reference syncs at lidar4d.py:143, hash_field.py:82, lidar4d.py:201).
 *   - level geometry (scale/resolution/entries) arrives as data in L4DGrid so that hash
 *     indices are bit-exact with whatever computed that geometry.
 */
#ifndef LIDAR4D_B200_H_
#define LIDAR4D_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define L4D_ABI_VERSION 1
#define L4D_MAX_LEVELS 16
#define L4D_MAX_PLANE_SCALES 4
#define L4D_MAX_TIME_SLICES 16
#define L4D_HIDDEN 64

enum {
  L4D_OK = 0,
  L4D_EINVAL = -1,   /* bad argument / unsupported configuration */
  L4D_ECUDA = -2,    /* a CUDA runtime call or launch failed      */
  L4D_ESIZE = -3     /* caller-provided buffer too small          */
};

/* One multi-resolution hash grid (one tcnn HashGrid encoding). */
typedef struct L4DGrid {
  uint32_t n_dims;        /* 2 or 3 */
  uint32_t n_levels;      /* <= L4D_MAX_LEVELS */
  uint32_t n_features;    /* 4 (hash_static / hash_dynamic) or 8 (flow) */
  uint32_t reserved;
  float    scale[L4D_MAX_LEVELS];
  uint32_t resolution[L4D_MAX_LEVELS];
  uint32_t entries[L4D_MAX_LEVELS];       /* hashmap_size of the level */
  uint32_t offset[L4D_MAX_LEVELS + 1];    /* first entry of the level; offset[n_levels] = total entries */
} L4DGrid;

/* Model hyper-parameters (LiDAR4D.__init__, model/lidar4d.py:23-45). */
typedef struct L4DConfig {
  L4DGrid  hash_static;          /* 3D, F=4 */
  L4DGrid  hash_dynamic[3];      /* 2D xy / xz / yz, F=4; one table per time slice */
  L4DGrid  flow;                 /* 3D, F=8 */
  uint32_t n_plane_scales;       /* 4 */
  uint32_t plane_res[L4D_MAX_PLANE_SCALES];  /* spatial resolution per scale (32,64,128,256) */
  uint32_t time_resolution;      /* 8: time planes' H and number of hash time slices */
  uint32_t num_frames;
  uint32_t active_sensor;        /* renderer.py:101 */
  uint32_t view_degree;          /* 12 */
  uint32_t sigma_in_dim;         /* 120 */
  uint32_t sigma_in_pad;         /* 128 */
  uint32_t attr_in_dim;          /* 87 */
  uint32_t attr_in_pad;          /* 96 */
  float    bound;
  float    near_lidar;
  float    far_lidar;
  float    density_scale;
  uint32_t mlp_fp16;             /* 1: MLP weights are consumed as fp16-rounded working copies (as tcnn's half
                                    params) and the dense kernels run on wgmma tensor cores; 0: fp32 FMA */
  uint32_t reserved;
} L4DConfig;

/* One (.,tau) query of the time-sliced grids (model/hash_field.py:76-88). */
typedef struct L4DTimeQuery {
  float    tau;
  uint32_t slice_lo, slice_hi;
  float    w_lo, w_hi;           /* (idx2-idx), (idx-idx1) */
  uint32_t single;               /* idx1==idx2: feature = G_lo only */
  float    basis[4];             /* cubic Lagrange basis at tau (hash_field.py:65-74) */
} L4DTimeQuery;

/* Per-frame constants decided on the host (model/lidar4d.py:143,157-173). */
typedef struct L4DFrame {
  float        time;
  uint32_t     frame_idx;
  uint32_t     has_fwd, has_bwd;
  L4DTimeQuery cur, fwd, bwd;
  float        flow_basis[4];    /* Lagrange basis at `time` (flow_field.py:102-111,122) */
} L4DFrame;

/* fp32 master parameters in the reference's state_dict layouts (SURVEY.md 8(b)). */
typedef struct L4DMasterParams {
  const float* hash_static;                                     /* hash_encoder.hash_static.params */
  const float* hash_dynamic[3][L4D_MAX_TIME_SLICES];            /* hash_encoder.hash_dynamic.P.hash_t.S.params */
  const float* flow_grid;                                       /* flow_net.grid_enc.params */
  const float* planes[L4D_MAX_PLANE_SCALES][6];                 /* planes_encoder.planes.S.C  [1,8,H,W] */
  const float* sigma_net;                                       /* [64*in_pad + 16*64] */
  const float* intensity_net;                                   /* [64*96 + 64*64 + 16*64] */
  const float* raydrop_net;
  const float* flow_mlp[3];                                     /* flow_net.mlp.{0,2,4}.weight */
} L4DMasterParams;

/* fp32 gradient buffers, same layouts as L4DMasterParams (accumulated into). */
typedef struct L4DMasterGrads {
  float* hash_static;
  float* hash_dynamic[3][L4D_MAX_TIME_SLICES];
  float* flow_grid;
  float* planes[L4D_MAX_PLANE_SCALES][6];
  float* sigma_net;
  float* intensity_net;
  float* raydrop_net;
  float* flow_mlp[3];
} L4DMasterGrads;

/* Ray batch + sampling arguments of LiDAR_Renderer.run (model/renderer.py:44-89). */
typedef struct L4DRays {
  const float* rays_o;      /* [n_rays,3] */
  const float* rays_d;      /* [n_rays,3] */
  uint32_t     n_rays;
  uint32_t     n_steps;     /* num_steps (768), in [2, 8192]: the reference renders nothing at 1 (empty deltas) */
  uint32_t     perturb;     /* z jitter on/off */
  uint32_t     reserved;
  uint64_t     seed;        /* counter-based jitter stream: u = f(seed, ray_offset+ray, sample) */
  uint64_t     ray_offset;  /* global index of ray 0 (rank-independent streams under ray sharding) */
} L4DRays;

int         l4d_abi_version(void);
const char* l4d_last_error(void);

/* --- parameter staging: fp32 masters -> kernel working set (fp16 tables, channels-last planes,
 *     MLP weights in both orientations).  Call after every optimiser step. ------------------- */
size_t l4d_staged_bytes(const L4DConfig* cfg);
int    l4d_stage_params(const L4DConfig* cfg, const L4DMasterParams* master,
                        void* staged, size_t staged_bytes, void* stream);

/* Same, selectively: L4D_STAGE_TABLES = the three hash-table groups (fp16 casts / slice-pair packing),
 * L4D_STAGE_SMALL = planes (channels-last), MLP working copies and tensor-core operand copies - ONE launch for all of
 * them.  `staged` must have been zero-filled once when it was allocated (operand padding is never rewritten).
 * After l4d_adam_step with a `master` table only L4D_STAGE_SMALL is left to do. */
#define L4D_STAGE_TABLES 1u
#define L4D_STAGE_SMALL  2u
int    l4d_stage_params_ex(const L4DConfig* cfg, const L4DMasterParams* master,
                           void* staged, size_t staged_bytes, uint32_t what, void* stream);

/* --- optimiser step (SURVEY.md 8(f) #4; replaces torch.optim.Adam of main_lidar4d.py:298-300 + the re-staging pass) -----
 * Adam (no weight decay, no amsgrad) over FLAT fp32 arenas: params, grads and the two moment buffers hold every tensor
 * of the hot path at the same offsets (each tensor starts on a multiple of L4D_ADAM_CHUNK floats).  params, exp_avg and
 * exp_avg_sq come out bit-identical to torch 2.11's fused Adam (torch._fused_adam_ with state_steps = step), including
 * its fp32 bias corrections, for every input.  `groups` = sorted, disjoint [begin,end) float ranges with their learning
 * rate (the reference's param groups, lidar4d.py:226-237); ranges not covered are left alone.  grads are MULTIPLIED by
 * inv_scale (1/loss-scale) on the fly, which equals torch's division by grad_scale exactly when the scale is a power of
 * two (all GradScaler produces); grads are not written back unscaled.  zero_grad=1 clears the covered ranges of grads in
 * the same pass.  If `master` is given (pointers INTO `params`),
 * a group that is exactly one hash table also emits that table's fp16 working copy into `staged` (static / flow: cast;
 * dynamic slice t: the lo half of pair t and the hi half of pair t-1), i.e. l4d_stage_params_ex(L4D_STAGE_TABLES) for free. */
#define L4D_ADAM_CHUNK 1024
#define L4D_ADAM_MAX_SEGMENTS 64
typedef struct L4DAdamGroup {
  uint64_t begin, end;     /* floats, relative to the arena start; begin % L4D_ADAM_CHUNK == 0, end % 4 == 0 */
  float    lr;
  uint32_t reserved;
} L4DAdamGroup;
int    l4d_adam_step(const L4DConfig* cfg, float* params, float* grads, float* exp_avg, float* exp_avg_sq,
                     uint64_t n_floats, const L4DAdamGroup* groups, uint32_t n_groups,
                     float beta1, float beta2, float eps, uint32_t step, float inv_scale, uint32_t zero_grad,
                     const L4DMasterParams* master_or_null, void* staged_or_null, size_t staged_bytes, void* stream);

/* --- LiDAR_Renderer.run forward (renderer.py:44-140 + lidar4d.py:139-223), one fused kernel.
 *     depth[n], image[n,2] (ch0 raydrop, ch1 intensity), wsum[n]; weights/z_vals [n,S] optional.
 *     `saved` (l4d_saved_bytes) enables a later backward; NULL = inference through the single kernel.
 *     With `saved` the split pipeline runs: the buffer is also its exchange workspace and receives the
 *     launch's contracted tables (dynamic hash x time constants of `frame`, time-plane rows) - the
 *     backward must be called with the same saved / frame / rays / staged as its forward. -------- */
size_t l4d_saved_bytes(const L4DConfig* cfg, uint32_t n_rays, uint32_t n_steps);
int    l4d_render_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                          const L4DRays* rays, float* depth, float* image, float* wsum,
                          float* weights_or_null, float* zvals_or_null,
                          void* saved_or_null, size_t saved_bytes, void* stream);

/* --- backward of the above: upstream grads g_depth[n], g_image[n,2], optional g_wsum[n],
 *     g_weights[n,S].  Hash-table gradients are accumulated straight into `grads`; plane and
 *     MLP gradients into `grad_work` (zero it ONCE after allocating it: every kernel that consumes a
 *     region - l4d_unstage_grads, the fold kernels of the slice- / basis- / time-row-independent
 *     accumulators it also holds - clears it again) and folded into `grads` by l4d_unstage_grads.
 *     One grad_work per stream that runs backwards concurrently. ------------------------------ */
size_t l4d_grad_work_bytes(const L4DConfig* cfg);
int    l4d_render_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                           const L4DRays* rays, const void* saved, size_t saved_bytes,
                           const float* g_depth, const float* g_image,
                           const float* g_wsum_or_null, const float* g_weights_or_null,
                           const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes,
                           void* stream);
/* Same; additionally records the CUDA event `ev_hash_done_or_null` (a cudaEvent_t) on `stream` at the point from which the
 * hash_static / hash_dynamic gradient buffers are final (after the static scatter and the dynamic fold, before the flow
 * backward): a data-parallel caller starts all-reducing that bucket - 60 % of the gradient bytes - on a side stream while the
 * rest of the backward still runs (lidar4d_b200/parallel.py). */
int    l4d_render_backward_ex(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                              const L4DRays* rays, const void* saved, size_t saved_bytes,
                              const float* g_depth, const float* g_image,
                              const float* g_wsum_or_null, const float* g_weights_or_null,
                              const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes,
                              void* ev_hash_done_or_null, void* stream);
/* The compositing backward of the tensor-core split pipeline alone (the first kernel l4d_render_backward runs there), on
 * the saved buffer of a training forward: afterwards feature columns 0..3 of the saved dL/dfeature hold dL/dsigma,
 * dL/da0, dL/da1 and the attribute mask (0 / 1) of every sample.  Tensor-core configurations only (L4D_EINVAL else). */
/* --- the same forward / backward over rays of SEVERAL frames in one launch (a training batch drawn across frames).
 *     Ray r of the launch belongs to frame frames[(first_ray_phase + r) / rays_per_frame]; the phase lets a launch start
 *     in the middle of a frame's rays.  Every frame gets its own contracted tables in `saved`
 *     (l4d_saved_bytes_frames(cfg, n_rays, n_steps, n_frames) bytes) and its own slice- / basis- / time-row-independent
 *     accumulators in `grad_work` (l4d_grad_work_bytes_frames(cfg, n_frames) bytes, zero-filled once like the single-frame
 *     buffer; the per-frame folds clear it again).  A ray's jitter stream is ray_offset + r, as for one frame, so a launch
 *     over B frames of N rays renders what B single-frame launches with ray_offset + b * N render, bit for bit.
 *     With n_frames = 1 the buffers and the results are those of l4d_render_forward / l4d_render_backward_ex, which are
 *     this call with a one-frame table.  L4D_EINVAL: n_frames = 0 or > L4D_MAX_FRAMES, rays_per_frame = 0,
 *     first_ray_phase >= rays_per_frame, or first_ray_phase + n_rays > n_frames * rays_per_frame.  The backward must be
 *     called with the same table as its forward.  The *_bytes_frames functions return 0 on a bad n_frames. */
#define L4D_MAX_FRAMES 16
typedef struct L4DFrameTable {
  uint32_t n_frames;           /* 1 .. L4D_MAX_FRAMES */
  uint32_t rays_per_frame;
  uint32_t first_ray_phase;    /* < rays_per_frame */
  uint32_t reserved;
  L4DFrame frames[L4D_MAX_FRAMES];
} L4DFrameTable;
size_t l4d_saved_bytes_frames(const L4DConfig* cfg, uint32_t n_rays, uint32_t n_steps, uint32_t n_frames);
size_t l4d_grad_work_bytes_frames(const L4DConfig* cfg, uint32_t n_frames);
int    l4d_render_forward_frames(const L4DConfig* cfg, const void* staged, const L4DFrameTable* frames,
                                 const L4DRays* rays, float* depth, float* image, float* wsum,
                                 float* weights_or_null, float* zvals_or_null,
                                 void* saved_or_null, size_t saved_bytes, void* stream);
int    l4d_render_backward_frames(const L4DConfig* cfg, const void* staged, const L4DFrameTable* frames,
                                  const L4DRays* rays, const void* saved, size_t saved_bytes,
                                  const float* g_depth, const float* g_image,
                                  const float* g_wsum_or_null, const float* g_weights_or_null,
                                  const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes,
                                  void* ev_hash_done_or_null, void* stream);
int    l4d_composite_backward(const L4DConfig* cfg, const L4DRays* rays, void* saved, size_t saved_bytes,
                              const float* g_depth, const float* g_image,
                              const float* g_wsum_or_null, const float* g_weights_or_null, void* stream);
int    l4d_unstage_grads(const L4DConfig* cfg, const void* grad_work, size_t grad_work_bytes,
                         const L4DMasterGrads* grads, void* stream);

/* --- LiDAR4D.flow (lidar4d.py:124-137): x[q,3] in [-bound,bound] -> flow[q,6].
 *     flow_saved (q*16 floats) enables the backward. ------------------------------------------ */
int    l4d_flow_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                        const float* x, uint32_t n_points, float* flow,
                        float* flow_saved_or_null, void* stream);
int    l4d_flow_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                         const float* x, uint32_t n_points, const float* flow_saved,
                         const float* g_flow, const L4DMasterGrads* grads,
                         void* grad_work, size_t grad_work_bytes, void* stream);

/* --- parity / debug entry points (not on the hot path) -------------------------------------- */
/* grid_id: 0 static, 1..3 dynamic xy/xz/yz, 4 flow.  x[n,D] -> idx[n,2^D] (uint32, modulo the
 * level's entries), w[n,2^D]. */
int    l4d_hash_indices(const L4DConfig* cfg, uint32_t grid_id, uint32_t level,
                        const float* x, uint32_t n, uint32_t* idx, float* w, void* stream);
/* LiDAR4D.density on explicit points x[n,3] in [-bound,bound]: sigma[n], geo[n,15],
 * optional features[n,sigma_in_dim] and flow[n,6]. */
int    l4d_density_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                           const float* x, uint32_t n, float* sigma, float* geo,
                           float* features_or_null, float* flow_or_null, void* stream);

/* LiDAR4D.attribute (lidar4d.py:191-223) on explicit points: unit directions d[n,3], geo_feat[n,15],
 * optional mask[n] (uint8, 0 = row stays zero) -> out[n,2] = (raydrop, intensity) after the sigmoid. */
int    l4d_attribute_forward(const L4DConfig* cfg, const void* staged, const float* d, const float* geo,
                             const unsigned char* mask_or_null, uint32_t n, float* out, void* stream);

/* --- LiDAR4D.density / .attribute on explicit points WITH a backward (the reference's field methods are differentiable;
 *     a LiDAR_Renderer subclass that samples its own points builds its loss on them).  Gradients reach every parameter the
 *     reference's autograd graph reaches; none flows to x or d.  Same conventions as the render entry points: caller-owned
 *     buffers, the caller's stream, L4D_EINVAL / L4D_ESIZE for null or short buffers, n == 0 is a no-op; the backwards
 *     ACCUMULATE (hash tables straight into `grads`, planes and MLP weights into `grad_work`) and the caller runs
 *     l4d_unstage_grads afterwards.
 * l4d_density_forward_ex: l4d_density_forward (sigma / geo / features / flow bit for bit the same) that also writes what the
 *     backward needs into `saved` (l4d_density_saved_bytes(cfg, n) bytes: the flow-MLP inputs, the sigma-MLP input
 *     features and the backward's scratch).  saved_or_null = NULL is l4d_density_forward.
 * l4d_density_backward: upstream g_sigma[n] and / or g_geo[n,15] (NULL = zero) with the saved buffer, frame and x of its
 *     forward.  Every gradient buffer of `grads` must be set.
 * l4d_attribute_backward: upstream g_out[n,2] of l4d_attribute_forward with the same d / geo / mask (nothing is saved:
 *     the heads are recomputed).  Writes g_geo[n,15] when not NULL (zero outside the mask); only the intensity_net and
 *     raydrop_net buffers of `grads` are used (and must be set). */
size_t l4d_density_saved_bytes(const L4DConfig* cfg, uint32_t n);
int    l4d_density_forward_ex(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                              const float* x, uint32_t n, float* sigma, float* geo,
                              float* features_or_null, float* flow_or_null,
                              void* saved_or_null, size_t saved_bytes, void* stream);
int    l4d_density_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame,
                            const float* x, uint32_t n, const void* saved, size_t saved_bytes,
                            const float* g_sigma_or_null, const float* g_geo_or_null,
                            const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes, void* stream);
int    l4d_attribute_backward(const L4DConfig* cfg, const void* staged, const float* d, const float* geo,
                              const unsigned char* mask_or_null, uint32_t n, const float* g_out,
                              float* g_geo_or_null, const L4DMasterGrads* grads,
                              void* grad_work, size_t grad_work_bytes, void* stream);

/* --- LiDAR4D's submodules called on their own (hash_field.py, planes_field.py, flow_field.py, the tcnn encodings and
 *     networks): inputs row-major fp32 in [0,1] (no bound normalisation; points outside are encoded as tcnn and
 *     grid_sample encode them), outputs row-major fp32, the staged working set of the render path (fp16 tables, MLP
 *     working copies of the precision mode).  Both families: null or not 4-byte aligned pointers, an unknown module / net
 *     or n > 2^31: L4D_EINVAL; n == 0 is a no-op without a launch; one launch on `stream`.  The backwards ACCUMULATE
 *     (hash tables straight into `grads`, planes and MLP weights into `grad_work`; the caller runs l4d_unstage_grads).
 * l4d_encoder_forward(module, query, slice, x[n, in], out[n, out]); (in -> out) per module, L = hash levels, S = plane
 *     scales:
 *       L4D_MOD_HASH_STATIC      x[n,3]  -> [n, 4L]    hash_encoder.hash_static
 *       L4D_MOD_HASH_T0 + p      x[n,2]  -> [n, L]     hash_encoder.hash_dynamic[p] at `query` (p: 0 xy, 1 xz, 2 yz)
 *       L4D_MOD_HASH_DYNAMIC     x[n,3]  -> [n, 3L]    hash_encoder.forward_dynamic at `query`
 *       L4D_MOD_HASH_SLICE0 + p  x[n,2]  -> [n, 4L]    hash_encoder.hash_dynamic[p].hash_t[slice]
 *       L4D_MOD_PLANES_STATIC    xt[n,4] -> [n, 8S]    planes_encoder.forward_static
 *       L4D_MOD_PLANES_DYNAMIC   xt[n,4] -> [n, 8S]    planes_encoder.forward_dynamic (time = column 3 of each row)
 *       L4D_MOD_FLOW_GRID        x[n,3]  -> [n, 64]    flow_net.grid_enc
 *       L4D_MOD_FLOW             xt[n,4] -> [n, 6]     flow_net; the time of EVERY row is xt[0,3], read on the device
 *       L4D_MOD_FREQ             v[n,3]  -> [n, 72]    view_encoder (degree 12)
 *     `query` is required by the two HASH_T / HASH_DYNAMIC kinds (ignored otherwise), `slice` < time_resolution by
 *     HASH_SLICE.
 * l4d_encoder_backward: upstream g_out[n, out] with the inputs of the forward.  Parameter gradients of the module; the
 *     planes also give dL/dxt into g_x[n,4] when it is not NULL (g_x must be NULL for every other module).  The FREQ
 *     encoding has no parameters (L4D_EINVAL).  The module's buffers of `grads` must be set.
 * l4d_mlp_forward(net, in[n, n_in], out[n, n_out]): net L4D_NET_SIGMA (n_in = sigma_in_dim, n_out = 16),
 *     L4D_NET_RAYDROP / L4D_NET_INTENSITY (n_in = attr_in_dim, n_out = 1: before LiDAR4D.attribute's sigmoid).  Inputs
 *     are padded with ones to the network width.
 * l4d_mlp_backward: upstream g_out[n, n_out]; weight gradients of the net, dL/din into g_in[n, n_in] when not NULL. */
#define L4D_MOD_HASH_STATIC    0u
#define L4D_MOD_HASH_T0        1u   /* 1..3 */
#define L4D_MOD_HASH_DYNAMIC   4u
#define L4D_MOD_HASH_SLICE0    5u   /* 5..7 */
#define L4D_MOD_PLANES_STATIC  8u
#define L4D_MOD_PLANES_DYNAMIC 9u
#define L4D_MOD_FLOW_GRID      10u
#define L4D_MOD_FLOW           11u
#define L4D_MOD_FREQ           12u
#define L4D_NET_SIGMA          0u
#define L4D_NET_RAYDROP        1u
#define L4D_NET_INTENSITY      2u
int    l4d_encoder_forward(const L4DConfig* cfg, const void* staged, uint32_t module, const L4DTimeQuery* query_or_null,
                           uint32_t slice, const float* x, uint32_t n, float* out, void* stream);
int    l4d_encoder_backward(const L4DConfig* cfg, const void* staged, uint32_t module, const L4DTimeQuery* query_or_null,
                            uint32_t slice, const float* x, uint32_t n, const float* g_out, float* g_x_or_null,
                            const L4DMasterGrads* grads, void* grad_work, size_t grad_work_bytes, void* stream);
int    l4d_mlp_forward(const L4DConfig* cfg, const void* staged, uint32_t net, const float* in, uint32_t n, float* out,
                       void* stream);
int    l4d_mlp_backward(const L4DConfig* cfg, const void* staged, uint32_t net, const float* in, uint32_t n,
                        const float* g_out, float* g_in_or_null, const L4DMasterGrads* grads, void* grad_work,
                        size_t grad_work_bytes, void* stream);

/* --- SURVEY 8(f) "next" row 1: the chamfer / nearest-neighbour op of utils/chamfer3D --------------------------
 * Replaces chamfer_cuda.cpp:17-32 `forward(xyz1,xyz2,dist1,dist2,idx1,idx2)` / `backward(...)` (kernels
 * chamfer3D.cu:11-133,154-174).  xyz1[b,n,3], xyz2[b,m,3] fp32 contiguous; dist1[b,n] = squared distance to the
 * nearest point of xyz2 and idx1[b,n] its index (the smallest index on ties), dist2/idx2 likewise for xyz2.
 * `work` = l4d_chamfer_work_bytes(b,n,m) scratch bytes.  backward ACCUMULATES into g_xyz1[b,n,3], g_xyz2[b,m,3]
 * (zero them first, as dist_chamfer_3D.py:66-70 does). */
size_t l4d_chamfer_work_bytes(uint32_t b, uint32_t n, uint32_t m);
int    l4d_chamfer_forward(const float* xyz1, const float* xyz2, uint32_t b, uint32_t n, uint32_t m,
                           float* dist1, float* dist2, int32_t* idx1, int32_t* idx2,
                           void* work, size_t work_bytes, void* stream);
int    l4d_chamfer_backward(const float* xyz1, const float* xyz2, uint32_t b, uint32_t n, uint32_t m,
                            const float* g_dist1, const float* g_dist2, const int32_t* idx1, const int32_t* idx2,
                            float* g_xyz1, float* g_xyz2, void* stream);

/* --- SURVEY 8(f) "next" row 2: the thin layers either side of the render kernels, one launch each ------------------------
 * l4d_lidar_rays replaces data/base_dataset.py:15-102 `get_lidar_rays` (+ the GT gather of kitti360_dataset.py:170-178):
 * pose = DEVICE [4][4] row-major cam2world; inds = n flat pixel ids row*W+col (NULL = all H*W pixels in order, n = H*W);
 * writes rays_o[n,3], rays_d[n,3] and, if gt != NULL, gt[n,C] = image[inds,C] (image = DEVICE [H*W,C]).
 * l4d_lidar_loss replaces model/runner.py:179-213 (default criteria: L1 depth, MSE intensity / raydrop, label smoothing):
 * ACCUMULATES the summed loss into *loss (zero it first) and writes d loss / d depth [n] and d loss / d image [n,2].
 * It is l4d_main_loss with the default criteria and no chamfer term (the same fixed-order sum, so the same bits on
 * every call); n = 0 adds nothing. */
int    l4d_lidar_rays(const float* pose, float fov_up, float fov, uint32_t H, uint32_t W, const long long* inds_or_null,
                      uint32_t n, const float* image_or_null, uint32_t C, float* rays_o, float* rays_d, float* gt_or_null,
                      void* stream);
int    l4d_lidar_loss(const float* depth, const float* image2, const float* gt3, uint32_t n, float alpha_d, float alpha_r,
                      float alpha_i, float smooth, float* loss, float* g_depth, float* g_image2, void* stream);

/* --- the rest of train_step: the patch losses (model/runner.py:278-369) and URF's line-of-sight loss (:255-276) ---------
 * Inputs are fp32 device arrays; gt3[n, 3] = (raydrop m, intensity, depth) as for l4d_lidar_loss.  Both WRITE the loss to
 * the device float *loss; sums are taken in a fixed order, so the same inputs give the same bits.  The backwards read the
 * incoming gradient from the device float *g_loss and WRITE their gradient.  Null pointers and bad sizes: L4D_EINVAL.
 * l4d_patch_loss: depth[n] read as n / (px*py) patches of px rows x py columns (get_lidar_rays' order), n % (px*py) == 0;
 *   pred = depth*m/scale, gt_d = gt_depth*m/scale.  Writes the branch's summed loss (criterion `crit` = L4D_GRAD_*, terms
 *   switched on by L4D_PATCH_* `flags`, weights alpha_*) and g_depth[n] = d loss / d depth.  px == 1 gives 0 and a zero
 *   gradient, as the reference's `patch_size_x > 1`.  One launch (one CTA).
 * l4d_patch_loss_backward: g_depth[n] = g_saved[n] * *g_loss (g_saved = the forward's g_depth).  One launch.
 * l4d_los_loss: weights[n, S], z_vals[n, S], n*S < 2^32, the host `eps` of the reference (0.02 * 0.1^min(step/iters, 1)).
 *   Writes 0.1*loss_empty + 0.1*loss_near; with no ray of gt depth > 0 that is the reference's inf / nan.  `work` =
 *   l4d_los_work_bytes() bytes (L4D_ESIZE when smaller), kept for the backward.  Two launches; the second re-reads
 *   [n, S] only when no sample lies outside its window (then max(distr) < its peak).
 * l4d_los_loss_backward: g_weights[n, S] = d loss / d weights times *g_loss, with the forward's inputs and `work`. */
#define L4D_GRAD_L1    0
#define L4D_GRAD_MSE   1
#define L4D_GRAD_HUBER 2
#define L4D_GRAD_BCE   3
#define L4D_GRAD_COS   4
#define L4D_PATCH_SOBEL     1u   /* 3x3 Sobel with zero padding instead of finite differences */
#define L4D_PATCH_GRAD      2u   /* grad_loss: the x-direction criterion, weight alpha_grad */
#define L4D_PATCH_GRAD_NORM 4u   /* grad_norm_smooth: mean(exp(-dx)) + mean(exp(-dy)), weight alpha_grad_norm */
#define L4D_PATCH_SPATIAL   8u   /* spatial_smooth: mean(dx^2) + mean(dy^2), weight alpha_spatial */
#define L4D_PATCH_TV       16u   /* tv_loss: mean(dx) + mean(dy), weight alpha_tv */
int    l4d_patch_loss(const float* depth, const float* gt3, uint32_t n, uint32_t px, uint32_t py, float scale, uint32_t crit,
                      uint32_t flags, float alpha_grad, float alpha_grad_norm, float alpha_spatial, float alpha_tv, float* loss,
                      float* g_depth, void* stream);
int    l4d_patch_loss_backward(const float* g_saved, const float* g_loss, uint32_t n, float* g_depth, void* stream);
size_t l4d_los_work_bytes(void);
int    l4d_los_loss(const float* weights, const float* z_vals, const float* gt3, uint32_t n, uint32_t S, double eps,
                    float* loss, void* work, size_t work_bytes, void* stream);
int    l4d_los_loss_backward(const float* weights, const float* z_vals, const float* gt3, uint32_t n, uint32_t S, double eps,
                             const void* work, const float* g_loss, float* g_weights, void* stream);

/* --- the main LiDAR loss of train_step (model/runner.py:193-220) and eval_step (:409-421), every criterion ----------------
 * Inputs are fp32 device arrays: depth[n], image2[n, 2] = (ray drop, intensity), gt3[n, 3] = (raydrop m, intensity,
 * depth).  crit_* are L4D_GRAD_* codes (main_lidar4d.py:183-188), delta the huber delta, (float)(0.2 * opt.scale) with
 * the product in double.  Sums are taken in double in a fixed order: the same inputs give the same bits.
 * l4d_main_loss: WRITES *loss = (a_d C_d(depth m, gt_d) + a_r C_r(r, clamp(m, s, 1 - s)) + a_i C_i(int m, gt_i)).sum()
 *   with r = image_0, or sigmoid(image_0) for bce (BCEWithLogits then applies its own sigmoid, as the reference does);
 *   a cos term is CosineSimilarity over all n rays, counted n times when another term is elementwise and once when all
 *   three are cos.  With rays_d[n, 3] != NULL it adds 0.5 mean(dist1 + dist2) of the chamfer distances between
 *   rays_d * depth m / scale and rays_d * gt_d / scale (scale > 0; ties go to the smallest index).  Writes g_depth[n]
 *   and g_image2[n, 2] = d loss / d (depth, image) for a unit upstream gradient.  work = l4d_main_loss_work_bytes(n)
 *   bytes when rays_d != NULL (L4D_ESIZE when smaller; it may be NULL otherwise); it begins with the two clouds,
 *   prediction then ground truth, [n, 3] each.  1 <= n < 2^31.  One launch without the chamfer term; with it the
 *   chamfer op's launches (l4d_chamfer_forward / _backward) and one more.
 * l4d_main_loss_backward: g_depth = g_saved_depth * *g_loss and g_image2 = g_saved_image2 * *g_loss, the incoming
 *   gradient read from device memory.  One launch.
 * l4d_main_eval_loss: WRITES *loss = a_d mean C_d(depth mask, gt_d) + a_r mean C_r(r, m) + a_i mean C_i(int mask, gt_i)
 *   over [B, H, W] images, mask = r > 0.5 (0 for NaN).  r is raydrop (B*H*W elements of dtype raydrop_dtype =
 *   L4D_DTYPE_*, the U-Net's output) when given, else image_0, or sigmoid(image_0) for bce.  A cos term is the mean
 *   of the per-column cosines over H, as CosineSimilarity(dim=1).  No gradient.  One launch.
 * Null required pointers, n = 0, unknown criteria or dtypes: L4D_EINVAL. */
size_t l4d_main_loss_work_bytes(uint32_t n);
int    l4d_main_loss(const float* depth, const float* image2, const float* gt3, const float* rays_d_or_null, uint32_t n,
                     uint32_t crit_d, uint32_t crit_r, uint32_t crit_i, float alpha_d, float alpha_r, float alpha_i,
                     double smooth, float scale, float delta, float* loss, float* g_depth, float* g_image2, void* work,
                     size_t work_bytes, void* stream);
int    l4d_main_loss_backward(const float* g_saved_depth, const float* g_saved_image2, uint32_t n, const float* g_loss,
                              float* g_depth, float* g_image2, void* stream);
int    l4d_main_eval_loss(const float* depth, const float* image2, const float* gt3, const void* raydrop_or_null,
                          uint32_t raydrop_dtype, uint32_t B, uint32_t H, uint32_t W, uint32_t crit_d, uint32_t crit_r,
                          uint32_t crit_i, float alpha_d, float alpha_r, float alpha_i, float delta, float* loss, void* stream);

/* --- exact nearest-neighbour search through a uniform grid, and the flow loss of train_step (model/runner.py:222-253) -----
 * For clouds that are searched many times (every optimiser step of the flow loss).  b = 1 only; xyz[n, 3] fp32, 1 <= n < 2^31.
 * l4d_nn_grid_build indexes a cloud into `grid` (l4d_nn_grid_bytes(n) bytes, 16-byte aligned, the caller's; it holds a copy
 *   of the points, so xyz may be released) with `work` = l4d_nn_grid_work_bytes(n) scratch bytes (L4D_ESIZE when smaller).
 *   Five launches, no device-to-host read.  Points with a non-finite coordinate are left out (they can never be nearest).
 * l4d_nn_grid_query: for q[nq, 3], dist[nq] / idx[nq] = squared distance to, and ORIGINAL index of, the nearest indexed
 *   point - bit for bit what l4d_chamfer_forward returns for (q, xyz), the smallest index on ties, (+inf, 0) for a query
 *   with a non-finite coordinate or a cloud without a finite point.  `n` is the n of the build.  dist may be NULL when
 *   sum_parts is given: sum_parts[L4D_FLOW_PARTS] doubles receive per-CTA sums of dist (entries beyond the launch's CTAs
 *   are not written: zero them first).  One launch.
 * The flow loss, for pc[n, 3], flow6[n, 6] = (forward | backward) flow of pc, and one neighbouring frame's cloud target[m, 3]
 * with its index `grid`:
 *   l4d_flow_warp_query: warped[n, 3] = pc + flow6[:, 3 dir .. 3 dir + 2] * step, idx1[n] = nearest target of every warped
 *     point, sum_parts as above.  One launch.  The caller then indexes `warped` (l4d_nn_grid_build) and queries it with
 *     `target` (l4d_nn_grid_query) for idx2[m].
 *   l4d_flow_term_backward ACCUMULATES d (0.5 (sum dist1 + sum dist2)) / d flow6 times the device float *g_loss into
 *     g_flow6[n, 6] (columns 3 dir .. 3 dir + 2).  One launch; the target gets no gradient.
 *   l4d_flow_ground: per-CTA sums of |flow6| over [n, 6] into sum_parts[L4D_FLOW_PARTS]; l4d_flow_ground_backward WRITES
 *     g_flow6 = 0.001 sign(flow6) *g_loss.
 *   l4d_flow_loss_finish: *loss = 0.5 * sum(sum_parts[0 .. n_chamfer)) + 0.001 * sum(sum_parts[n_chamfer .. + n_ground)),
 *     in double and in a fixed order: the same inputs give the same bits. */
#define L4D_FLOW_PARTS 2048
size_t l4d_nn_grid_bytes(uint32_t n);
size_t l4d_nn_grid_work_bytes(uint32_t n);
int    l4d_nn_grid_build(const float* xyz, uint32_t n, void* grid, size_t grid_bytes, void* work, size_t work_bytes, void* stream);
int    l4d_nn_grid_query(const void* grid, size_t grid_bytes, uint32_t n, const float* q, uint32_t nq, float* dist_or_null,
                         int32_t* idx, double* sum_parts_or_null, void* stream);
int    l4d_flow_warp_query(const float* pc, const float* flow6, uint32_t n, uint32_t dir, float step, const void* grid,
                           size_t grid_bytes, uint32_t m, float* warped, int32_t* idx1, double* sum_parts, void* stream);
int    l4d_flow_term_backward(const float* warped, uint32_t n, const float* target, uint32_t m, const int32_t* idx1,
                              const int32_t* idx2, uint32_t dir, float step, const float* g_loss, float* g_flow6, void* stream);
int    l4d_flow_ground(const float* flow6, uint32_t n, double* sum_parts, void* stream);
int    l4d_flow_ground_backward(const float* flow6, uint32_t n, const float* g_loss, float* g_flow6, void* stream);
int    l4d_flow_loss_finish(const double* sum_parts, uint32_t n_chamfer, uint32_t n_ground, float* loss, void* stream);

/* --- range image <-> point cloud (utils/convert.py) and the point-cloud metric of PointsMeter (utils/metrics.py:229-279) ---
 * Images are H x W row-major with 1 <= H, W and H*W <= 2^31; otherwise, and for null required pointers, L4D_EINVAL.
 * l4d_pano_project = lidar_to_pano_with_intensities: points[n, stride] (stride 3, or 4 with the intensity in column 3) ->
 *   pano[H,W] (nearest distance per pixel, 0 = empty) and, if not NULL, intensities[H,W], with the reference's float32
 *   arithmetic and its sequential z-buffer (a zero-distance point empties its pixel, keeping its own intensity; ties go to
 *   the earlier point).  fov_up / fov are in degrees and double, as the reference's Python floats; points at distance
 *   >= max_depth, or at a NaN distance, are skipped.  n = 0 gives an empty image.
 *   work = l4d_pano_project_work_bytes(H, W) bytes (L4D_ESIZE when smaller).
 * l4d_pano_unproject = pano_to_lidar_with_intensities: every pixel with pano != 0 (NaN included) becomes a row
 *   (dir * pano[, intensity]) of out[H*W, 4] when intensities is given, else out[H*W, 3], in row-major pixel order;
 *   the number of rows goes to the DEVICE uint32 *count.  work = l4d_pano_unproject_work_bytes(H, W) bytes.
 * l4d_point_metrics: squared nearest-neighbour distances dist1[n] and dist2[m] (l4d_chamfer_forward), n, m >= 1 ->
 *   out[5] = {mean(dist1) + mean(dist2), F-score, precision = count(dist1 < thr)/n, recall = count(dist2 < thr)/m, 0};
 *   the F-score is 0 where 2pr/(p+r) is NaN.  Deterministic: the same inputs give the same bits. */
size_t l4d_pano_project_work_bytes(uint32_t H, uint32_t W);
int    l4d_pano_project(const float* points, uint32_t n, uint32_t stride, double fov_up, double fov, uint32_t H, uint32_t W,
                        float max_depth, float* pano, float* intensities_or_null, void* work, size_t work_bytes, void* stream);
size_t l4d_pano_unproject_work_bytes(uint32_t H, uint32_t W);
int    l4d_pano_unproject(const float* pano, const float* intensities_or_null, uint32_t H, uint32_t W, float fov_up, float fov,
                          float* out, uint32_t* count, void* work, size_t work_bytes, void* stream);
int    l4d_point_metrics(const float* dist1, uint32_t n, const float* dist2, uint32_t m, float thr, float* out, void* stream);

/* --- the depth / intensity / ray-drop meters (utils/metrics.py DepthMeter, IntensityMeter, RaydropMeter) -------------
 * Results are WRITTEN as doubles to device memory; no host read, the caller's stream, and sums in a fixed order, so the
 * same inputs give the same bits.  Null pointers and bad sizes: L4D_EINVAL.
 * l4d_image_metrics = compute_depth_errors / compute_intensity_errors on fp32 pred, gt [H, W] (7 <= H, W, H*W < 2^31):
 *   both clamped to [lo, hi] in float32 (NaN stays NaN), then out[5] = {rmse, medae, NaN (the LPIPS slot), ssim, psnr}:
 *   rmse = sqrt(f32 mean of f32((gt - pred)^2)), medae = np.median(|gt - pred|) exactly, ssim = skimage's
 *   structural_similarity(pred, gt, data_range = max(gt) - min(gt)) with its constants squared as x*x, and
 *   psnr = f32(10 log10(f32(peak / mse))) (peak 80^2 for depth, 1 for intensity).  work = l4d_image_metrics_work_bytes(H, W)
 *   bytes, 16-byte aligned (L4D_ESIZE when smaller); on return it holds the clamped pred at byte offset 0 and the clamped
 *   gt at byte offset L4D_IM_GT_OFFSET(H, W), each [H, W] fp32.  Four launches.
 * l4d_raydrop_metrics = RaydropMeter.update on fp32 pred, gt [n] (1 <= n < 2^31): out[3] = {rmse, acc, f1} with
 *   mask = pred > ratio, acc = count(mask == gt) / n, f1 = 2pr/(p+r) over 64-bit counts (NaN when TP + FP = 0 or
 *   TP + FN = 0, as in the reference).  One launch. */
#define L4D_IM_GT_OFFSET(H, W) ((((size_t)(H) * (W) * 4u) + 255u) & ~(size_t)255u)
size_t l4d_image_metrics_work_bytes(uint32_t H, uint32_t W);
int    l4d_image_metrics(const float* pred, const float* gt, uint32_t H, uint32_t W, float lo, float hi, float peak,
                         double* out, void* work, size_t work_bytes, void* stream);
int    l4d_raydrop_metrics(const float* pred, const float* gt, uint32_t n, float ratio, double* out, void* stream);

/* --- the flow loss's point-cloud preparation (utils/misc.py point_removal, model/runner.py process_pointcloud) ---------
 * Points are row-major [n, 3] float64 unless said otherwise, 1 <= n < 2^31 (else L4D_EINVAL, as for null required
 * pointers).  Compactions keep index order and write their row counts to DEVICE uint32 memory; work buffers of at least
 * the matching *_work_bytes(n) bytes are the caller's (L4D_ESIZE when smaller).  Every op runs on `stream`.
 * l4d_range_filter = range_filter: float32 points[n, stride] (stride >= 3, columns beyond z copied) -> the rows with
 *   dist_min <= |p| <= dist_max, z_lo < z < z_hi and outside the ego box |x| < 2, |y| < 1, |z| < 2, in float32 as NumPy.
 * l4d_knn_mean_dist: avg[i] = mean of sqrt(d2) over the min(k, n) nearest points of point i (itself included, 1 <= k
 *   <= 64), d2 = ((dx*dx) + dy*dy) + dz*dz in float64, summed in ascending order.  Exact selection, no work buffer.
 * l4d_outlier_select: Open3D's statistical outlier rule on those means: mean = sum_{avg>0} avg / n, std =
 *   sqrt(sum_{avg>0} (avg - mean)^2 / (n - 1)); keep avg > 0 && avg < mean + std_ratio * std -> out[count, 3] and, if
 *   not NULL, the kept int32 indices.  stats_or_null (device, 3 doubles) receives {threshold, mean, std}.
 * l4d_plane_scores: counts[h] = #{i : |((a x_i + b y_i) + c z_i) + d| / r < threshold} for the m hypotheses
 *   hypotheses[h] = (a, b, c, d, r) (device [m, 5] float64), every operation rounded on its own (no FMA).
 * l4d_plane_mask: mask[i] = 1 where point i is an inlier of (a, b, c, d, r); other bytes are left as they are, so calls
 *   on a zeroed mask build the union of several hypotheses' inliers.
 * l4d_ground_split: ground = rows with mask[i] != 0 && z < z_max, rest = all other rows, each in index order with
 *   optional int32 indices; counts (device, 2 x uint32) = {ground rows, rest rows}.
 * l4d_pose_transform: out[i] = (pose @ [scale * p_i, 1])[:3] in float64, ((p_r0 X + p_r1 Y) + p_r2 Z) + p_r3, with
 *   pose a HOST row-major 4x4 float32 matrix. */
size_t l4d_range_filter_work_bytes(uint32_t n);
int    l4d_range_filter(const float* points, uint32_t n, uint32_t stride, float dist_min, float dist_max, float z_lo, float z_hi,
                        float* out, uint32_t* count, void* work, size_t work_bytes, void* stream);
int    l4d_knn_mean_dist(const double* points, uint32_t n, uint32_t k, double* avg, void* stream);
size_t l4d_outlier_select_work_bytes(uint32_t n);
int    l4d_outlier_select(const double* points, uint32_t n, const double* avg, double std_ratio, double* out,
                          int32_t* index_or_null, uint32_t* count, double* stats_or_null, void* work, size_t work_bytes,
                          void* stream);
int    l4d_plane_scores(const double* points, uint32_t n, const double* hypotheses, uint32_t m, double threshold,
                        uint32_t* counts, void* stream);
int    l4d_plane_mask(const double* points, uint32_t n, double a, double b, double c, double d, double r, double threshold,
                      uint8_t* mask, void* stream);
size_t l4d_ground_split_work_bytes(uint32_t n);
int    l4d_ground_split(const double* points, uint32_t n, const uint8_t* mask, double z_max, double* ground,
                        int32_t* ground_index_or_null, double* rest, int32_t* rest_index_or_null, uint32_t* counts,
                        void* work, size_t work_bytes, void* stream);
int    l4d_pose_transform(const double* points, uint32_t n, double scale, const float* pose, double* out, void* stream);

/* --- LiDAR sweep images (model/simulator.py Simulator.render, model/runner.py Trainer.test / evaluate_one_epoch) --------
 * l4d_sweep_images: one rendered frame, depth[H*W] and image[H*W, 2] (channel 0 ray drop, channel 1 intensity) float32,
 *   and optionally the refined ray drop raydrop[H*W] (dtype L4D_SWEEP_F32 or L4D_SWEEP_F16; when NULL, image channel 0
 *   is the ray drop and dtype must be L4D_SWEEP_F32) -> the 8-bit images the reference writes and the inputs of its
 *   point cloud.  With r the ray drop, m = r > 0.5 in r's dtype, I the intensity, D the depth:
 *   L4D_SWEEP_SIM:  panel [3H, W, 3] BGR = {grey u8(r 255), lut_intensity[u8(I m 255)], lut_depth[u8(D m 255)]};
 *                   pano[H*W] = D m / scale, intensities[H*W] = I m.
 *   L4D_SWEEP_TEST: with I', D' = I m, D m if test_mask else I, D: panel = [H, W] u8(m 255), then [H, W, 3]
 *                   lut_intensity[u8(I' 255)], then [H, W, 3] lut_depth[u8(D' 255)]; pano[H*W] = D' / scale.
 *   L4D_SWEEP_EVAL: panel [6H, W, 3] = {grey u8(r 255), lut_intensity[u8(I 255)], lut_depth[u8(D 255)], grey u8(m 255),
 *                   lut_intensity[u8(I m 255)], lut_depth[u8(D m 255)]}, the last two products in double.
 *   r 255 is rounded in r's dtype, everything else in float32 unless said; u8() is NumPy's float -> uint8 cast (truncate,
 *   low byte of the int32; NaN, inf and values outside the int32 range give 0).  The luts are [256, 3] BGR device tables
 *   (cv2.applyColorMap of 0..255 with COLORMAP_BONE and COLORMAP_TURBO), required by every layout.  pano is required by
 *   SIM and TEST, intensities by SIM; the others are ignored.  Panel bytes: L4D_SWEEP_PANEL_BYTES(layout, H, W).
 *   Null required pointers, H or W = 0, H*W >= 2^31, unknown layout or dtype: L4D_EINVAL.  One launch on `stream`. */
#define L4D_SWEEP_SIM  0u
#define L4D_SWEEP_TEST 1u
#define L4D_SWEEP_EVAL 2u
#define L4D_SWEEP_F32  0u
#define L4D_SWEEP_F16  1u
#define L4D_SWEEP_PANEL_BYTES(layout, H, W) \
  ((size_t)(H) * (W) * ((layout) == L4D_SWEEP_EVAL ? 18u : (layout) == L4D_SWEEP_TEST ? 7u : 9u))
int    l4d_sweep_images(const float* depth, const float* image, const void* raydrop_or_null, uint32_t raydrop_dtype,
                        uint32_t H, uint32_t W, uint32_t layout, float scale, uint32_t test_mask,
                        const uint8_t* lut_intensity, const uint8_t* lut_depth, uint8_t* panel, float* pano_or_null,
                        float* intensities_or_null, void* stream);

/* --- the ray-drop refinement loop (model/runner.py Trainer.refine:865-913) ---------------------------------------------
 * l4d_box_mask: out = x * m over x[B, C, H, W] float32 (out may alias x), with m = 0 inside any of the n_boxes <=
 *   L4D_MAX_BOXES boxes and 1 elsewhere, the same for every batch item and channel.  boxes is a HOST int32 array
 *   [n_boxes, 4] of (y0, x0, h, w) with h, w >= 1, y0, x0 >= 0, y0 + h <= H and x0 + w <= W (it may be NULL when
 *   n_boxes = 0); it is passed to the kernel by value, so there is no copy and no sync.  The mask is multiplied, not
 *   selected: a negative x in a box gives -0.0, an inf or NaN in a box gives NaN.  B*C*H*W < 2^31.  One launch.
 * l4d_bce_loss = torch.nn.BCELoss() (mean reduction): pred[n] of dtype L4D_DTYPE_*, target[n] float32, 1 <= n < 2^31,
 *   each element in float32 as ((t - 1) * max(log1p(-x), -100)) - (t * max(log(x), -100)).  A pred outside [0, 1] or NaN
 *   gives a NaN element (torch's CUDA kernel asserts instead).  WRITES *loss (device float) = float32(sum / n) with the
 *   sum taken in double in a fixed order.  work = l4d_bce_loss_work_bytes() bytes (L4D_ESIZE when smaller).  Two
 *   launches (the partial sums, then a one-CTA finish).
 * l4d_bce_loss_backward: g_pred[n], in pred's dtype, = ((*g_loss * (x - t)) / max((1 - x) * x, 1e-12)) / n in float32,
 *   torch's gradient; NaN where pred is outside [0, 1] or NaN.  *g_loss is read from device memory.  One launch.
 * Null required pointers, bad sizes, dtypes, box counts or boxes: L4D_EINVAL. */
#define L4D_MAX_BOXES 32
#define L4D_DTYPE_F32  0u
#define L4D_DTYPE_F16  1u
#define L4D_DTYPE_BF16 2u
int    l4d_box_mask(const float* x, float* out, uint32_t B, uint32_t C, uint32_t H, uint32_t W, const int32_t* boxes_or_null,
                    uint32_t n_boxes, void* stream);
size_t l4d_bce_loss_work_bytes(void);
int    l4d_bce_loss(const void* pred, uint32_t pred_dtype, const float* target, uint32_t n, float* loss, void* work,
                    size_t work_bytes, void* stream);
int    l4d_bce_loss_backward(const void* pred, uint32_t pred_dtype, const float* target, uint32_t n, const float* g_loss,
                             void* g_pred, void* stream);

/* --- profiling aid: while started, CUDA events are recorded on the launch stream around every kernel of
 *     l4d_render_forward / l4d_render_backward.  l4d_profile_stop returns the number of (kernel name, ms)
 *     pairs written (static strings), or a negative error code.  Not thread-safe. --------------------------- */
/* kernels this library has launched in this process so far (bench.py "gpu_launches"; counted at the launch sites). */
unsigned long long l4d_launch_count(void);
int    l4d_profile_start(void);
int    l4d_profile_stop(const char** names, float* ms, int cap);

/* wgmma self-test of the MLP engine's building blocks: C[128,N] = A[128,K] * B[N,K]^T,
 * fp16 operands, fp32 accumulate (N%16==0 in [16,256], K%16==0 in [16,512]). */
int    l4d_tc_selftest(const void* A_half, const void* B_half, float* C, uint32_t N, uint32_t K, void* stream);
/* same with operands pre-arranged in the engine's tile format, M in {64,128}, K-major or MN-major operands
 * (the weight-gradient GEMMs X^T*delta read sample-major tiles as MN-major operands). */
int    l4d_tc_selftest2(const void* A_tile, const void* B_tile, float* C, uint32_t M, uint32_t N, uint32_t K,
                        uint32_t a_mn_major, uint32_t b_mn_major, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LIDAR4D_B200_H_ */
