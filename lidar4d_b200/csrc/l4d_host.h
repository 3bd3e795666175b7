// l4d_host.h - host-side layouts shared by the kernels' launchers (l4d_kernels.cu)
// and the CPU host-sim test harness (tests/hostsim/hostsim.cu).
#pragma once
#include <string.h>
#include "l4d_core.cuh"

int l4d_fail(int code, const char* fmt, const char* a = "", const char* b = "");

// =============================================================================
// layouts of the staged working set and of the gradient work buffer
// =============================================================================
struct StagedLayout {
  size_t hs, hd[3], hf;
  size_t planes[L4D_MAX_PLANE_SCALES][6];
  size_t sig_w1t, sig_w2t, sig_w2;
  size_t att_w1t[2], att_w2t[2], att_w2[2], att_w3[2];
  size_t flo_w0t, flo_w1t, flo_w1, flo_w2t, flo_w2;
  size_t tc_sig_w1, tc_sig_w2, tc_att_w1g, tc_att_w2[2], tc_att_w1g_net[2], tc_flo_w0, tc_flo_w1, tc_flo_w2;
  size_t total;
};
struct GradWorkLayout {
  size_t planes[L4D_MAX_PLANE_SCALES][6];
  size_t sig_w1t, sig_w2;
  size_t att_w1t[2], att_w2t[2], att_w3[2];
  size_t flo_w0t, flo_w1t, flo_w2;
  size_t scatter_tickets;  // 3 x uint32: k_bwd_encoders' work-ticket counters
  size_t hd_comb[3], hf_comb;
  size_t pl_rows;          // [query][scale][plane 2|4|5][R][8]
  size_t comb_frame;       // bytes of one frame's hd_comb .. pl_rows block; frame f's block is at + f * comb_frame
  size_t total;
};

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static inline void plane_hw(const L4DConfig* c, int s, int ci, int& H, int& W) {
  // itertools.combinations(range(4),2): (0,1)(0,2)(0,3)(1,2)(1,3)(2,3); tensor [1,8,reso[b],reso[a]]
  const bool dyn = (ci == 2 || ci == 4 || ci == 5);
  W = (int)c->plane_res[s];
  H = dyn ? (int)c->time_resolution : (int)c->plane_res[s];
}

static inline StagedLayout staged_layout(const L4DConfig* c) {
  StagedLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  L.hs = take((size_t)c->hash_static.offset[c->hash_static.n_levels] * 4 * sizeof(__half));
  for (int p = 0; p < 3; ++p)
    L.hd[p] = take((size_t)c->hash_dynamic[p].offset[c->hash_dynamic[p].n_levels] * 8 * sizeof(__half) * (c->time_resolution - 1));
  L.hf = take((size_t)c->flow.offset[c->flow.n_levels] * 8 * sizeof(__half));
  for (uint32_t s = 0; s < c->n_plane_scales; ++s)
    for (int ci = 0; ci < 6; ++ci) {
      int H, W;
      plane_hw(c, s, ci, H, W);
      L.planes[s][ci] = take((size_t)H * W * 8 * sizeof(float));
    }
  const size_t f = sizeof(float);
  L.sig_w1t = take((size_t)c->sigma_in_pad * 64 * f);
  L.sig_w2t = take(64 * 16 * f);
  L.sig_w2 = take(16 * 64 * f);
  for (int n = 0; n < 2; ++n) {
    L.att_w1t[n] = take((size_t)c->attr_in_pad * 64 * f);
    L.att_w2t[n] = take(64 * 64 * f);
    L.att_w2[n] = take(64 * 64 * f);
    L.att_w3[n] = take(64 * f);
  }
  L.flo_w0t = take(16 * 64 * f);
  L.flo_w1t = take(64 * 64 * f);
  L.flo_w1 = take(64 * 64 * f);
  L.flo_w2t = take(64 * 8 * f);
  L.flo_w2 = take(8 * 64 * f);
  L.tc_sig_w1 = take((size_t)c->sigma_in_pad * 64 * 2);
  L.tc_sig_w2 = take(64 * 16 * 2);
  L.tc_att_w1g = take(16 * 128 * 2);
  for (int n = 0; n < 2; ++n) L.tc_att_w2[n] = take(64 * 64 * 2);
  for (int n = 0; n < 2; ++n) L.tc_att_w1g_net[n] = take(16 * 64 * 2);
  L.tc_flo_w0 = take(16 * 64 * 2); L.tc_flo_w1 = take(64 * 64 * 2); L.tc_flo_w2 = take(64 * 16 * 2);
  L.total = o;
  return L;
}

// floats of one full set of time-plane rows: [query 3][scale][plane 3][R][8]
static inline size_t time_rows_floats(const L4DConfig* c) {
  size_t n = 0;
  for (uint32_t s = 0; s < c->n_plane_scales; ++s) n += (size_t)c->plane_res[s] * 8 * 3;
  return 3 * n;
}
// the [scale][plane][query] pointer table over such a set at base (every row starts on a multiple of 32 bytes)
template <class T>
static inline void point_time_rows(const L4DConfig* c, T* base, T* (&tab)[L4D_MAX_PLANE_SCALES][3][3]) {
  for (int q = 0; q < 3; ++q)
    for (uint32_t s = 0; s < c->n_plane_scales; ++s)
      for (int t = 0; t < 3; ++t) {
        tab[s][t][q] = base;
        base += (size_t)c->plane_res[s] * 8;
      }
}

// n_frames: the per-frame accumulators (hd_comb, hf_comb, pl_rows) once per frame of a multi-frame launch, frame-major
static inline GradWorkLayout grad_work_layout(const L4DConfig* c, uint32_t n_frames = 1) {
  GradWorkLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  for (uint32_t s = 0; s < c->n_plane_scales; ++s)
    for (int ci = 0; ci < 6; ++ci) {
      int H, W;
      plane_hw(c, s, ci, H, W);
      L.planes[s][ci] = take((size_t)H * W * 8 * sizeof(float));
    }
  const size_t f = sizeof(float);
  L.sig_w1t = take((size_t)c->sigma_in_pad * 64 * f);
  L.sig_w2 = take(16 * 64 * f);
  for (int n = 0; n < 2; ++n) {
    L.att_w1t[n] = take((size_t)c->attr_in_pad * 64 * f);
    L.att_w2t[n] = take(64 * 64 * f);
    L.att_w3[n] = take(64 * f);
  }
  L.flo_w0t = take(16 * 64 * f);
  L.flo_w1t = take(64 * 64 * f);
  L.flo_w2 = take(8 * 64 * f);
  L.scatter_tickets = take(3 * sizeof(uint32_t));
  for (int p = 0; p < 3; ++p) L.hd_comb[p] = take((size_t)c->hash_dynamic[p].offset[c->hash_dynamic[p].n_levels] * f);
  L.hf_comb = take((size_t)c->flow.offset[c->flow.n_levels] * 2 * f);
  L.pl_rows = take(time_rows_floats(c) * f);
  L.comb_frame = o - L.hd_comb[0];
  L.total = L.hd_comb[0] + (size_t)n_frames * L.comb_frame;
  return L;
}

static inline int check_config(const L4DConfig* c) {
  if (!c) return l4d_fail(L4D_EINVAL, "null config");
  if (c->hash_static.n_dims != 3 || c->hash_static.n_features != 4) return l4d_fail(L4D_EINVAL, "hash_static must be 3D F=4");
  for (int p = 0; p < 3; ++p) {
    if (c->hash_dynamic[p].n_dims != 2 || c->hash_dynamic[p].n_features != 4) return l4d_fail(L4D_EINVAL, "hash_dynamic must be 2D F=4");
    if (c->hash_dynamic[p].n_levels != c->hash_static.n_levels) return l4d_fail(L4D_EINVAL, "hash level counts differ");
    // tiny-cuda-nn rounds every level up to a multiple of 8 entries; the scalar per-entry accumulators / contracted tables
    // of the dynamic hash are accessed as aligned quads of entries and rely on it
    for (uint32_t l = 0; l <= c->hash_dynamic[p].n_levels && l <= L4D_MAX_LEVELS; ++l)
      if (c->hash_dynamic[p].offset[l] % 8u) return l4d_fail(L4D_EINVAL, "hash_dynamic level offsets must be multiples of 8 entries");
  }
  if (c->flow.n_dims != 3 || c->flow.n_features != 8 || c->flow.n_levels != 8) return l4d_fail(L4D_EINVAL, "flow grid must be 3D F=8 L=8");
  if (c->hash_static.n_levels < 1 || c->hash_static.n_levels > L4D_MAX_LEVELS) return l4d_fail(L4D_EINVAL, "bad n_levels");
  if (c->n_plane_scales < 1 || c->n_plane_scales > L4D_MAX_PLANE_SCALES) return l4d_fail(L4D_EINVAL, "bad n_plane_scales");
  if (c->time_resolution < 2 || c->time_resolution > L4D_MAX_TIME_SLICES) return l4d_fail(L4D_EINVAL, "bad time_resolution");
  if (c->view_degree != 12 || c->attr_in_dim != 87 || c->attr_in_pad != 96) return l4d_fail(L4D_EINVAL, "attribute heads must be 72+15 -> pad 96");
  const uint32_t din = 2 * c->n_plane_scales * 8 + c->hash_static.n_levels * 4 + 3 * c->hash_static.n_levels;
  if (c->sigma_in_dim != din || c->sigma_in_pad != (din + 15) / 16 * 16) return l4d_fail(L4D_EINVAL, "sigma_in_dim mismatch");
  if (c->sigma_in_pad > 256) return l4d_fail(L4D_EINVAL, "sigma_in_pad too large");
  if (!(c->bound > 0.f) || !(c->far_lidar > c->near_lidar)) return l4d_fail(L4D_EINVAL, "bad bound/near/far");
  return L4D_OK;
}

static inline void fill_grid(DevGrid& d, const L4DGrid& g) {
  memset(&d, 0, sizeof(d));
  for (uint32_t l = 0; l < g.n_levels; ++l) {
    d.scale[l] = g.scale[l];
    d.res[l] = g.resolution[l];
    d.entries[l] = g.entries[l];
    d.offset[l] = g.offset[l];
  }
  d.offset[g.n_levels] = g.offset[g.n_levels];
  d.n_levels = g.n_levels;
}

static inline void build_model(const L4DConfig* c, const void* staged, DevModel& M) {
  StagedLayout L = staged_layout(c);
  const char* b = reinterpret_cast<const char*>(staged);
  memset(&M, 0, sizeof(M));
  fill_grid(M.gs, c->hash_static);
  for (int p = 0; p < 3; ++p) fill_grid(M.gd[p], c->hash_dynamic[p]);
  fill_grid(M.gf, c->flow);
  M.hs = reinterpret_cast<const __half*>(b + L.hs);
  for (int p = 0; p < 3; ++p) {
    M.hd[p] = reinterpret_cast<const __half*>(b + L.hd[p]);
    M.hd_slice_entries[p] = c->hash_dynamic[p].offset[c->hash_dynamic[p].n_levels];
  }
  M.hf = reinterpret_cast<const __half*>(b + L.hf);
  for (uint32_t s = 0; s < c->n_plane_scales; ++s) {
    M.plane_res[s] = c->plane_res[s];
    for (int ci = 0; ci < 6; ++ci) M.planes[s][ci] = reinterpret_cast<const float*>(b + L.planes[s][ci]);
  }
  M.n_scales = c->n_plane_scales;
  M.time_res = c->time_resolution;
  auto F = [&](size_t off) { return reinterpret_cast<const float*>(b + off); };
  M.sig_w1t = F(L.sig_w1t); M.sig_w2t = F(L.sig_w2t); M.sig_w2 = F(L.sig_w2);
  for (int n = 0; n < 2; ++n) {
    M.att_w1t[n] = F(L.att_w1t[n]); M.att_w2t[n] = F(L.att_w2t[n]);
    M.att_w2[n] = F(L.att_w2[n]); M.att_w3[n] = F(L.att_w3[n]);
  }
  M.flo_w0t = F(L.flo_w0t); M.flo_w1t = F(L.flo_w1t); M.flo_w1 = F(L.flo_w1);
  M.flo_w2t = F(L.flo_w2t); M.flo_w2 = F(L.flo_w2);
  auto Hh = [&](size_t off) { return reinterpret_cast<const __half*>(b + off); };
  M.tc_sig_w1 = Hh(L.tc_sig_w1); M.tc_sig_w2 = Hh(L.tc_sig_w2); M.tc_att_w1g = Hh(L.tc_att_w1g);
  M.tc_att_w2[0] = Hh(L.tc_att_w2[0]); M.tc_att_w2[1] = Hh(L.tc_att_w2[1]);
  M.tc_att_w1g_net[0] = Hh(L.tc_att_w1g_net[0]); M.tc_att_w1g_net[1] = Hh(L.tc_att_w1g_net[1]);
  M.tc_flo_w0 = Hh(L.tc_flo_w0); M.tc_flo_w1 = Hh(L.tc_flo_w1); M.tc_flo_w2 = Hh(L.tc_flo_w2);
  M.mlp_fp16 = c->mlp_fp16;
  M.sigma_in_dim = c->sigma_in_dim; M.sigma_in_pad = c->sigma_in_pad;
  M.attr_in_dim = c->attr_in_dim; M.attr_in_pad = c->attr_in_pad;
  M.view_degree = c->view_degree; M.active_sensor = c->active_sensor;
  M.bound = c->bound; M.near_lidar = c->near_lidar; M.far_lidar = c->far_lidar;
  M.density_scale = c->density_scale;
}

static inline void build_grads(const L4DConfig* c, const L4DMasterGrads* g, void* grad_work, DevGrads& G, bool comb = false) {
  GradWorkLayout L = grad_work_layout(c);      // frame 0's accumulators: the others follow at L.comb_frame strides
  char* b = reinterpret_cast<char*>(grad_work);
  memset(&G, 0, sizeof(G));
  G.hs = g->hash_static;
  for (int p = 0; p < 3; ++p)
    for (uint32_t s = 0; s < c->time_resolution; ++s) G.hd[p][s] = g->hash_dynamic[p][s];
  G.hf = g->flow_grid;
  auto F = [&](size_t off) { return reinterpret_cast<float*>(b + off); };
  for (uint32_t s = 0; s < c->n_plane_scales; ++s)
    for (int ci = 0; ci < 6; ++ci) G.planes_cl[s][ci] = F(L.planes[s][ci]);
  G.sig_w1t = F(L.sig_w1t); G.sig_w2 = F(L.sig_w2);
  for (int n = 0; n < 2; ++n) { G.att_w1t[n] = F(L.att_w1t[n]); G.att_w2t[n] = F(L.att_w2t[n]); G.att_w3[n] = F(L.att_w3[n]); }
  G.flo_w0t = F(L.flo_w0t); G.flo_w1t = F(L.flo_w1t); G.flo_w2 = F(L.flo_w2);
  if (comb) {
    for (int p = 0; p < 3; ++p) G.hd_comb[p] = F(L.hd_comb[p]);
    G.hf_comb = F(L.hf_comb);
    point_time_rows(c, F(L.pl_rows), G.pl_rows);
  }
}


#define L4D_NT 128
#define L4D_BWD_SCRATCH_CTAS 1024
struct SavedLayout { size_t feat, flow_in, sigma, attr, hidden, flow, dfeat, dflow, tstart, hd_con, pl_con, con_frame, total; };
// n_frames: the contracted tables (hd_con, pl_con) once per frame of a multi-frame launch, frame-major, con_frame bytes apart
static inline SavedLayout saved_layout(const L4DConfig* c, uint32_t n_rays, uint32_t S, uint32_t n_frames = 1) {
  SavedLayout L;
  const size_t P = (size_t)n_rays * S;
  const size_t tiles = (size_t)n_rays * ((S + 127) / 128);
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  // features: SoA fp32 planes (fp32-FMA kernels) or fp16 hi|lo operand tiles (tensor-core kernels), same region
  const size_t feat_soa = P * c->sigma_in_dim * sizeof(float);
  const size_t feat_tc = tiles * ((c->sigma_in_dim + 7) / 8) * 4096;
  L.feat = take(feat_soa > feat_tc ? feat_soa : feat_tc);
  L.flow_in = take(P * 16 * sizeof(float));
  L.sigma = take(P * sizeof(float));
  L.attr = take(P * 2 * sizeof(float));
  L.hidden = take((size_t)L4D_BWD_SCRATCH_CTAS * 64 * L4D_NT * sizeof(float));
  L.flow = take(P * 6 * sizeof(float));
  L.dfeat = take(tiles * ((c->sigma_in_dim + 3) / 4) * 2048);
  L.dflow = take(P * 6 * sizeof(float));
  L.tstart = take(tiles * sizeof(float));
  // contracted dynamic tables of the launch (DevModel::hd_con): [query cur|fwd|bwd][plane][entries] fp32
  size_t dyn_entries = 0;
  for (int p = 0; p < 3; ++p) dyn_entries += c->hash_dynamic[p].offset[c->hash_dynamic[p].n_levels];
  L.hd_con = take(3 * dyn_entries * sizeof(float));
  L.pl_con = take(time_rows_floats(c) * sizeof(float));      // contracted time-plane rows (DevModel::pl_con)
  L.con_frame = o - L.hd_con;
  L.total = L.hd_con + (size_t)n_frames * L.con_frame;
  return L;
}
// what l4d_density_forward_ex saves for l4d_density_backward on n explicit points: the Lagrange-contracted flow-MLP
// inputs [16][n] and the sigma-MLP input features [sigma_in_dim][n] as SoA planes (thread == point: every warp access is
// one 128 B line), and the per-CTA hidden scratch of k_density_bwd, one [64][L4D_NT] column block per CTA.  The backward
// runs at most `ctas` CTAs (one per 128-point tile, capped at L4D_BWD_SCRATCH_CTAS), so the buffer stays O(n).
struct DensitySavedLayout { size_t flow_in, feat, hidden, total; uint32_t ctas; };
static inline DensitySavedLayout density_saved_layout(const L4DConfig* c, uint32_t n) {
  DensitySavedLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
  const uint32_t tiles = (uint32_t)(((size_t)n + L4D_NT - 1) / L4D_NT);
  L.ctas = tiles < L4D_BWD_SCRATCH_CTAS ? tiles : L4D_BWD_SCRATCH_CTAS;
  L.flow_in = take((size_t)n * L4D_FLOW_IN * sizeof(float));
  L.feat = take((size_t)n * c->sigma_in_dim * sizeof(float));
  L.hidden = take((size_t)L.ctas * L4D_H * L4D_NT * sizeof(float));
  L.total = o;
  return L;
}

// DevModel::hd_con (dynamic-hash tables) and ::pl_con (time-plane rows) inside the saved buffer of a launch (level offsets,
// hence plane sizes, are multiples of 8 entries): those of the launch's first frame
static inline void point_contracted(const L4DConfig* c, void* saved, uint32_t n_rays, uint32_t S, DevModel& M) {
  SavedLayout L = saved_layout(c, n_rays, S);
  float* b = reinterpret_cast<float*>(reinterpret_cast<char*>(saved) + L.hd_con);
  for (int q = 0; q < 3; ++q)
    for (int p = 0; p < 3; ++p) {
      M.hd_con[p][q] = b;
      b += c->hash_dynamic[p].offset[c->hash_dynamic[p].n_levels];
    }
  point_time_rows<const float>(c, reinterpret_cast<const float*>(reinterpret_cast<char*>(saved) + L.pl_con), M.pl_con);
}
static inline SavedView saved_view(const L4DConfig* c, void* saved, uint32_t n_rays, uint32_t S) {
  SavedLayout L = saved_layout(c, n_rays, S);
  char* b = reinterpret_cast<char*>(saved);
  SavedView v;
  v.feat = reinterpret_cast<float*>(b + L.feat);
  v.feat_tc = reinterpret_cast<unsigned char*>(b + L.feat);
  v.n_tiles = (S + 127) / 128;
  v.x_chunks = (c->sigma_in_dim + 7) / 8;
  v.d_quads = (c->sigma_in_dim + 3) / 4;
  v.flow_in = reinterpret_cast<float*>(b + L.flow_in);
  v.sigma = reinterpret_cast<float*>(b + L.sigma);
  v.attr = reinterpret_cast<float*>(b + L.attr);
  v.hidden = reinterpret_cast<float*>(b + L.hidden);
  v.flow = reinterpret_cast<float*>(b + L.flow);
  v.dfeat = reinterpret_cast<float*>(b + L.dfeat);
  v.dflow = reinterpret_cast<float*>(b + L.dflow);
  v.tstart = reinterpret_cast<float*>(b + L.tstart);
  v.P = (size_t)n_rays * S;
  return v;
}

