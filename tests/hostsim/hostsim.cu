// hostsim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// Compiles the __host__ __device__ per-sample functions of
// lidar4d_b200/csrc/l4d_core.cuh + l4d_bwd.cuh for the CPU and drives them with
// plain loops that mirror the kernels' tile structure (thread == sample, tiles
// of L4D_NT samples, cooperative outer products replaced by loops).  This lets
// `pytest -m "not gpu"` check the kernels' arithmetic against the oracle in the
// build container, which has no GPU.  All pointers are HOST pointers here.
#include <math.h>
#include <stdio.h>
#include <algorithm>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../lidar4d_b200/csrc/l4d_bwd.cuh"
#include "../../lidar4d_b200/csrc/l4d_core.cuh"
#include "../../lidar4d_b200/csrc/l4d_host.h"

static char g_err[512];
int l4d_fail(int code, const char* fmt, const char* a, const char* b) {
  snprintf(g_err, sizeof(g_err), fmt, a, b);
  return code;
}
extern "C" const char* hs_last_error(void) { return g_err; }

extern "C" size_t hs_staged_bytes(const L4DConfig* c) { return check_config(c) == L4D_OK ? staged_layout(c).total : 0; }
extern "C" size_t hs_grad_work_bytes(const L4DConfig* c) { return check_config(c) == L4D_OK ? grad_work_layout(c).total : 0; }
extern "C" size_t hs_saved_bytes(const L4DConfig* c, uint32_t n, uint32_t S) {
  return check_config(c) == L4D_OK ? saved_layout(c, n, S).total : 0;
}

// ---- host mirror of l4d_stage_params ---------------------------------------------------
extern "C" int hs_stage_params(const L4DConfig* cfg, const L4DMasterParams* m, void* staged) {
  int rc = check_config(cfg);
  if (rc) return rc;
  StagedLayout L = staged_layout(cfg);
  char* b = (char*)staged;
  auto cast = [&](const float* src, __half* dst, size_t n) { for (size_t i = 0; i < n; ++i) dst[i] = __float2half_rn(src[i]); };
  cast(m->hash_static, (__half*)(b + L.hs), (size_t)cfg->hash_static.offset[cfg->hash_static.n_levels] * 4);
  for (int p = 0; p < 3; ++p) {      // pair records {slice k F4, slice k+1 F4}
    const size_t ne = (size_t)cfg->hash_dynamic[p].offset[cfg->hash_dynamic[p].n_levels];
    for (uint32_t s = 0; s + 1 < cfg->time_resolution; ++s) {
      __half* dst = (__half*)(b + L.hd[p]) + (size_t)s * ne * 8;
      for (size_t e = 0; e < ne; ++e)
        for (int f = 0; f < 4; ++f) {
          dst[e * 8 + f] = __float2half_rn(m->hash_dynamic[p][s][e * 4 + f]);
          dst[e * 8 + 4 + f] = __float2half_rn(m->hash_dynamic[p][s + 1][e * 4 + f]);
        }
    }
  }
  cast(m->flow_grid, (__half*)(b + L.hf), (size_t)cfg->flow.offset[cfg->flow.n_levels] * 8);
  for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
    for (int ci = 0; ci < 6; ++ci) {
      int H, W;
      plane_hw(cfg, s, ci, H, W);
      float* dst = (float*)(b + L.planes[s][ci]);
      for (int px = 0; px < H * W; ++px)
        for (int c = 0; c < 8; ++c) dst[px * 8 + c] = m->planes[s][ci][(size_t)c * H * W + px];
    }
  auto T = [&](const float* src, int src_ld, float* dst, int rows, int cols, int vr, int vc) {
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < cols; ++c) dst[r * cols + c] = (r < vr && c < vc) ? src[(size_t)c * src_ld + r] : 0.f;
  };
  auto C = [&](const float* src, float* dst, int nv, int nt) { for (int i = 0; i < nt; ++i) dst[i] = i < nv ? src[i] : 0.f; };
  auto F = [&](size_t off) { return (float*)(b + off); };
  const int ip = cfg->sigma_in_pad, ap = cfg->attr_in_pad;
  T(m->sigma_net, ip, F(L.sig_w1t), ip, 64, ip, 64);
  T(m->sigma_net + 64 * ip, 64, F(L.sig_w2t), 64, 16, 64, 16);
  C(m->sigma_net + 64 * ip, F(L.sig_w2), 16 * 64, 16 * 64);
  const float* att[2] = {m->raydrop_net, m->intensity_net};
  for (int n = 0; n < 2; ++n) {
    T(att[n], ap, F(L.att_w1t[n]), ap, 64, ap, 64);
    T(att[n] + 64 * ap, 64, F(L.att_w2t[n]), 64, 64, 64, 64);
    C(att[n] + 64 * ap, F(L.att_w2[n]), 64 * 64, 64 * 64);
    C(att[n] + 64 * ap + 64 * 64, F(L.att_w3[n]), 64, 64);
  }
  T(m->flow_mlp[0], 16, F(L.flo_w0t), 16, 64, 16, 64);
  T(m->flow_mlp[1], 64, F(L.flo_w1t), 64, 64, 64, 64);
  C(m->flow_mlp[1], F(L.flo_w1), 64 * 64, 64 * 64);
  T(m->flow_mlp[2], 64, F(L.flo_w2t), 64, 8, 64, 6);
  C(m->flow_mlp[2], F(L.flo_w2), 6 * 64, 8 * 64);
  if (cfg->mlp_fp16) {      // mirror of k_round_fp16 over the fp32 MLP working copies
    float* w = F(L.sig_w1t);
    const size_t n = (L.tc_sig_w1 - L.sig_w1t) / 4;
    for (size_t i = 0; i < n; ++i) w[i] = __half2float(__float2half_rn(w[i]));
  }
  return L4D_OK;
}

// ---- host mirror of l4d_unstage_grads ----------------------------------------------------
extern "C" int hs_unstage_grads(const L4DConfig* cfg, const void* grad_work, const L4DMasterGrads* g) {
  GradWorkLayout L = grad_work_layout(cfg);
  const char* b = (const char*)grad_work;
  auto F = [&](size_t off) { return (const float*)(b + off); };
  for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
    for (int ci = 0; ci < 6; ++ci) {
      int H, W;
      plane_hw(cfg, s, ci, H, W);
      const float* src = F(L.planes[s][ci]);
      for (int px = 0; px < H * W; ++px)
        for (int c = 0; c < 8; ++c) g->planes[s][ci][(size_t)c * H * W + px] += src[px * 8 + c];
    }
  auto AT = [&](const float* src, float* dst, int rows, int cols) {   // dst[r][c] += src[c][r], src cols = 64
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < cols; ++c) dst[r * cols + c] += src[(size_t)c * 64 + r];
  };
  auto A = [&](const float* src, float* dst, int n) { for (int i = 0; i < n; ++i) dst[i] += src[i]; };
  const int ip = cfg->sigma_in_pad, ap = cfg->attr_in_pad;
  AT(F(L.sig_w1t), g->sigma_net, 64, ip);
  A(F(L.sig_w2), g->sigma_net + 64 * ip, 16 * 64);
  float* att[2] = {g->raydrop_net, g->intensity_net};
  for (int n = 0; n < 2; ++n) {
    AT(F(L.att_w1t[n]), att[n], 64, ap);
    AT(F(L.att_w2t[n]), att[n] + 64 * ap, 64, 64);
    A(F(L.att_w3[n]), att[n] + 64 * ap + 64 * 64, 64);
  }
  AT(F(L.flo_w0t), g->flow_mlp[0], 64, 16);
  AT(F(L.flo_w1t), g->flow_mlp[1], 64, 64);
  A(F(L.flo_w2), g->flow_mlp[2], 6 * 64);
  return L4D_OK;
}

// ---- host mirror of k_contract_dynamic / k_contract_planes: fills `store`, points M.hd_con / M.pl_con at it ----------
static void contract_for_frame(const L4DConfig* cfg, const L4DFrame* frame, DevModel& M, std::vector<float>& store) {
  size_t tot = 0;
  for (int p = 0; p < 3; ++p) tot += M.hd_slice_entries[p];
  store.assign(3 * tot + time_rows_floats(cfg), 0.f);
  float* b = store.data();
  const L4DTimeQuery* qs[3] = {&frame->cur, &frame->fwd, &frame->bwd};
  const bool live[3] = {true, frame->has_fwd != 0, frame->has_bwd != 0};
  for (int q = 0; q < 3; ++q)
    for (int p = 0; p < 3; ++p) {
      const uint32_t n = M.hd_slice_entries[p];
      M.hd_con[p][q] = b;
      if (live[q]) {
        const uint4* tab = reinterpret_cast<const uint4*>(M.hd[p]) + (size_t)l4d_time_pair(*qs[q], cfg->time_resolution) * n;
        for (uint32_t e = 0; e < n; ++e) b[e] = l4d_contract_entry(tab[e], *qs[q], cfg->time_resolution);
      }
      b += n;
    }
  float* rows[L4D_MAX_PLANE_SCALES][3][3];
  point_time_rows(cfg, b, rows);
  for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
    for (int t = 0; t < 3; ++t)
      for (int q = 0; q < 3; ++q) {
        M.pl_con[s][t][q] = rows[s][t][q];
        if (!live[q]) continue;
        const int R = (int)cfg->plane_res[s];
        const Bilerp bl = l4d_bilerp(0.f, 2, qs[q]->tau, (int)cfg->time_resolution);
        const float* P = M.planes[s][t == 0 ? 2 : (t == 1 ? 4 : 5)];
        for (int x = 0; x < R; ++x)
          for (int c = 0; c < 8; ++c) rows[s][t][q][x * 8 + c] = l4d_contract_texel(P, R, bl, x, c);
      }
}

// ---- forward (mirror of k_render_fwd) ---------------------------------------------------
extern "C" int hs_render_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const L4DRays* rays,
                                 float* depth, float* image, float* wsum, float* weights, float* zvals, void* saved) {
  int rc = check_config(cfg);
  if (rc) return rc;
  DevModel M;
  build_model(cfg, staged, M);
  const L4DFrame& F = *frame;
  const uint32_t S = rays->n_steps;
  SavedView sv;
  memset(&sv, 0, sizeof(sv));
  if (saved) sv = saved_view(cfg, saved, rays->n_rays, S);
  // rays->reserved bit 2 (host-sim only): gather the dynamic hash and the time planes from the per-launch contracted
  // tables / rows (DevModel::hd_con, pl_con)
  std::vector<float> con_store;
  if (rays->reserved & 4u) contract_for_frame(cfg, frame, M, con_store);
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, S, rays->perturb, rays->seed);
  for (uint32_t ray = 0; ray < rays->n_rays; ++ray) {
    const float* o = rays->rays_o + 3 * ray;
    const float* d = rays->rays_d + 3 * ray;
    float enc[L4D_ENC], cdir[128];
    for (int i = 0; i < L4D_ENC; ++i) enc[i] = l4d_freq(d[i / 24], (i % 24) >> 1, i & 1);
    for (int i = 0; i < 128; ++i) cdir[i] = l4d_attr_cdir(M, i >> 6, i & 63, enc);
    float carry = 1.f, pd = 0.f, p0 = 0.f, p1 = 0.f, pw = 0.f;
    const uint64_t rg = rays->ray_offset + ray;
    for (uint32_t j = 0; j < S; ++j) {
      const size_t p = (size_t)ray * S + j;
      float xb[64];
      const float zj = l4d_z(rs, rg, j);
      const float delta = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zj) : rs.sample_dist;
      const float x = l4d_x01(o[0], d[0], zj, M.bound), y = l4d_x01(o[1], d[1], zj, M.bound), z = l4d_x01(o[2], d[2], zj, M.bound);
      FeatSink sink;
      sink.feat = saved ? sv.feat : nullptr; sink.P = sv.P; sink.p = p; sink.dense = nullptr;
      float sigma, h0, geo[L4D_GEO], fl[6];
      l4d_density_sample(M, F, x, y, z, xb, 1, sink, saved ? sv.flow_in + p : nullptr, sv.P, sigma, h0, geo, fl);
      const float alpha = l4d_alpha(M, delta, sigma);
      const float T = carry;
      carry *= (1.0f - alpha) + 1e-15f;
      const float w = alpha * T;
      float a0 = 0.f, a1 = 0.f;
      if (w > 1e-4f) { a0 = l4d_attr_net(M, 0, cdir, geo, xb, 1); a1 = l4d_attr_net(M, 1, cdir, geo, xb, 1); }
      pd += w * zj; p0 += w * a0; p1 += w * a1; pw += w;
      if (saved) {      // flow as the split pipeline saves it (the warped positions of the sample)
        sv.sigma[p] = sigma; sv.attr[p] = a0; sv.attr[sv.P + p] = a1;
        for (int k = 0; k < 6; ++k) sv.flow[(size_t)k * sv.P + p] = fl[k];
      }
      if (weights) weights[p] = w;
      if (zvals) zvals[p] = zj;
    }
    depth[ray] = pd; image[2 * ray] = p0; image[2 * ray + 1] = p1; wsum[ray] = pw;
  }
  return L4D_OK;
}

// ---- cooperative pieces as plain loops ---------------------------------------------------
static void outer_accum(const float* TA, const float* TB, int NT, int K, float* dW) {
  for (int m = 0; m < NT; ++m)
    for (int k = 0; k < K; ++k) {
      const float a = TA[(size_t)m * L4D_TILE_LD + k];
      if (a == 0.f) continue;
      for (int j = 0; j < 64; ++j) dW[(size_t)k * 64 + j] += a * TB[(size_t)m * L4D_TILE_LD + j];
    }
}
static void colsum(const float* T, int NT, float* out) {
  for (int j = 0; j < 64; ++j) {
    float s = 0.f;
    for (int m = 0; m < NT; ++m) s += T[(size_t)m * L4D_TILE_LD + j];
    out[j] += s;
  }
}

// ---- backward (mirror of k_render_bwd) --------------------------------------------------
extern "C" int hs_render_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const L4DRays* rays,
                                  void* saved, const float* g_depth, const float* g_image, const float* g_wsum,
                                  const float* g_weights, const L4DMasterGrads* grads, void* grad_work) {
  int rc = check_config(cfg);
  if (rc) return rc;
  DevModel M;
  build_model(cfg, staged, M);
  DevGrads G;
  // rays->reserved bit 1 (host-sim only): use the slice-independent dynamic-hash accumulators of the split pipeline
  // (DevGrads::hd_comb) and fold them afterwards exactly like k_fold_dynamic does
  const bool comb = (rays->reserved & 2u) != 0;
  build_grads(cfg, grads, grad_work, G, comb);
  std::vector<float> con_store;          // comb also runs the time planes through the contracted rows + gradient rows + fold
  if (comb) { contract_for_frame(cfg, frame, M, con_store); for (int p = 0; p < 3; ++p) for (int q = 0; q < 3; ++q) M.hd_con[p][q] = nullptr; }
  if (comb) G.hf_comb = nullptr;          // the flow-grid accumulator belongs to k_bwd_flowgrid (no host mirror)
  const L4DFrame& F = *frame;
  const uint32_t S = rays->n_steps;
  const int NT = L4D_NT;
  SavedView sv = saved_view(cfg, saved, rays->n_rays, S);
  const RaySampling rs = l4d_make_sampling(M.near_lidar, M.far_lidar, S, rays->perturb, rays->seed);
  const int n_tiles = (int)((S + NT - 1) / NT);
  const float kk = M.active_sensor ? 2.f : 1.f;
  const int n_chunks = (int)(M.sigma_in_pad + 63) / 64;
  std::vector<float> TA((size_t)NT * L4D_TILE_LD), TB((size_t)NT * L4D_TILE_LD), xbuf((size_t)NT * 64), hidden((size_t)NT * 64);
  std::vector<BwSample> st(NT);
  std::vector<uint32_t> m1a(NT), m1b(NT);
  for (uint32_t ray = 0; ray < rays->n_rays; ++ray) {
    const float* o = rays->rays_o + 3 * ray;
    const float* d = rays->rays_d + 3 * ray;
    const float gd = g_depth[ray], gi0 = g_image[2 * ray], gi1 = g_image[2 * ray + 1];
    const float gws = g_wsum ? g_wsum[ray] : 0.f;
    const uint64_t rg = rays->ray_offset + ray;
    float enc[L4D_ENC], cdir[128], csum[128];
    for (int i = 0; i < L4D_ENC; ++i) enc[i] = l4d_freq(d[i / 24], (i % 24) >> 1, i & 1);
    for (int i = 0; i < 128; ++i) { cdir[i] = l4d_attr_cdir(M, i >> 6, i & 63, enc); csum[i] = 0.f; }
    // transmittance, weights for the whole ray (sequential cumprod as the reference)
    std::vector<float> zs(S), dl(S), al(S), Tv(S), wv(S), gw(S), suf(S);
    float carry = 1.f;
    for (uint32_t j = 0; j < S; ++j) {
      const size_t p = (size_t)ray * S + j;
      zs[j] = l4d_z(rs, rg, j);
      dl[j] = (j + 1 < S) ? (l4d_z(rs, rg, j + 1) - zs[j]) : rs.sample_dist;
      al[j] = l4d_alpha(M, dl[j], sv.sigma[p]);
      Tv[j] = carry;
      carry *= (1.0f - al[j]) + 1e-15f;
      wv[j] = al[j] * Tv[j];
      gw[j] = gd * zs[j] + gi0 * sv.attr[p] + gi1 * sv.attr[sv.P + p] + gws + (g_weights ? g_weights[p] : 0.f);
    }
    float run = 0.f;
    for (int j = (int)S - 1; j >= 0; --j) { suf[j] = run; run += gw[j] * wv[j]; }

    for (int t = n_tiles - 1; t >= 0; --t) {
      for (int m = 0; m < NT; ++m) {
        BwSample& s = st[m];
        const uint32_t j = (uint32_t)t * NT + m;
        memset(&s, 0, sizeof(s));
        s.active = j < S;
        if (s.active) {
          s.x = l4d_x01(o[0], d[0], zs[j], M.bound); s.y = l4d_x01(o[1], d[1], zs[j], M.bound); s.z = l4d_x01(o[2], d[2], zs[j], M.bound);
          const float v = (1.0f - al[j]) + 1e-15f;
          const float dalpha = gw[j] * Tv[j] - suf[j] / v;
          s.dsigma = dalpha * (kk * dl[j] * M.density_scale) * (1.0f - al[j]);
          s.masked = wv[j] > 1e-4f;
          if (s.masked) { s.da[0] = wv[j] * gi0; s.da[1] = wv[j] * gi1; }
        }
      }
      auto P = [&](int m) { size_t j = (size_t)t * NT + m; return (size_t)ray * S + (j < S ? j : 0); };
#define XB(m) (xbuf.data() + (size_t)(m) * 64)
#define TAR(m) (TA.data() + (size_t)(m) * L4D_TILE_LD)
#define TBR(m) (TB.data() + (size_t)(m) * L4D_TILE_LD)
#define HID(m) (hidden.data() + (size_t)(m) * 64)
      for (int m = 0; m < NT; ++m) {
        l4d_bw_flow_fwd(M, st[m], sv.flow_in + P(m), sv.P, XB(m), 1);
        l4d_bw_sigma_fwd(M, st[m], sv.feat + P(m), sv.P, XB(m), 1, HID(m), 1);
      }
      for (int net = 0; net < 2; ++net) {
        for (int m = 0; m < NT; ++m) l4d_bw_attr_a(M, net, st[m], cdir, XB(m), 1, TAR(m), TBR(m), m1a[m], m1b[m]);
        colsum(TB.data(), NT, G.att_w3[net]);
        for (int m = 0; m < NT; ++m) l4d_bw_attr_b(XB(m), 1, TBR(m));
        outer_accum(TA.data(), TB.data(), NT, 64, G.att_w2t[net]);
        for (int m = 0; m < NT; ++m) l4d_bw_attr_c(M, net, st[m], XB(m), 1, TAR(m), TBR(m), m1a[m], m1b[m]);
        outer_accum(TA.data(), TB.data(), NT, 16, G.att_w1t[net] + (size_t)L4D_ENC * 64);
        colsum(TB.data(), NT, csum + net * 64);
      }
      for (int m = 0; m < NT; ++m) l4d_bw_sigma_a(M, st[m], HID(m), 1, XB(m), 1, TAR(m), TBR(m));
      outer_accum(TA.data(), TB.data(), NT, 16, G.sig_w2);
      for (int m = 0; m < NT; ++m) l4d_bw_sigma_b(M, st[m], XB(m), 1, TBR(m));
      for (int c = 0; c < n_chunks; ++c) {
        for (int m = 0; m < NT; ++m) l4d_bw_sigma_c(M, st[m], sv.feat + P(m), sv.P, c, TAR(m));
        const int rows = std::min(64, (int)M.sigma_in_pad - c * 64);
        outer_accum(TA.data(), TB.data(), NT, rows, G.sig_w1t + (size_t)c * 64 * 64);
      }
      for (int m = 0; m < NT; ++m) { if (comb) l4d_bw_scatter<true>(M, F, G, st[m]); else l4d_bw_scatter<false>(M, F, G, st[m]); }
      for (int m = 0; m < NT; ++m) l4d_bw_flow_a(M, st[m], sv.flow_in + P(m), sv.P, st[m].dflow, XB(m), 1, TAR(m), TBR(m));
      outer_accum(TA.data(), TB.data(), NT, 8, G.flo_w2);
      for (int m = 0; m < NT; ++m) l4d_bw_flow_b(M, st[m], st[m].dflow, XB(m), 1, TAR(m), TBR(m));
      outer_accum(TA.data(), TB.data(), NT, 64, G.flo_w1t);
      for (int m = 0; m < NT; ++m) l4d_bw_flow_c(M, F, G, st[m], sv.flow_in + P(m), sv.P, XB(m), 1, TAR(m), TBR(m));
      outer_accum(TA.data(), TB.data(), NT, 16, G.flo_w0t);
    }
    for (int net = 0; net < 2; ++net)
      for (int r = 0; r < L4D_ENC + 9; ++r)
        for (int j = 0; j < 64; ++j) {
          const float cs = csum[net * 64 + j];
          if (r < L4D_ENC) G.att_w1t[net][(size_t)r * 64 + j] += enc[r] * cs;
          else G.att_w1t[net][(size_t)(M.attr_in_dim + (r - L4D_ENC)) * 64 + j] += cs;
        }
  }
  if (comb) {          // mirror of k_fold_planes (l4d_kernels.cu)
    const L4DTimeQuery* qs[3] = {&frame->cur, &frame->fwd, &frame->bwd};
    const bool live[3] = {true, frame->has_fwd != 0, frame->has_bwd != 0};
    for (uint32_t s = 0; s < cfg->n_plane_scales; ++s)
      for (int t = 0; t < 3; ++t) {
        const int R = (int)cfg->plane_res[s];
        float* Gp = G.planes_cl[s][t == 0 ? 2 : (t == 1 ? 4 : 5)];
        for (int q = 0; q < 3; ++q) {
          if (!live[q]) continue;
          const Bilerp bl = l4d_bilerp(0.f, 2, qs[q]->tau, (int)cfg->time_resolution);
          float* row = G.pl_rows[s][t][q];
          for (int i = 0; i < R * 8; ++i) {
            const float v = row[i];
            if (v == 0.f) continue;
            Gp[(size_t)bl.y0 * R * 8 + i] = fmaf(bl.wy0, v, Gp[(size_t)bl.y0 * R * 8 + i]);
            if (bl.wy1 != 0.f) Gp[(size_t)bl.y1 * R * 8 + i] = fmaf(bl.wy1, v, Gp[(size_t)bl.y1 * R * 8 + i]);
            row[i] = 0.f;
          }
        }
      }
  }
  if (comb) {          // mirror of k_fold_dynamic (l4d_kernels.cu)
    const bool single = F.cur.single != 0;
    const float w_lo = single ? 1.0f : F.cur.w_lo, w_hi = F.cur.w_hi;
    for (int p = 0; p < 3; ++p) {
      const size_t n = (size_t)cfg->hash_dynamic[p].offset[cfg->hash_dynamic[p].n_levels];
      float* c = G.hd_comb[p];
      float* glo = G.hd[p][F.cur.slice_lo];
      float* ghi = single ? nullptr : G.hd[p][F.cur.slice_hi];
      for (size_t i = 0; i < n; ++i) {
        if (c[i] == 0.f) continue;
        for (int k = 0; k < 4; ++k) {
          const float e = c[i] * F.cur.basis[k];
          glo[4 * i + k] = fmaf(w_lo, e, glo[4 * i + k]);
          if (ghi) ghi[4 * i + k] = fmaf(w_hi, e, ghi[4 * i + k]);
        }
        c[i] = 0.f;
      }
    }
  }
  return L4D_OK;
}

// ---- flow forward / backward ---------------------------------------------------------------
extern "C" int hs_flow_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x, uint32_t n,
                               float* flow, float* saved) {
  DevModel M;
  build_model(cfg, staged, M);
  for (uint32_t i = 0; i < n; ++i) {
    float xb[64];
    const float b2 = L4D_MUL(2.0f, M.bound);
    const float px = L4D_DIV(L4D_ADD(x[3 * i], M.bound), b2), py = L4D_DIV(L4D_ADD(x[3 * i + 1], M.bound), b2),
                pz = L4D_DIV(L4D_ADD(x[3 * i + 2], M.bound), b2);
    l4d_flow_inputs(M, frame->flow_basis, px, py, pz, xb, 1, saved ? saved + i : nullptr, n);
    float fl[8];
    uint32_t a, b, c, d;
    l4d_flow_mlp(M, xb, 1, fl, a, b, c, d);
    for (int k = 0; k < 6; ++k) flow[(size_t)i * 6 + k] = fl[k];
  }
  return L4D_OK;
}

extern "C" int hs_flow_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x, uint32_t n,
                                const float* saved, const float* g_flow, const L4DMasterGrads* grads, void* grad_work) {
  DevModel M;
  build_model(cfg, staged, M);
  DevGrads G;
  memset(&G, 0, sizeof(G));
  GradWorkLayout L = grad_work_layout(cfg);
  char* b = (char*)grad_work;
  G.hf = grads->flow_grid;
  G.flo_w0t = (float*)(b + L.flo_w0t); G.flo_w1t = (float*)(b + L.flo_w1t); G.flo_w2 = (float*)(b + L.flo_w2);
  const int NT = L4D_NT;
  std::vector<float> TA((size_t)NT * L4D_TILE_LD), TB((size_t)NT * L4D_TILE_LD), xbuf((size_t)NT * 64);
  std::vector<BwSample> st(NT);
  std::vector<float> gg((size_t)NT * 6);
  for (uint32_t base = 0; base < n; base += NT) {
    for (int m = 0; m < NT; ++m) {
      BwSample& s = st[m];
      memset(&s, 0, sizeof(s));
      const uint32_t i = base + m;
      s.active = i < n;
      for (int k = 0; k < 6; ++k) gg[m * 6 + k] = 0.f;
      if (s.active) {
        const float b2 = L4D_MUL(2.0f, M.bound);
        s.x = L4D_DIV(L4D_ADD(x[3 * i], M.bound), b2); s.y = L4D_DIV(L4D_ADD(x[3 * i + 1], M.bound), b2);
        s.z = L4D_DIV(L4D_ADD(x[3 * i + 2], M.bound), b2);
        for (int k = 0; k < 6; ++k) gg[m * 6 + k] = g_flow[(size_t)i * 6 + k];
      }
    }
    auto I = [&](int m) { return (size_t)(base + m < n ? base + m : 0); };
    for (int m = 0; m < NT; ++m) {
      l4d_bw_flow_fwd(M, st[m], saved + I(m), n, XB(m), 1);
      l4d_bw_flow_a(M, st[m], saved + I(m), n, &gg[m * 6], XB(m), 1, TAR(m), TBR(m));
    }
    outer_accum(TA.data(), TB.data(), NT, 8, G.flo_w2);
    for (int m = 0; m < NT; ++m) l4d_bw_flow_b(M, st[m], &gg[m * 6], XB(m), 1, TAR(m), TBR(m));
    outer_accum(TA.data(), TB.data(), NT, 64, G.flo_w1t);
    for (int m = 0; m < NT; ++m) l4d_bw_flow_c(M, *frame, G, st[m], saved + I(m), n, XB(m), 1, TAR(m), TBR(m));
    outer_accum(TA.data(), TB.data(), NT, 16, G.flo_w0t);
  }
  return L4D_OK;
}

// ---- debug entry points ------------------------------------------------------------------
extern "C" int hs_hash_indices(const L4DConfig* cfg, uint32_t grid_id, uint32_t level, const float* x, uint32_t n,
                               uint32_t* idx, float* w) {
  const L4DGrid& g = grid_id == 0 ? cfg->hash_static : (grid_id == 4 ? cfg->flow : cfg->hash_dynamic[grid_id - 1]);
  DevGrid d;
  fill_grid(d, g);
  for (uint32_t i = 0; i < n; ++i) {
    if (g.n_dims == 3) l4d_corners3(d, level, x[3 * i], x[3 * i + 1], x[3 * i + 2], idx + 8 * i, w + 8 * i);
    else l4d_corners2(d, level, x[2 * i], x[2 * i + 1], idx + 4 * i, w + 4 * i);
  }
  return L4D_OK;
}

// l4d_bilerp of n coordinate pairs: idx [n][4] = x0 x1 y0 y1, w [n][6] = wx0 wx1 wy0 wy1 gx_mult gy_mult
extern "C" int hs_bilerp(const float* cx, const float* cy, uint32_t n, int W, int H, int* idx, float* w) {
  for (uint32_t i = 0; i < n; ++i) {
    const Bilerp b = l4d_bilerp(cx[i], W, cy[i], H);
    idx[4 * i] = b.x0; idx[4 * i + 1] = b.x1; idx[4 * i + 2] = b.y0; idx[4 * i + 3] = b.y1;
    w[6 * i] = b.wx0; w[6 * i + 1] = b.wx1; w[6 * i + 2] = b.wy0; w[6 * i + 3] = b.wy1;
    w[6 * i + 4] = b.gx_mult; w[6 * i + 5] = b.gy_mult;
  }
  return L4D_OK;
}

extern "C" int hs_density_forward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x, uint32_t n,
                                  float* sigma, float* geo, float* features, float* flow) {
  DevModel M;
  build_model(cfg, staged, M);
  for (uint32_t i = 0; i < n; ++i) {
    float xb[64];
    const float b2 = L4D_MUL(2.0f, M.bound);
    const float px = L4D_DIV(L4D_ADD(x[3 * i], M.bound), b2), py = L4D_DIV(L4D_ADD(x[3 * i + 1], M.bound), b2),
                pz = L4D_DIV(L4D_ADD(x[3 * i + 2], M.bound), b2);
    FeatSink sink;
    sink.feat = nullptr; sink.P = 0; sink.p = 0;
    sink.dense = features ? features + (size_t)i * M.sigma_in_dim : nullptr;
    float sg, h0, g[L4D_GEO], fl[6];
    l4d_density_sample(M, *frame, px, py, pz, xb, 1, sink, nullptr, 0, sg, h0, g, fl);
    sigma[i] = sg;
    for (int k = 0; k < L4D_GEO; ++k) geo[(size_t)i * L4D_GEO + k] = g[k];
    if (flow) for (int k = 0; k < 6; ++k) flow[(size_t)i * 6 + k] = fl[k];
  }
  return L4D_OK;
}
