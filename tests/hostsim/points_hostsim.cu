// points_hostsim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// Host mirrors of the explicit-point kernels of lidar4d_b200/csrc/l4d_points.cuh (LiDAR4D.density / .attribute with a
// backward), built like tests/hostsim/hostsim.cu: the __host__ __device__ per-sample phases of l4d_core.cuh +
// l4d_bwd.cuh driven by plain loops over tiles of L4D_NT points, cooperative products replaced by loops.  Staging and
// unstaging come from the host-sim library (hs_stage_params / hs_unstage_grads); all pointers are HOST pointers.
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
extern "C" const char* hs_points_last_error(void) { return g_err; }

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
#define XB(m) (xbuf.data() + (size_t)(m) * 64)
#define TAR(m) (TA.data() + (size_t)(m) * L4D_TILE_LD)
#define TBR(m) (TB.data() + (size_t)(m) * L4D_TILE_LD)
#define HID(m) (hidden.data() + (size_t)(m) * 64)

// ---- explicit-point density / attribute with a backward ---------------------------------------------------------
extern "C" size_t hs_density_saved_bytes(const L4DConfig* cfg, uint32_t n) {
  return check_config(cfg) == L4D_OK ? density_saved_layout(cfg, n).total : 0;
}

// mirror of k_density_train: l4d_density_sample with the flow-MLP inputs and the features saved as SoA planes
extern "C" int hs_density_forward_ex(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x, uint32_t n,
                                     float* sigma, float* geo, float* features, float* flow, void* saved) {
  int rc = check_config(cfg);
  if (rc) return rc;
  DevModel M;
  build_model(cfg, staged, M);
  const DensitySavedLayout L = density_saved_layout(cfg, n);
  float* flow_in = saved ? (float*)((char*)saved + L.flow_in) : nullptr;
  float* feat = saved ? (float*)((char*)saved + L.feat) : nullptr;
  for (uint32_t i = 0; i < n; ++i) {
    float xb[64];
    const float b2 = L4D_MUL(2.0f, M.bound);
    const float px = L4D_DIV(L4D_ADD(x[3 * i], M.bound), b2), py = L4D_DIV(L4D_ADD(x[3 * i + 1], M.bound), b2),
                pz = L4D_DIV(L4D_ADD(x[3 * i + 2], M.bound), b2);
    FeatSink sink;
    sink.feat = feat; sink.P = n; sink.p = i;
    sink.dense = features ? features + (size_t)i * M.sigma_in_dim : nullptr;
    float sg, h0, g[L4D_GEO], fl[6];
    l4d_density_sample(M, *frame, px, py, pz, xb, 1, sink, flow_in ? flow_in + i : nullptr, n, sg, h0, g, fl);
    sigma[i] = sg;
    for (int k = 0; k < L4D_GEO; ++k) geo[(size_t)i * L4D_GEO + k] = g[k];
    if (flow) for (int k = 0; k < 6; ++k) flow[(size_t)i * 6 + k] = fl[k];
  }
  return L4D_OK;
}

// mirror of k_density_bwd: B0, B1, B3 (dsigma = g_sigma[i], dgeo = g_geo[i]), B4, B5 per tile of L4D_NT points
extern "C" int hs_density_backward(const L4DConfig* cfg, const void* staged, const L4DFrame* frame, const float* x, uint32_t n,
                                   const void* saved, const float* g_sigma, const float* g_geo, const L4DMasterGrads* grads,
                                   void* grad_work) {
  int rc = check_config(cfg);
  if (rc) return rc;
  DevModel M;
  build_model(cfg, staged, M);
  DevGrads G;
  build_grads(cfg, grads, grad_work, G);
  const L4DFrame& F = *frame;
  const DensitySavedLayout L = density_saved_layout(cfg, n);
  const float* flow_in = (const float*)((const char*)saved + L.flow_in);
  const float* feat = (const float*)((const char*)saved + L.feat);
  const int NT = L4D_NT;
  const int n_chunks = (int)(M.sigma_in_pad + 63) / 64;
  const bool flow_live = F.has_fwd || F.has_bwd;
  std::vector<float> TA((size_t)NT * L4D_TILE_LD), TB((size_t)NT * L4D_TILE_LD), xbuf((size_t)NT * 64), hidden((size_t)NT * 64);
  std::vector<BwSample> st(NT);
  for (uint32_t base = 0; base < n; base += NT) {
    auto I = [&](int m) { return (size_t)(base + m < n ? base + m : 0); };
    for (int m = 0; m < NT; ++m) {
      BwSample& s = st[m];
      memset(&s, 0, sizeof(s));
      const uint32_t i = base + m;
      s.active = i < n;
      if (s.active) {
        const float b2 = L4D_MUL(2.0f, M.bound);
        s.x = L4D_DIV(L4D_ADD(x[3 * i], M.bound), b2); s.y = L4D_DIV(L4D_ADD(x[3 * i + 1], M.bound), b2);
        s.z = L4D_DIV(L4D_ADD(x[3 * i + 2], M.bound), b2);
      }
      l4d_bw_flow_fwd(M, s, flow_in + I(m), n, XB(m), 1);
      l4d_bw_sigma_fwd(M, s, feat + I(m), n, XB(m), 1, HID(m), 1);
      if (s.active) {
        s.dsigma = g_sigma ? g_sigma[i] : 0.f;
        for (int k = 0; k < L4D_GEO; ++k) s.dgeo[k] = g_geo ? g_geo[(size_t)i * L4D_GEO + k] : 0.f;
      }
    }
    for (int m = 0; m < NT; ++m) l4d_bw_sigma_a(M, st[m], HID(m), 1, XB(m), 1, TAR(m), TBR(m));
    outer_accum(TA.data(), TB.data(), NT, 16, G.sig_w2);
    for (int m = 0; m < NT; ++m) l4d_bw_sigma_b(M, st[m], XB(m), 1, TBR(m));
    for (int c = 0; c < n_chunks; ++c) {
      for (int m = 0; m < NT; ++m) l4d_bw_sigma_c(M, st[m], feat + I(m), n, c, TAR(m));
      const int rows = std::min(64, (int)M.sigma_in_pad - c * 64);
      outer_accum(TA.data(), TB.data(), NT, rows, G.sig_w1t + (size_t)c * 64 * 64);
    }
    for (int m = 0; m < NT; ++m) l4d_bw_scatter<false>(M, F, G, st[m]);
    if (!flow_live) continue;
    for (int m = 0; m < NT; ++m) l4d_bw_flow_a(M, st[m], flow_in + I(m), n, st[m].dflow, XB(m), 1, TAR(m), TBR(m));
    outer_accum(TA.data(), TB.data(), NT, 8, G.flo_w2);
    for (int m = 0; m < NT; ++m) l4d_bw_flow_b(M, st[m], st[m].dflow, XB(m), 1, TAR(m), TBR(m));
    outer_accum(TA.data(), TB.data(), NT, 64, G.flo_w1t);
    for (int m = 0; m < NT; ++m) l4d_bw_flow_c(M, F, G, st[m], flow_in + I(m), n, XB(m), 1, TAR(m), TBR(m));
    outer_accum(TA.data(), TB.data(), NT, 16, G.flo_w0t);
  }
  return L4D_OK;
}

// mirror of k_attribute_bwd: per-point direction term and encoding rows, B2 steps a/b/c with masked = mask[i], da = g_out[i]
extern "C" int hs_attribute_backward(const L4DConfig* cfg, const void* staged, const float* d, const float* geo,
                                     const unsigned char* mask, uint32_t n, const float* g_out, float* g_geo,
                                     const L4DMasterGrads* grads, void* grad_work) {
  int rc = check_config(cfg);
  if (rc) return rc;
  DevModel M;
  build_model(cfg, staged, M);
  DevGrads G;
  build_grads(cfg, grads, grad_work, G);
  const int NT = L4D_NT;
  std::vector<float> TA((size_t)NT * L4D_TILE_LD), TB((size_t)NT * L4D_TILE_LD), xbuf((size_t)NT * 64);
  std::vector<float> enc((size_t)NT * L4D_ENC), cdir((size_t)NT * 128);
  std::vector<BwSample> st(NT);
  std::vector<uint32_t> m1a(NT), m1b(NT);
  float csum[128] = {0.f};
  for (uint32_t base = 0; base < n; base += NT) {
    for (int m = 0; m < NT; ++m) {
      BwSample& s = st[m];
      memset(&s, 0, sizeof(s));
      const uint32_t i = base + m;
      s.active = i < n;
      s.masked = s.active && (!mask || mask[i]);
      float* e = &enc[(size_t)m * L4D_ENC];
      for (int k = 0; k < L4D_ENC; ++k) e[k] = s.masked ? l4d_freq(d[3 * (size_t)i + k / 24], (k % 24) >> 1, k & 1) : 0.f;
      for (int k = 0; k < 128; ++k) cdir[(size_t)m * 128 + k] = s.masked ? l4d_attr_cdir(M, k >> 6, k & 63, e) : 0.f;
      if (!s.masked) continue;
      for (int net = 0; net < 2; ++net) s.da[net] = g_out[2 * (size_t)i + net];
      for (int k = 0; k < L4D_GEO; ++k) s.geo[k] = geo[(size_t)i * L4D_GEO + k];
    }
    for (int net = 0; net < 2; ++net) {
      for (int m = 0; m < NT; ++m) l4d_bw_attr_a(M, net, st[m], &cdir[(size_t)m * 128], XB(m), 1, TAR(m), TBR(m), m1a[m], m1b[m]);
      colsum(TB.data(), NT, G.att_w3[net]);
      for (int m = 0; m < NT; ++m) l4d_bw_attr_b(XB(m), 1, TBR(m));
      outer_accum(TA.data(), TB.data(), NT, 64, G.att_w2t[net]);
      for (int m = 0; m < NT; ++m) l4d_bw_attr_c(M, net, st[m], XB(m), 1, TAR(m), TBR(m), m1a[m], m1b[m]);
      outer_accum(TA.data(), TB.data(), NT, 16, G.att_w1t[net] + (size_t)L4D_ENC * 64);
      colsum(TB.data(), NT, csum + net * 64);
      // encoding rows: per-point outer products enc (x) dh1 (TB rows hold dh1 after step c)
      for (int m = 0; m < NT; ++m)
        for (int k = 0; k < L4D_ENC; ++k) {
          const float a = enc[(size_t)m * L4D_ENC + k];
          if (a == 0.f) continue;
          for (int j = 0; j < 64; ++j) G.att_w1t[net][(size_t)k * 64 + j] += a * TBR(m)[j];
        }
    }
    for (int m = 0; m < NT; ++m) {
      const uint32_t i = base + m;
      if (st[m].active && g_geo)
        for (int k = 0; k < L4D_GEO; ++k) g_geo[(size_t)i * L4D_GEO + k] = st[m].masked ? st[m].dgeo[k] : 0.f;
    }
  }
  for (int net = 0; net < 2; ++net)
    for (int k = (int)M.attr_in_dim; k < (int)M.attr_in_pad; ++k)
      for (int j = 0; j < 64; ++j) G.att_w1t[net][(size_t)k * 64 + j] += csum[net * 64 + j];
  return L4D_OK;
}
