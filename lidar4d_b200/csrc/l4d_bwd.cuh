// l4d_bwd.cuh - per-sample phases of the backward pass (host+device, see
// l4d_core.cuh).  The reference has no backward code: it relies on autograd
// over model/renderer.py:98-129 and model/lidar4d.py:139-223; SURVEY.md
// Appendix A.12 derives what is restated here.
//
// Data flow of one tile of NT samples (thread == sample).  "TA"/"TB" are
// shared-memory tiles [NT][LD] in which every thread owns one row; between the
// phases the block runs cooperative outer products  dW += TA^T * TB  (device:
// l4d_kernels.cu; host: plain loops in tests/hostsim).
//
//   B0  flow MLP recompute from saved flow_in           -> flow[6], relu masks
//   B1  sigma MLP recompute from saved features         -> h0, geo, relu mask, hidden (scratch)
//   B2  per attribute net: recompute + backprop         -> dW tiles, dgeo
//   B3  sigma MLP backprop                              -> dW tiles, dh[64]
//   B4  scatter dh through the encoders                 -> table / plane REDs, dflow
//   B5  flow MLP backprop + flow-grid scatter
#pragma once
#include "l4d_core.cuh"

#define L4D_TILE_LD 68     // tile leading dimension: 64 + 4 keeps float4 alignment

struct BwSample {
  bool active;             // sample index < n_steps
  bool masked;             // w > 1e-4
  float x, y, z;           // position in [0,1]^3
  float flow[8];
  uint32_t mf1a, mf1b, mf2a, mf2b;   // flow MLP relu patterns
  uint32_t msa, msb;                 // sigma hidden relu pattern
  float h0;                          // pre-exp sigma output
  float geo[L4D_GEO];
  float dsigma;                      // dL/dsigma from the compositing backward
  float da[2];                       // dL/d(raydrop, intensity) (0 when not masked)
  float dgeo[L4D_GEO];
  float dh[L4D_H];                   // dL/d(sigma hidden pre-activation)
  float dflow[6];
};

// ---- B0: flow MLP forward from the saved Lagrange-contracted inputs -------------------
L4D_HD void l4d_bw_flow_fwd(const DevModel& M, BwSample& s, const float* flow_in, size_t stride,
                            float* xb, int xs) {
#pragma unroll
  for (int k = 0; k < L4D_FLOW_IN; ++k) xb[k * xs] = s.active ? flow_in[(size_t)k * stride] : 0.f;
  l4d_flow_mlp(M, xb, xs, s.flow, s.mf1a, s.mf1b, s.mf2a, s.mf2b);
}

// ---- B1: sigma MLP forward from the saved features --------------------------------------
// writes relu(hidden) to xb[0..64) and to hidden_out (scratch plane, stride hs)
L4D_HD void l4d_bw_sigma_fwd(const DevModel& M, BwSample& s, const float* feat, size_t stride,
                             float* xb, int xs, float* hidden_out, size_t hs) {
  float acc[L4D_H];
  l4d_sigma_hidden_from_feats(M, feat, stride, s.active, acc);
  l4d_relu_store(acc, xb, xs, s.msa, s.msb);
  if (s.active) {
#pragma unroll
    for (int k = 0; k < L4D_H; ++k) hidden_out[(size_t)k * hs] = xb[k * xs];
  }
  float out[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) out[k] = 0.f;
  l4d_layer_small<16>(out, xb, xs, L4D_H, M.sig_w2t);
  s.h0 = out[0];
#pragma unroll
  for (int k = 0; k < L4D_GEO; ++k) { s.geo[k] = out[1 + k]; s.dgeo[k] = 0.f; }
}

// ---- B2: one attribute head.  Split in three steps around the cooperative products. ----
// step a: forward; TA row <- h1 ; TB row <- d_o * h2 (for dw3 = colsum) ; returns d_o and keeps
//         dh2 (masked by relu2) in xb[0..64)
L4D_HD void l4d_bw_attr_a(const DevModel& M, int net, BwSample& s, const float* cdir, float* xb, int xs,
                          float* ta_row, float* tb_row, uint32_t& m1a, uint32_t& m1b) {
  float y[L4D_H];
  const bool on = s.active && s.masked;
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = cdir[net * L4D_H + k];
#pragma unroll
  for (int k = 0; k < L4D_GEO; ++k) xb[k * xs] = s.geo[k];
  l4d_layer64(y, xb, xs, L4D_GEO, M.att_w1t[net] + (size_t)L4D_ENC * L4D_H);
  l4d_relu_store(y, xb, xs, m1a, m1b);
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) ta_row[k] = on ? xb[k * xs] : 0.f;
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) y[k] = 0.f;
  l4d_layer64(y, xb, xs, L4D_H, M.att_w2t[net]);
  uint32_t m2a = 0u, m2b = 0u;
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) {
    bool p = y[k] > 0.f;
    y[k] = p ? y[k] : 0.f;
    if (k < 32) m2a |= p ? (1u << k) : 0u; else m2b |= p ? (1u << (k - 32)) : 0u;
  }
  const float a = l4d_sigmoid(l4d_dot64(y, M.att_w3[net]));
  const float d_o = on ? s.da[net] * a * (1.0f - a) : 0.f;
#pragma unroll
  for (int q = 0; q < L4D_H / 4; ++q) {
    float4 w3 = l4d_ld4(M.att_w3[net] + 4 * q);
    const float wv[4] = {w3.x, w3.y, w3.z, w3.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = 4 * q + i;
      tb_row[k] = d_o * y[k];
      xb[k * xs] = l4d_bit(m2a, m2b, k) ? wv[i] * d_o : 0.f;     // dh2
    }
  }
}
// step b: (after dw3 colsum) TB row <- dh2
L4D_HD void l4d_bw_attr_b(float* xb, int xs, float* tb_row) {
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) tb_row[k] = xb[k * xs];
}
// step c: (after dW2t product) dh1 = (W2^T dh2) * relu1 ; TB row <- dh1 ; TA row[0..16) <- geo|0 ;
//         dgeo += W1g^T dh1
L4D_HD void l4d_bw_attr_c(const DevModel& M, int net, BwSample& s, float* xb, int xs,
                          float* ta_row, float* tb_row, uint32_t m1a, uint32_t m1b) {
  float d[L4D_H];
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) d[k] = 0.f;
  l4d_layer64(d, xb, xs, L4D_H, M.att_w2[net]);          // native rows [o][k]: d[k] += dh2[o] W2[o][k]
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) {
    d[k] = l4d_bit(m1a, m1b, k) ? d[k] : 0.f;
    tb_row[k] = d[k];
  }
  const bool on = s.active && s.masked;
#pragma unroll
  for (int k = 0; k < 16; ++k) ta_row[k] = (on && k < L4D_GEO) ? s.geo[k] : 0.f;
#pragma unroll
  for (int k = 0; k < L4D_GEO; ++k) s.dgeo[k] += l4d_dot64(d, M.att_w1t[net] + (size_t)(L4D_ENC + k) * L4D_H);
}

// ---- B3: sigma MLP backprop ------------------------------------------------------------
// step a: TA row[0..16) <- dout ; TB row <- hidden (from scratch) ; xb[0..16) <- dout
L4D_HD void l4d_bw_sigma_a(const DevModel& M, BwSample& s, const float* hidden, size_t hs, float* xb, int xs,
                           float* ta_row, float* tb_row) {
  // trunc_exp backward: g * exp(clamp(x,-15,15))  (activation.py:17)
  const float d0 = s.active ? s.dsigma * expf(fminf(fmaxf(s.h0, -15.f), 15.f)) : 0.f;
  ta_row[0] = d0;
  xb[0] = d0;
#pragma unroll
  for (int k = 0; k < L4D_GEO; ++k) {
    const float v = s.active ? s.dgeo[k] : 0.f;
    ta_row[1 + k] = v;
    xb[(1 + k) * xs] = v;
  }
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) tb_row[k] = s.active ? hidden[(size_t)k * hs] : 0.f;
}
// step b: dh = (W2^T dout) * relu ; TB row <- dh
L4D_HD void l4d_bw_sigma_b(const DevModel& M, BwSample& s, const float* xb, int xs, float* tb_row) {
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) s.dh[k] = 0.f;
  l4d_layer64(s.dh, xb, xs, 16, M.sig_w2);               // native [16][64]
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) {
    s.dh[k] = l4d_bit(s.msa, s.msb, k) ? s.dh[k] : 0.f;
    tb_row[k] = s.dh[k];
  }
}
// step c (per 64-wide chunk of the input): TA row <- features[chunk]
L4D_HD void l4d_bw_sigma_c(const DevModel& M, const BwSample& s, const float* feat, size_t stride, int chunk,
                           float* ta_row) {
  for (int k = 0; k < L4D_H; ++k) {
    const int r = chunk * L4D_H + k;
    float v = 0.f;
    if (s.active && r < (int)M.sigma_in_pad) v = r < (int)M.sigma_in_dim ? feat[(size_t)r * stride] : 1.0f;
    ta_row[k] = v;
  }
}

// ---- B4: scatter dh through the encoders ------------------------------------------------
// ---- warp-level pre-aggregation of plane gradients (device only) ---------------------------------
// Lanes of a warp are consecutive samples of a ray: they hit the same plane texel in long runs (a
// warp spans ~5 texels at resolution 256, <1 at 32).  The SM retires only ~1 fp32 RED per 1.3 cycles
// (a RED.F32x4 counts as 4) and plane gradients are half of all atomics of the backward, so each run
// is summed with a segmented warp scan and only its last lane issues the REDs.
#if defined(__CUDACC__)
// warp-collective helpers: device code.  tests/hostsim/warpsim.cu (test infrastructure) compiles them for the host with the warp
// intrinsics redirected to a 32-thread lockstep emulator, which is why the qualifier is a macro.
#ifndef L4D_WARP_FN
#define L4D_WARP_FN __device__ __forceinline__
#endif
struct WarpRuns {
  int dist;       // lane - first lane of this lane's run of equal keys
  int maxdist;    // longest run of the warp - 1 (warp-uniform): the scans stop after ceil(log2(maxdist+1)) steps
  bool tail;      // last lane of its run
  unsigned mask;  // the lanes of this lane's run
};
L4D_WARP_FN WarpRuns l4d_warp_runs(int key) {
  const unsigned lane = threadIdx.x & 31u;
  const int prev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool head = (lane == 0u) || (prev != key);
  const unsigned heads = __ballot_sync(0xffffffffu, head);
  const unsigned below = heads & (0xffffffffu >> (31u - lane));
  WarpRuns r;
  const int first = 31 - __clz(below);
  r.dist = (int)lane - first;
  r.maxdist = (int)__reduce_max_sync(0xffffffffu, (unsigned)r.dist);
  r.tail = (lane == 31u) || ((heads >> (lane + 1u)) & 1u);
  const unsigned above = lane == 31u ? 0u : (heads & (0xffffffffu << (lane + 1u)));      // heads of later runs
  const int last = above ? (__ffs(above) - 2) : 31;                                         // last lane of this run
  r.mask = (0xffffffffu >> (31 - last)) & (0xffffffffu << first);
  return r;
}
// inclusive segmented scans of 8 values at once (8 independent shuffles per step); the tail lane of a run ends up
// with the run's sums
L4D_WARP_FN void l4d_seg_sum8(float (&v)[8], const WarpRuns& r) {
  // only as many steps as the longest run of the warp needs (measured against a fixed 5-step scan: 14.2 -> 11.8 ms)
#pragma unroll 1
  for (int d = 1; d <= r.maxdist; d <<= 1) {
    // one FFMA per value instead of FSEL + FADD (the scans are 40 % of this kernel's instructions): fma(t, 1, v) rounds
    // like t + v, fma(t, 0, v) = v for every finite t
    const float take = r.dist >= d ? 1.0f : 0.0f;
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = fmaf(__shfl_up_sync(0xffffffffu, v[c], d), take, v[c]);
  }
}
// all 32 lanes must call; g may be zero for lanes without a contribution
L4D_WARP_FN void l4d_plane_scatter_warp(float* G, int W, const Bilerp& b, const float g[8]) {
  const WarpRuns r = l4d_warp_runs(b.y0 * W + b.x0);
  const float wgt[4] = {b.wx0 * b.wy0, b.wx1 * b.wy0, b.wx0 * b.wy1, b.wx1 * b.wy1};
  const int xs[4] = {b.x0, b.x1, b.x0, b.x1};
  const int ys[4] = {b.y0, b.y0, b.y1, b.y1};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float s[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) s[c] = g[c] * wgt[k];
    l4d_seg_sum8(s, r);
    if (r.tail) {
      float* p = G + ((size_t)ys[k] * W + xs[k]) * 8;
      l4d_red4(p, s[0], s[1], s[2], s[3]);
      l4d_red4(p + 4, s[4], s[5], s[6], s[7]);
    }
  }
}
// time planes: the y (time) weights are the same for every lane, so two sums per channel suffice
L4D_WARP_FN void l4d_plane_scatter_warp_t(float* G, int W, const Bilerp& b, const float g[8]) {
  const WarpRuns r = l4d_warp_runs(b.x0);
  float s0[8], s1[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) { s0[c] = g[c] * b.wx0; s1[c] = g[c] * b.wx1; }
  l4d_seg_sum8(s0, r);
  l4d_seg_sum8(s1, r);
  if (r.tail) {
    float* p00 = G + ((size_t)b.y0 * W + b.x0) * 8;
    float* p01 = G + ((size_t)b.y0 * W + b.x1) * 8;
    float* p10 = G + ((size_t)b.y1 * W + b.x0) * 8;
    float* p11 = G + ((size_t)b.y1 * W + b.x1) * 8;
    l4d_red4(p00, s0[0] * b.wy0, s0[1] * b.wy0, s0[2] * b.wy0, s0[3] * b.wy0);
    l4d_red4(p00 + 4, s0[4] * b.wy0, s0[5] * b.wy0, s0[6] * b.wy0, s0[7] * b.wy0);
    l4d_red4(p01, s1[0] * b.wy0, s1[1] * b.wy0, s1[2] * b.wy0, s1[3] * b.wy0);
    l4d_red4(p01 + 4, s1[4] * b.wy0, s1[5] * b.wy0, s1[6] * b.wy0, s1[7] * b.wy0);
    if (b.wy1 != 0.f) {
      l4d_red4(p10, s0[0] * b.wy1, s0[1] * b.wy1, s0[2] * b.wy1, s0[3] * b.wy1);
      l4d_red4(p10 + 4, s0[4] * b.wy1, s0[5] * b.wy1, s0[6] * b.wy1, s0[7] * b.wy1);
      l4d_red4(p11, s1[0] * b.wy1, s1[1] * b.wy1, s1[2] * b.wy1, s1[3] * b.wy1);
      l4d_red4(p11 + 4, s1[4] * b.wy1, s1[5] * b.wy1, s1[6] * b.wy1, s1[7] * b.wy1);
    }
  }
}
// gradient rows of the contracted time planes (DevGrads::pl_rows): the same run sums, and the tail lane only issues the two
// texels of the row - the time-row weights are applied once per frame by k_fold_planes.  seg: the lane's frame in the launch
// (lanes of different frames write different rows and never share a run; rows are far shorter than 2^16 texels)
L4D_WARP_FN void l4d_row_scatter_warp(float* Grow, const Bilerp& b, const float g[8], int seg = 0) {
  const WarpRuns r = l4d_warp_runs(b.x0 + (seg << 16));
  float s0[8], s1[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) { s0[c] = g[c] * b.wx0; s1[c] = g[c] * b.wx1; }
  l4d_seg_sum8(s0, r);
  l4d_seg_sum8(s1, r);
  if (r.tail) {
    float* p0 = Grow + (size_t)b.x0 * 8;
    float* p1 = Grow + (size_t)b.x1 * 8;
    l4d_red4(p0, s0[0], s0[1], s0[2], s0[3]);
    l4d_red4(p0 + 4, s0[4], s0[5], s0[6], s0[7]);
    l4d_red4(p1, s1[0], s1[1], s1[2], s1[3]);
    l4d_red4(p1 + 4, s1[4], s1[5], s1[6], s1[7]);
  }
}
// one level of the static hash for a warp of consecutive samples: runs of lanes with equal `key` (= equal cells, hence equal
// corner indices) are summed and the last lane of a run issues the 8 corner reductions; two passes of 4 corners x 4 features keep
// 16 values live.  All 32 lanes must call; lanes without a sample pass dd = 0.
L4D_WARP_FN void l4d_static_scatter_warp(float* gbase, const uint32_t (&idx)[8], const float (&w)[8], const float4 dd, int key) {
  const WarpRuns r = l4d_warp_runs(key);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float s0[8], s1[8];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      s0[2 * c] = w[4 * h + c] * dd.x; s0[2 * c + 1] = w[4 * h + c] * dd.y;
      s1[2 * c] = w[4 * h + c] * dd.z; s1[2 * c + 1] = w[4 * h + c] * dd.w;
    }
    l4d_seg_sum8(s0, r);
    l4d_seg_sum8(s1, r);
    if (r.tail) {
#pragma unroll
      for (int c = 0; c < 4; ++c) l4d_red4(gbase + (size_t)idx[4 * h + c] * 4, s0[2 * c], s0[2 * c + 1], s1[2 * c], s1[2 * c + 1]);
    }
  }
}
// ---- vertex runs: one gradient update per distinct grid vertex of a warp ------------------------------------------------------
// Consecutive samples of a ray sit in the same or in neighbouring cells of a level, and neighbouring cells share 4 of their 8
// corners (2 of 4 in 2D), each lane reaching a shared vertex through a different corner slot.  Slot s of a lane is the vertex
// cell + bits(s).  Between lanes j < i with every |cell_i - cell_j| <= 1, slot s of lane i is slot s + delta of lane j (per axis;
// delta = cell_i - cell_j); with any |delta| >= 2 they share nothing.  The lanes that touch one vertex are found per slot
// from the neighbouring lanes only (head: the previous lane does not touch it; tail: the next one does not), and a segmented
// Hillis-Steele scan carries, per slot, the partial sum of the vertex's run together with an "open" bit (the run starts further
// back), routing lane i-d's slots onto lane i's.  It is exact for any cell sequence: a vertex whose lanes are not contiguous
// simply gets one update per contiguous run.  Keyed on cell coordinates, never on table indices, so two vertices that hash to
// one entry stay two updates.
template <int D>
L4D_WARP_FN constexpr unsigned l4d_slots_with_bit(int a) {      // corner slots whose offset along axis a is 1
  return D == 3 ? (a == 0 ? 0xAAu : (a == 1 ? 0xCCu : 0xF0u)) : (a == 0 ? 0xAu : 0xCu);
}
struct VertexRuns {
  unsigned open;    // slots whose vertex the previous lane also touches
  unsigned issue;   // slots this lane reduces: it is active and the next lane does not touch that vertex
  bool any;         // warp-uniform: some lane shares a vertex with its predecessor (else open = 0 everywhere)
};
// cell: this lane's cell at the level; seg: lanes only link to a neighbour with the same seg (the ray); inactive lanes link to
// nobody and issue nothing.  All 32 lanes must call.
template <int D>
L4D_WARP_FN VertexRuns l4d_vertex_runs(const int (&cell)[D], int seg, bool active) {
  constexpr unsigned ALL = (1u << (1 << D)) - 1u;
  const unsigned lane = threadIdx.x & 31u;
  const int key = active ? seg : -1;
  const int prev_key = __shfl_up_sync(0xffffffffu, key, 1);
  bool linked = lane > 0u && key >= 0 && prev_key == key;
  int code = 0;                                    // per axis 2 bits: delta + 1 (delta = cell - previous lane's cell)
#pragma unroll
  for (int a = 0; a < D; ++a) {
    const int dlt = cell[a] - __shfl_up_sync(0xffffffffu, cell[a], 1);
    linked = linked && dlt >= -1 && dlt <= 1;
    code |= (dlt + 1) << (2 * a);
  }
  // what the next lane sees (its link and its delta per axis) comes back through ballots: shuffles only go upwards here
  const unsigned links = __ballot_sync(0xffffffffu, linked);
  const unsigned next_bit = lane < 31u ? (1u << (lane + 1u)) : 0u;
  unsigned prev_sh = linked ? ALL : 0u, next_sh = (links & next_bit) ? ALL : 0u;
#pragma unroll
  for (int a = 0; a < D; ++a) {
    const unsigned hi = l4d_slots_with_bit<D>(a);
    const int dp = (code >> (2 * a)) & 3;
    const unsigned up = __ballot_sync(0xffffffffu, linked && dp == 2), down = __ballot_sync(0xffffffffu, linked && dp == 0);
    prev_sh &= dp == 2 ? ~hi : (dp == 0 ? hi : ALL);          // moved +1 since the previous lane: its upper corners are our lower
    next_sh &= (up & next_bit) ? hi : ((down & next_bit) ? ~hi : ALL);
  }
  VertexRuns r;
  r.open = prev_sh;
  r.issue = active ? (ALL & ~next_sh) : 0u;
  r.any = links != 0u;
  return r;
}
// v[slot][f]: this lane's contribution to the vertex of each slot.  On return the issuing slots (VertexRuns::issue) hold the sum
// over the vertex's run of lanes.  Steps only while some slot is still open (at most 5).
template <int D, int F>
L4D_WARP_FN void l4d_vertex_sum(float (&v)[1 << D][F], const int (&cell)[D], const VertexRuns& r) {
  constexpr int K = 1 << D;
  constexpr unsigned ALL = (1u << K) - 1u;
  unsigned open = r.open;
  int low = 0;                                     // the cells' low 2 bits: enough to tell delta in {-1, 0, 1}
#pragma unroll
  for (int a = 0; a < D; ++a) low |= (cell[a] & 3) << (K + 2 * a);
#pragma unroll 1
  for (int d = 1; d < 32 && __ballot_sync(0xffffffffu, open != 0u) != 0u; d <<= 1) {
    const int m = __shfl_up_sync(0xffffffffu, (int)open | low, d);
    // an open slot guarantees that lane i-d touches its vertex: |delta| <= 1, and slot s here is slot s + delta there
    int dc[D];
    unsigned po = (unsigned)m & ALL;
#pragma unroll
    for (int a = 0; a < D; ++a) {
      dc[a] = (cell[a] - (m >> (K + 2 * a))) & 3;   // 1: +1, 3: -1, 0: same cell along a
      const unsigned hi = l4d_slots_with_bit<D>(a);
      const int sh = 1 << a;
      po = dc[a] == 1 ? (((po >> sh) & ~hi) | (po & hi)) : (dc[a] == 3 ? (((po << sh) & hi) | (po & ~hi)) : po);
    }
    float take[K];
#pragma unroll
    for (int s = 0; s < K; ++s) take[s] = ((open >> s) & 1u) ? 1.0f : 0.0f;
    open &= po;
#pragma unroll
    for (int f = 0; f < F; ++f) {
      float t[K];
#pragma unroll
      for (int s = 0; s < K; ++s) t[s] = __shfl_up_sync(0xffffffffu, v[s][f], d);
#pragma unroll
      for (int a = 0; a < D; ++a) {          // select network, one stage per axis (no dynamically indexed registers)
        float u[K];
#pragma unroll
        for (int s = 0; s < K; ++s) u[s] = (s >> a) & 1 ? (dc[a] == 3 ? t[s & ~(1 << a)] : t[s]) : (dc[a] == 1 ? t[s | (1 << a)] : t[s]);
#pragma unroll
        for (int s = 0; s < K; ++s) t[s] = u[s];
      }
      // fma(t, 1, v) rounds like t + v; fma(t, 0, v) = v for every finite t
#pragma unroll
      for (int s = 0; s < K; ++s) v[s][f] = fmaf(t[s], take[s], v[s][f]);
    }
  }
}
// one level of the static hash for a warp of consecutive samples: every distinct vertex of the warp gets one 16-byte reduction.
// At levels where no lane shares a vertex with its neighbour (the fine ones) this is the plain per-lane scatter after one ballot.
// All 32 lanes must call; lanes without a sample pass active = false and dd = 0.
L4D_WARP_FN void l4d_static_vertex_scatter_warp(float* gbase, const uint32_t (&idx)[8], const float (&w)[8], const float4 dd,
                                         const int (&cell)[3], int seg, bool active) {
  const VertexRuns r = l4d_vertex_runs<3>(cell, seg, active);
  if (!r.any) {
    if (active) {
#pragma unroll
      for (int c = 0; c < 8; ++c) l4d_red4(gbase + (size_t)idx[c] * 4, w[c] * dd.x, w[c] * dd.y, w[c] * dd.z, w[c] * dd.w);
    }
    return;
  }
  float v[8][4];
#pragma unroll
  for (int c = 0; c < 8; ++c) { v[c][0] = w[c] * dd.x; v[c][1] = w[c] * dd.y; v[c][2] = w[c] * dd.z; v[c][3] = w[c] * dd.w; }
  l4d_vertex_sum<3, 4>(v, cell, r);
#pragma unroll
  for (int c = 0; c < 8; ++c)
    if ((r.issue >> c) & 1u) l4d_red4(gbase + (size_t)idx[c] * 4, v[c][0], v[c][1], v[c][2], v[c][3]);
}
#endif

// sink of a contracted time-plane row
template <bool WARP_AGG>
L4D_HD void l4d_row_sink(float* Grow, const Bilerp& b, const float g[8], int seg = 0) {
#if defined(__CUDA_ARCH__)
  if (WARP_AGG) { l4d_row_scatter_warp(Grow, b, g, seg); return; }
#endif
  l4d_row_scatter(Grow, b, g);
}
// plane-gradient sink: plain per-lane REDs, or the warp-aggregated version (device, full warps only)
template <bool WARP_AGG>
L4D_HD void l4d_plane_sink(float* G, int W, const Bilerp& b, const float g[8], bool time_plane) {
#if defined(__CUDA_ARCH__)
  if (WARP_AGG) {
    if (time_plane) l4d_plane_scatter_warp_t(G, W, b, g); else l4d_plane_scatter_warp(G, W, b, g);
    return;
  }
#endif
  l4d_plane_scatter(G, W, b, g);
}

// where dL/dfeature comes from: recomputed on demand from dh (single-kernel path) or read from the
// SoA plane the dense backward kernel wrote (split pipeline)
struct DfeatFromDh {
  const DevModel* M;
  const BwSample* s;
  L4D_HD float operator()(int row) const { return l4d_dot64(s->dh, M->sig_w1t + (size_t)row * L4D_H); }
  L4D_HD void ld4(int row, float (&o)[4]) const { for (int i = 0; i < 4; ++i) o[i] = (*this)(row + i); }
};
struct DfeatFromPlane {
  const float* base;     // dfeat + p
  size_t stride;         // P
  L4D_HD float operator()(int row) const { return l4d_ld1(base + (size_t)row * stride); }
  L4D_HD void ld4(int row, float (&o)[4]) const { for (int i = 0; i < 4; ++i) o[i] = (*this)(row + i); }
};

struct DynHashCursor {
  int p, l;            // next (plane, level)
  float dq[4];         // dL/dfeature of levels (l & ~3) .. +3 of plane p (valid when the level count is a multiple of 4)
};
// up to n (plane, level) pairs of the dynamic-hash gradient: only the (x,t) query carries gradient
// (lidar4d.py:160-161,169-170 are no_grad)
// WARP_AGG (device): every lane of the warp calls, inactive ones with active = false; the contracted path then sums each
// vertex over its run of lanes (l4d_vertex_sum) before it reduces.  seg: the lane's ray.
template <bool WARP_AGG, class DF>
L4D_HD void l4d_bw_dynhash_slice(const DevModel& M, const L4DFrame& F, const DevGrads& G, float x, float y, float z, float wc,
                                 const DF& l4d_dfeat_fn, int row_hash_d, DynHashCursor& cur, int n, int seg, bool active,
                                 size_t comb_off = 0) {
  if (!WARP_AGG && !active) return;
  const int L = (int)M.gs.n_levels;
  const bool quads = (L & 3) == 0;             // rows of a plane start on a multiple of 4: one 16-byte load per 4 levels
#pragma unroll 1
  for (; n > 0 && cur.p < 3; --n) {
    const int p = cur.p, l = cur.l;
    const float ca = p == 2 ? y : x, cb = p == 0 ? y : z;
    uint32_t idx[4]; float w[4];
    l4d_corners2(M.gd[p], l, ca, cb, idx, w);
    if (quads && (l & 3) == 0) l4d_dfeat_fn.ld4(row_hash_d + p * L + l, cur.dq);
    const int li = l & 3;
    const float dsel = li == 0 ? cur.dq[0] : (li == 1 ? cur.dq[1] : (li == 2 ? cur.dq[2] : cur.dq[3]));
    const float d = wc * (quads ? dsel : l4d_dfeat_fn(row_hash_d + p * L + l));
    float* gcomb = G.hd_comb[p];
    if (gcomb) {
      gcomb += comb_off;
      // comb[entry] accumulates w_corner * d: ONE float per entry (the four features of an entry get basis[k] times it,
      // and the slice weights, in k_fold_dynamic).  The two x-corners of a cell are neighbours in the table (index =
      // cx ^ h(cy) or cx + cy * res) and fall into the same aligned quad of entries three times out of four: they go out
      // as one 16-byte RED on that quad, 2.5 instead of 4 L2 atomic operations per level (the backward is bound by them:
      // 1.5 SM-cycles per lane-operation whatever its width, profiles/r02_micro_red.txt).
      // With WARP_AGG each vertex of the warp is first summed over its run of lanes and reduced once, by the run's last lane.
      float v[4][1] = {{w[0] * d}, {w[1] * d}, {w[2] * d}, {w[3] * d}};
      unsigned issue = 0xFu;
#if defined(__CUDA_ARCH__)
      if (WARP_AGG) {
        int cell[2];
        float fa, fb;
        uint32_t ua, ub;
        l4d_pos_fract(M.gd[p].scale[l], ca, ua, fa);
        l4d_pos_fract(M.gd[p].scale[l], cb, ub, fb);
        cell[0] = (int)ua; cell[1] = (int)ub;
        const VertexRuns vr = l4d_vertex_runs<2>(cell, seg, active);
        if (vr.any) l4d_vertex_sum<2, 1>(v, cell, vr);
        issue = vr.issue;
      }
#endif
      float* cb = gcomb + M.gd[p].offset[l];          // level offsets are multiples of 8 entries: quads stay 16-byte aligned
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const uint32_t i0 = idx[2 * r], i1 = idx[2 * r + 1];
        const float a = v[2 * r][0], b = v[2 * r + 1][0];
        const bool e0 = (issue >> (2 * r)) & 1u, e1 = (issue >> (2 * r + 1)) & 1u;
        if (e0 && e1 && (i0 >> 2) == (i1 >> 2)) {
          const uint32_t s0 = i0 & 3u, s1 = i1 & 3u;
          l4d_red4(cb + (i0 & ~3u), (s0 == 0u ? a : 0.f) + (s1 == 0u ? b : 0.f), (s0 == 1u ? a : 0.f) + (s1 == 1u ? b : 0.f),
                   (s0 == 2u ? a : 0.f) + (s1 == 2u ? b : 0.f), (s0 == 3u ? a : 0.f) + (s1 == 3u ? b : 0.f));
        } else {
          if (e0) l4d_red1(cb + i0, a);
          if (e1) l4d_red1(cb + i1, b);
        }
      }
    } else if (active) {
      const float e0 = d * F.cur.basis[0], e1 = d * F.cur.basis[1], e2 = d * F.cur.basis[2], e3 = d * F.cur.basis[3];
      const size_t off = (size_t)M.gd[p].offset[l] * 4;
      float* glo = G.hd[p][F.cur.slice_lo];
      float* ghi = G.hd[p][F.cur.slice_hi];
      const float slo = F.cur.single ? 1.0f : F.cur.w_lo;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float ww = w[c] * slo;
        l4d_red4(glo + off + (size_t)idx[c] * 4, ww * e0, ww * e1, ww * e2, ww * e3);
      }
      if (!F.cur.single) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float ww = w[c] * F.cur.w_hi;
          l4d_red4(ghi + off + (size_t)idx[c] * 4, ww * e0, ww * e1, ww * e2, ww * e3);
        }
      }
    }
    if (++cur.l == L) { cur.l = 0; ++cur.p; }
  }
}

// scatter dL/dfeature through the encoders of one sample at (x,y,z) with its flow; dflow[6] out
template <bool WARP_AGG, class DF, bool STATIC_HASH = true, bool ROWS = false>
L4D_HD void l4d_bw_scatter_t(const DevModel& M, const L4DFrame& F, const DevGrads& G, float x, float y, float z,
                             const float* flow, const DF& l4d_dfeat_fn, float (&dflow)[6], bool active, int seg = 0,
                             uint32_t frame = 0, size_t con_off = 0, size_t comb_off = 0);

template <bool ROWS = false>
L4D_HD void l4d_bw_scatter(const DevModel& M, const L4DFrame& F, const DevGrads& G, BwSample& s) {
#pragma unroll
  for (int k = 0; k < 6; ++k) s.dflow[k] = 0.f;
  if (!s.active) return;
  DfeatFromDh df{&M, &s};
  l4d_bw_scatter_t<false, DfeatFromDh, true, ROWS>(M, F, G, s.x, s.y, s.z, s.flow, df, s.dflow, true);
}

// ROWS: time planes are sampled from DevModel::pl_con and their gradients go to DevGrads::pl_rows (both must be set)
// WARP_AGG: every lane of the warp must call (lanes without a sample pass active=false and a
// provider that returns 0; they take part in the plane aggregation with zero contributions); seg: the sample's ray.
// frame / con_off / comb_off: the sample's frame in a multi-frame launch and the float offsets of that frame's contracted
// tables (DevModel::hd_con, pl_con) and accumulators (DevGrads::hd_comb, pl_rows) from the launch's first ones.
template <bool WARP_AGG, class DF, bool STATIC_HASH, bool ROWS>
L4D_HD void l4d_bw_scatter_t(const DevModel& M, const L4DFrame& F, const DevGrads& G, float x, float y, float z,
                             const float* flow, const DF& l4d_dfeat_fn, float (&dflow)[6], bool active, int seg,
                             uint32_t frame, size_t con_off, size_t comb_off) {
#pragma unroll
  for (int k = 0; k < 6; ++k) dflow[k] = 0.f;
  const int nS = (int)M.n_scales;
  const int L = (int)M.gs.n_levels;
  const int row_plane_d = nS * 8;
  const int row_hash_s = 2 * nS * 8;
  const int row_hash_d = row_hash_s + L * 4;
  float wc, wf, wb;
  l4d_agg_weights(F, wc, wf, wb);
  const float xf0 = x + flow[0], xf1 = y + flow[1], xf2 = z + flow[2];
  const float xw0 = x + flow[3], xw1 = y + flow[4], xw2 = z + flow[5];
  DynHashCursor hc;
  hc.p = 0;
  hc.l = 0;
  hc.dq[0] = hc.dq[1] = hc.dq[2] = hc.dq[3] = 0.f;

#pragma unroll 1
  for (int sc = 0; sc < nS; ++sc) {
    const int R = (int)M.plane_res[sc];
    const int T = (int)M.time_res;
    {   // static planes: product rule over (x,y) (x,z) (y,z)
      float d[8], v0[8], v1[8], v2[8], dummy[8], g[8];
#pragma unroll
      for (int c = 0; c < 8; c += 4) l4d_dfeat_fn.ld4(sc * 8 + c, *reinterpret_cast<float(*)[4]>(d + c));
      Bilerp b0 = l4d_bilerp(x, R, y, R), b1 = l4d_bilerp(x, R, z, R), b2 = l4d_bilerp(y, R, z, R);
      l4d_plane_sample<false>(M.planes[sc][0], R, b0, v0, dummy);
      l4d_plane_sample<false>(M.planes[sc][1], R, b1, v1, dummy);
      l4d_plane_sample<false>(M.planes[sc][3], R, b2, v2, dummy);
#pragma unroll
      for (int c = 0; c < 8; ++c) g[c] = d[c] * v1[c] * v2[c];
      l4d_plane_sink<WARP_AGG>(G.planes_cl[sc][0], R, b0, g, false);
#pragma unroll
      for (int c = 0; c < 8; ++c) g[c] = d[c] * v0[c] * v2[c];
      l4d_plane_sink<WARP_AGG>(G.planes_cl[sc][1], R, b1, g, false);
#pragma unroll
      for (int c = 0; c < 8; ++c) g[c] = d[c] * v0[c] * v1[c];
      l4d_plane_sink<WARP_AGG>(G.planes_cl[sc][3], R, b2, g, false);
    }
    {   // time planes (x,t) (y,t) (z,t): three queries, warped ones also feed d(coords) -> flow
      float d[8];
#pragma unroll
      for (int c = 0; c < 8; c += 4) l4d_dfeat_fn.ld4(row_plane_d + sc * 8 + c, *reinterpret_cast<float(*)[4]>(d + c));
#pragma unroll 1
      for (int qi = 0; qi < 3; ++qi) {
        const float wq = qi == 0 ? wc : (qi == 1 ? wf : wb);
        // the warp sinks need every lane: a query is skipped when no lane of the warp has it (lanes of a frame without
        // that neighbour then take part with zero contributions; their frame has no contracted row for it to read)
#if defined(__CUDA_ARCH__)
        if (WARP_AGG ? !__any_sync(0xffffffffu, wq != 0.f) : wq == 0.f) continue;
#else
        if (wq == 0.f) continue;
#endif
        const float q0 = qi == 0 ? x : (qi == 1 ? xf0 : xw0);
        const float q1 = qi == 0 ? y : (qi == 1 ? xf1 : xw1);
        const float q2 = qi == 0 ? z : (qi == 1 ? xf2 : xw2);
        const float tau = qi == 0 ? F.cur.tau : (qi == 1 ? F.fwd.tau : F.bwd.tau);
        float v0[8], v1[8], v2[8], x0[8], x1[8], x2[8], g[8];
        Bilerp b0 = l4d_bilerp(q0, R, tau, T), b1 = l4d_bilerp(q1, R, tau, T), b2 = l4d_bilerp(q2, R, tau, T);
        // rows: the forward's contracted time planes (2 texels per sample) and their gradient rows, when the launch has them
        constexpr bool rows = ROWS;       // (a template parameter: the kernel is large, keep the other path out of it)
        if (rows && wq == 0.f) {
#pragma unroll
          for (int c = 0; c < 8; ++c) v0[c] = v1[c] = v2[c] = x0[c] = x1[c] = x2[c] = 0.f;
        } else if (rows) {
          l4d_row_sample<true>(M.pl_con[sc][0][qi] + con_off, b0, v0, x0);
          l4d_row_sample<true>(M.pl_con[sc][1][qi] + con_off, b1, v1, x1);
          l4d_row_sample<true>(M.pl_con[sc][2][qi] + con_off, b2, v2, x2);
        } else {
          l4d_plane_sample<true>(M.planes[sc][2], R, b0, v0, x0);
          l4d_plane_sample<true>(M.planes[sc][4], R, b1, v1, x1);
          l4d_plane_sample<true>(M.planes[sc][5], R, b2, v2, x2);
        }
        float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) { g[c] = wq * d[c] * v1[c] * v2[c]; c0 = fmaf(g[c], x0[c], c0); }
        if (rows) l4d_row_sink<WARP_AGG>(G.pl_rows[sc][0][qi] + comb_off, b0, g, (int)frame); else l4d_plane_sink<WARP_AGG>(G.planes_cl[sc][2], R, b0, g, true);
#pragma unroll
        for (int c = 0; c < 8; ++c) { g[c] = wq * d[c] * v0[c] * v2[c]; c1 = fmaf(g[c], x1[c], c1); }
        if (rows) l4d_row_sink<WARP_AGG>(G.pl_rows[sc][1][qi] + comb_off, b1, g, (int)frame); else l4d_plane_sink<WARP_AGG>(G.planes_cl[sc][4], R, b1, g, true);
#pragma unroll
        for (int c = 0; c < 8; ++c) { g[c] = wq * d[c] * v0[c] * v1[c]; c2 = fmaf(g[c], x2[c], c2); }
        if (rows) l4d_row_sink<WARP_AGG>(G.pl_rows[sc][2][qi] + comb_off, b2, g, (int)frame); else l4d_plane_sink<WARP_AGG>(G.planes_cl[sc][5], R, b2, g, true);
        if (qi == 1) { dflow[0] += c0; dflow[1] += c1; dflow[2] += c2; }
        if (qi == 2) { dflow[3] += c0; dflow[4] += c1; dflow[5] += c2; }
      }
    }
  }

  // static hash: dL/dtable[entry] += w_corner * dfeat[0..4)   (the split pipeline does this level-major in
  // k_bwd_encoders so that only one level's 8 MB of gradients is live in L2 at a time)
#pragma unroll 1
  for (int l = 0; STATIC_HASH && active && l < L; ++l) {
    uint32_t idx[8]; float w[8];
    l4d_corners3(M.gs, l, x, y, z, idx, w);
    float dd[4];
    l4d_dfeat_fn.ld4(row_hash_s + 4 * l, dd);
    const float d0 = dd[0], d1 = dd[1], d2 = dd[2], d3 = dd[3];
    float* base = G.hs + (size_t)M.gs.offset[l] * 4;
#pragma unroll
    for (int c = 0; c < 8; ++c) l4d_red4(base + (size_t)idx[c] * 4, w[c] * d0, w[c] * d1, w[c] * d2, w[c] * d3);
  }

  // dynamic hash
  l4d_bw_dynhash_slice<WARP_AGG>(M, F, G, x, y, z, wc, l4d_dfeat_fn, row_hash_d, hc, 3 * L, seg, active, comb_off);
}

// ---- B5: flow MLP backprop.  g[6] = dL/dflow of this sample. ----------------------------
// step a: recompute h1,h2 (and their relu patterns when RECORD) ; TA row[0..8) <- g ; TB row <- h2 ; xb keeps h1
template <bool RECORD>
L4D_HD void l4d_bw_flow_a_t(const DevModel& M, BwSample& s, const float* flow_in, size_t stride,
                            const float g[6], float* xb, int xs, float* ta_row, float* tb_row) {
  float yv[L4D_H];
#pragma unroll
  for (int k = 0; k < L4D_FLOW_IN; ++k) xb[k * xs] = s.active ? flow_in[(size_t)k * stride] : 0.f;
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) yv[k] = 0.f;
  l4d_layer64(yv, xb, xs, L4D_FLOW_IN, M.flo_w0t);
  if (RECORD) {
    l4d_relu_store(yv, xb, xs, s.mf1a, s.mf1b);                               // h1
  } else {
#pragma unroll
    for (int k = 0; k < L4D_H; ++k) xb[k * xs] = fmaxf(yv[k], 0.f);           // h1
  }
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) yv[k] = 0.f;
  l4d_layer64(yv, xb, xs, L4D_H, M.flo_w1t);
  if (RECORD) { s.mf2a = 0u; s.mf2b = 0u; }
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) {
    const bool on = yv[k] > 0.f;
    if (RECORD) { if (k < 32) s.mf2a |= on ? (1u << k) : 0u; else s.mf2b |= on ? (1u << (k - 32)) : 0u; }
    tb_row[k] = (s.active && on) ? yv[k] : 0.f;                               // h2
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) ta_row[k] = (s.active && k < 6) ? g[k] : 0.f;
}
L4D_HD void l4d_bw_flow_a(const DevModel& M, const BwSample& s, const float* flow_in, size_t stride,
                          const float g[6], float* xb, int xs, float* ta_row, float* tb_row) {
  l4d_bw_flow_a_t<false>(M, const_cast<BwSample&>(s), flow_in, stride, g, xb, xs, ta_row, tb_row);
}
// step b: dh2 = (W2^T g) * relu2 ; TB row <- dh2 ; TA row <- h1 (from xb) ; xb <- dh2
L4D_HD void l4d_bw_flow_b(const DevModel& M, const BwSample& s, const float g[6], float* xb, int xs,
                          float* ta_row, float* tb_row) {
  float d[L4D_H];
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) { d[k] = 0.f; ta_row[k] = s.active ? xb[k * xs] : 0.f; }
  if (s.active) {
#pragma unroll
    for (int o = 0; o < 6; ++o) l4d_axpy64(d, g[o], M.flo_w2 + (size_t)o * L4D_H);
  }
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) {
    d[k] = l4d_bit(s.mf2a, s.mf2b, k) ? d[k] : 0.f;
    tb_row[k] = d[k];
    xb[k * xs] = d[k];
  }
}
// step c: dh1 = (W1^T dh2) * relu1 ; TB row <- dh1 ; TA row[0..16) <- flow_in ; then the grid scatter
L4D_HD void l4d_bw_flow_c(const DevModel& M, const L4DFrame& F, const DevGrads& G, const BwSample& s,
                          const float* flow_in, size_t stride, float* xb, int xs, float* ta_row, float* tb_row) {
  float d[L4D_H];
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) d[k] = 0.f;
  l4d_layer64(d, xb, xs, L4D_H, M.flo_w1);                 // native [o][k]
#pragma unroll
  for (int k = 0; k < L4D_H; ++k) {
    d[k] = l4d_bit(s.mf1a, s.mf1b, k) ? d[k] : 0.f;
    tb_row[k] = d[k];
  }
#pragma unroll
  for (int k = 0; k < L4D_FLOW_IN; ++k) ta_row[k] = s.active ? flow_in[(size_t)k * stride] : 0.f;
  if (!s.active) return;
  // d(flow_in)[i] = W0[:, i] . dh1 ; feature (l, 2i+c) of the grid gets basis[i] * d(flow_in)[2l+c]
#pragma unroll 1
  for (int l = 0; l < 8; ++l) {
    const float d0 = l4d_dot64(d, M.flo_w0t + (size_t)(2 * l) * L4D_H);
    const float d1 = l4d_dot64(d, M.flo_w0t + (size_t)(2 * l + 1) * L4D_H);
    uint32_t idx[8]; float w[8];
    l4d_corners3(M.gf, l, s.x, s.y, s.z, idx, w);
    float* base = G.hf + (size_t)M.gf.offset[l] * 8;
    const float* b = F.flow_basis;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float* p = base + (size_t)idx[c] * 8;
      l4d_red4(p, w[c] * b[0] * d0, w[c] * b[0] * d1, w[c] * b[1] * d0, w[c] * b[1] * d1);
      l4d_red4(p + 4, w[c] * b[2] * d0, w[c] * b[2] * d1, w[c] * b[3] * d0, w[c] * b[3] * d1);
    }
  }
}
