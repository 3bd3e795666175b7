// warpsim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The warp-aggregated gradient sinks of lidar4d_b200/csrc/l4d_bwd.cuh (segmented warp scans, run detection, "only the last
// lane of a run reduces") are device code built on warp intrinsics, which the host-sim of hostsim.cu cannot reach.  This file
// compiles exactly those functions for the CPU: L4D_WARP_FN makes them plain host functions, the intrinsics they use are
// redirected to a small emulator in which 32 host threads play the 32 lanes of a warp in lockstep (every collective is a
// rendezvous; between collectives one lane runs at a time, so the plain `+=` that stands in for RED on the host cannot race).
// `pytest -m "not gpu"` then checks the aggregated sinks against the plain per-lane scatter in the build container.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>
#include <vector>

// ---- the emulator ----------------------------------------------------------------------------------------------------
namespace ws {
struct Warp {
  pthread_barrier_t bar;
  pthread_mutex_t run;      // held by the one lane that is executing between collectives
  uint32_t slot[32];
};
static thread_local Warp* t_warp = nullptr;
static thread_local unsigned t_lane = 0;
struct Tid { unsigned x; };
static inline Tid tid() { return Tid{t_lane}; }

// deposit -> everybody reads -> continue (serialised again)
static inline void begin(uint32_t v) {
  t_warp->slot[t_lane] = v;
  pthread_mutex_unlock(&t_warp->run);
  pthread_barrier_wait(&t_warp->bar);
}
static inline void end() {
  pthread_barrier_wait(&t_warp->bar);
  pthread_mutex_lock(&t_warp->run);
}
static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

static inline int shfl_up(unsigned, int v, int d) {
  begin((uint32_t)v);
  const int r = (int)t_lane >= d ? (int)t_warp->slot[t_lane - d] : v;
  end();
  return r;
}
static inline float shfl_up(unsigned m, float v, int d) { return u2f((uint32_t)shfl_up(m, (int)f2u(v), d)); }
static inline unsigned ballot(unsigned, int pred) {
  begin(pred ? 1u : 0u);
  unsigned r = 0;
  for (int i = 0; i < 32; ++i) r |= (t_warp->slot[i] & 1u) << i;
  end();
  return r;
}
static inline unsigned reduce_max(unsigned mask, unsigned v) {
  begin(v);
  unsigned r = 0;
  for (int i = 0; i < 32; ++i) if ((mask >> i) & 1u) r = t_warp->slot[i] > r ? t_warp->slot[i] : r;
  end();
  return r;
}
static inline int clz(int v) { return v == 0 ? 32 : __builtin_clz((unsigned)v); }
static inline int ffs(int v) { return __builtin_ffs(v); }
}  // namespace ws

// ---- compile the device-only warp functions for the host -----------------------------------------------------------------
#define L4D_WARP_FN inline
#define threadIdx (ws::tid())
#define __shfl_up_sync(m, v, d) ws::shfl_up((m), (v), (d))
#define __ballot_sync(m, p) ws::ballot((m), (p))
#define __reduce_max_sync(m, v) ws::reduce_max((m), (v))
#define __clz(v) ws::clz((v))
#define __ffs(v) ws::ffs((v))
#include "../../lidar4d_b200/csrc/l4d_bwd.cuh"

// ---- drivers -------------------------------------------------------------------------------------------------------------
struct LaneJob {
  ws::Warp* warp;
  unsigned lane;
  int mode;                 // 0 static plane (l4d_plane_scatter_warp), 1 time plane (.._warp_t), 2 contracted row, 3 static hash level
  float* G;
  int W;
  Bilerp b;
  float g[8];
  uint32_t idx[8];
  float w[8];
  float4 dd;
  int key;
};
static void* lane_main(void* p) {
  LaneJob* j = (LaneJob*)p;
  ws::t_warp = j->warp;
  ws::t_lane = j->lane;
  pthread_mutex_lock(&j->warp->run);
  if (j->mode == 0) l4d_plane_scatter_warp(j->G, j->W, j->b, j->g);
  else if (j->mode == 1) l4d_plane_scatter_warp_t(j->G, j->W, j->b, j->g);
  else if (j->mode == 2) l4d_row_scatter_warp(j->G, j->b, j->g);
  else l4d_static_scatter_warp(j->G, j->idx, j->w, j->dd, j->key);
  pthread_mutex_unlock(&j->warp->run);
  return nullptr;
}
static void run_warp(std::vector<LaneJob>& jobs) {
  ws::Warp W;
  pthread_barrier_init(&W.bar, nullptr, 32);
  pthread_mutex_init(&W.run, nullptr);
  pthread_t th[32];
  for (unsigned l = 0; l < 32; ++l) { jobs[l].warp = &W; jobs[l].lane = l; pthread_create(&th[l], nullptr, lane_main, &jobs[l]); }
  for (unsigned l = 0; l < 32; ++l) pthread_join(th[l], nullptr);
  pthread_mutex_destroy(&W.run);
  pthread_barrier_destroy(&W.bar);
}

// Plane sinks.  n samples (a multiple of 32; consecutive samples = consecutive lanes), coordinates cx[n], cy[n] in [0,1],
// gradients g[n][8]; plane [H][W][8] (mode 2: a row [W][8], cy is the launch-constant time coordinate and only gives the
// Bilerp its y half).  G_agg receives the warp-aggregated result, G_ref the plain per-lane scatter of the same samples.
extern "C" int ws_plane_sinks(int mode, int H, int W, int n, const float* cx, const float* cy, const float* g, float* G_agg, float* G_ref) {
  if (n % 32 || mode < 0 || mode > 2) return -1;
  for (int base = 0; base < n; base += 32) {
    std::vector<LaneJob> jobs(32);
    for (int l = 0; l < 32; ++l) {
      LaneJob& j = jobs[l];
      j.mode = mode; j.G = G_agg; j.W = W;
      j.b = l4d_bilerp(cx[base + l], W, cy[base + l], H);
      for (int c = 0; c < 8; ++c) j.g[c] = g[(size_t)(base + l) * 8 + c];
      if (mode == 2) l4d_row_scatter(G_ref, j.b, j.g); else l4d_plane_scatter(G_ref, W, j.b, j.g);
    }
    run_warp(jobs);
  }
  return 0;
}

// One static-hash level.  n samples (multiple of 32) at x[n][3] in [0,1] with dL/dfeature dd[n][4]; grid = level `l` of a 3D grid
// described like DevGrid (scale, res, entries); G_* = [entries][4].
extern "C" int ws_static_level(float scale, uint32_t res, uint32_t entries, int n, const float* x, const float* dd, float* G_agg, float* G_ref) {
  if (n % 32) return -1;
  DevGrid g;
  memset(&g, 0, sizeof(g));
  g.scale[0] = scale; g.res[0] = res; g.entries[0] = entries; g.offset[0] = 0; g.offset[1] = entries; g.n_levels = 1;
  for (int base = 0; base < n; base += 32) {
    std::vector<LaneJob> jobs(32);
    for (int l = 0; l < 32; ++l) {
      LaneJob& j = jobs[l];
      const float* p = x + (size_t)(base + l) * 3;
      j.mode = 3; j.G = G_agg;
      l4d_corners3(g, 0, p[0], p[1], p[2], j.idx, j.w);
      const float* d = dd + (size_t)(base + l) * 4;
      j.dd = make_float4(d[0], d[1], d[2], d[3]);
      uint32_t cx, cy, cz; float fx, fy, fz;
      l4d_pos_fract(scale, p[0], cx, fx); l4d_pos_fract(scale, p[1], cy, fy); l4d_pos_fract(scale, p[2], cz, fz);
      j.key = (int)(cx + res * (cy + res * cz));          // as k_bwd_scatter_static forms it
      for (int c = 0; c < 8; ++c) l4d_red4(G_ref + (size_t)j.idx[c] * 4, j.w[c] * d[0], j.w[c] * d[1], j.w[c] * d[2], j.w[c] * d[3]);
    }
    run_warp(jobs);
  }
  return 0;
}

// run structure of one warp (l4d_warp_runs): dist / maxdist / tail / mask per lane
extern "C" int ws_warp_runs(const int* keys, int* dist, int* maxdist, int* tail, unsigned* mask);
struct RunsJob { ws::Warp* warp; unsigned lane; int key; WarpRuns out; };
static void* runs_main(void* p) {
  RunsJob* j = (RunsJob*)p;
  ws::t_warp = j->warp; ws::t_lane = j->lane;
  pthread_mutex_lock(&j->warp->run);
  j->out = l4d_warp_runs(j->key);
  pthread_mutex_unlock(&j->warp->run);
  return nullptr;
}
extern "C" int ws_warp_runs(const int* keys, int* dist, int* maxdist, int* tail, unsigned* mask) {
  ws::Warp W;
  pthread_barrier_init(&W.bar, nullptr, 32);
  pthread_mutex_init(&W.run, nullptr);
  RunsJob jobs[32];
  pthread_t th[32];
  for (unsigned l = 0; l < 32; ++l) { jobs[l].warp = &W; jobs[l].lane = l; jobs[l].key = keys[l]; pthread_create(&th[l], nullptr, runs_main, &jobs[l]); }
  for (unsigned l = 0; l < 32; ++l) pthread_join(th[l], nullptr);
  for (int l = 0; l < 32; ++l) { dist[l] = jobs[l].out.dist; maxdist[l] = jobs[l].out.maxdist; tail[l] = jobs[l].out.tail ? 1 : 0; mask[l] = jobs[l].out.mask; }
  pthread_mutex_destroy(&W.run);
  pthread_barrier_destroy(&W.bar);
  return 0;
}
