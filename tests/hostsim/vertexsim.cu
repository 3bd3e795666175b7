// vertexsim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// Drivers for the vertex-run reduction of lidar4d_b200/csrc/l4d_bwd.cuh (l4d_vertex_runs, l4d_vertex_sum,
// l4d_static_vertex_scatter_warp) on the CPU.  warpsim.cu supplies the 32-thread lockstep warp emulator and compiles the header
// with the warp intrinsics redirected to it; this file adds the entry points tests/test_warpsim_vertex_runs.py calls.
#include "warpsim.cu"

// vertex runs of one warp, D = 2 (F = 1 value per corner) or 3 (F = 4): cells[32][D], seg[32], active[32], v[32][K][F] in; the
// scanned v and the issue masks out
template <int D, int F>
struct VrJob { ws::Warp* warp; unsigned lane; int cell[D]; int seg; bool active; float v[1 << D][F]; unsigned issue; };
template <int D, int F>
static void* vr_main(void* p) {
  VrJob<D, F>* j = (VrJob<D, F>*)p;
  ws::t_warp = j->warp; ws::t_lane = j->lane;
  pthread_mutex_lock(&j->warp->run);
  const VertexRuns r = l4d_vertex_runs<D>(j->cell, j->seg, j->active);
  if (r.any) l4d_vertex_sum<D, F>(j->v, j->cell, r);
  j->issue = r.issue;
  pthread_mutex_unlock(&j->warp->run);
  return nullptr;
}
template <int D, int F>
static int vertex_runs(const int* cells, const int* seg, const int* active, float* v, unsigned* issue) {
  constexpr int K = 1 << D;
  ws::Warp W;
  pthread_barrier_init(&W.bar, nullptr, 32);
  pthread_mutex_init(&W.run, nullptr);
  VrJob<D, F> jobs[32];
  pthread_t th[32];
  for (unsigned l = 0; l < 32; ++l) {
    VrJob<D, F>& j = jobs[l];
    j.warp = &W; j.lane = l; j.seg = seg[l]; j.active = active[l] != 0;
    for (int a = 0; a < D; ++a) j.cell[a] = cells[l * D + a];
    for (int s = 0; s < K; ++s) for (int f = 0; f < F; ++f) j.v[s][f] = v[(l * K + s) * F + f];
    pthread_create(&th[l], nullptr, vr_main<D, F>, &j);
  }
  for (unsigned l = 0; l < 32; ++l) pthread_join(th[l], nullptr);
  for (unsigned l = 0; l < 32; ++l) {
    issue[l] = jobs[l].issue;
    for (int s = 0; s < K; ++s) for (int f = 0; f < F; ++f) v[(l * K + s) * F + f] = jobs[l].v[s][f];
  }
  pthread_mutex_destroy(&W.run);
  pthread_barrier_destroy(&W.bar);
  return 0;
}
extern "C" int vs_vertex_runs(int D, const int* cells, const int* seg, const int* active, float* v, unsigned* issue) {
  if (D == 2) return vertex_runs<2, 1>(cells, seg, active, v, issue);
  if (D == 3) return vertex_runs<3, 4>(cells, seg, active, v, issue);
  return -1;
}

// One static-hash level through l4d_static_vertex_scatter_warp, as k_bwd_scatter_static runs it.  n samples (multiple of 32) at
// x[n][3] in [0,1] with dL/dfeature dd[n][4], ray ids seg[n]; grid = level 0 of a 3D grid (scale, res, entries); G_* = [entries][4].
struct SvJob { ws::Warp* warp; unsigned lane; float* G; uint32_t idx[8]; float w[8]; float4 dd; int cell[3]; int seg; };
static void* sv_main(void* p) {
  SvJob* j = (SvJob*)p;
  ws::t_warp = j->warp; ws::t_lane = j->lane;
  pthread_mutex_lock(&j->warp->run);
  l4d_static_vertex_scatter_warp(j->G, j->idx, j->w, j->dd, j->cell, j->seg, true);
  pthread_mutex_unlock(&j->warp->run);
  return nullptr;
}
extern "C" int vs_static_level(float scale, uint32_t res, uint32_t entries, int n, const float* x, const float* dd, const int* seg,
                               float* G_agg, float* G_ref) {
  if (n % 32) return -1;
  DevGrid g;
  memset(&g, 0, sizeof(g));
  g.scale[0] = scale; g.res[0] = res; g.entries[0] = entries; g.offset[0] = 0; g.offset[1] = entries; g.n_levels = 1;
  for (int base = 0; base < n; base += 32) {
    ws::Warp W;
    pthread_barrier_init(&W.bar, nullptr, 32);
    pthread_mutex_init(&W.run, nullptr);
    SvJob jobs[32];
    pthread_t th[32];
    for (int l = 0; l < 32; ++l) {
      SvJob& j = jobs[l];
      const float* p = x + (size_t)(base + l) * 3;
      const float* d = dd + (size_t)(base + l) * 4;
      j.warp = &W; j.lane = (unsigned)l; j.G = G_agg; j.seg = seg[base + l];
      l4d_corners3(g, 0, p[0], p[1], p[2], j.idx, j.w);
      j.dd = make_float4(d[0], d[1], d[2], d[3]);
      uint32_t cx, cy, cz; float fx, fy, fz;
      l4d_pos_fract(scale, p[0], cx, fx); l4d_pos_fract(scale, p[1], cy, fy); l4d_pos_fract(scale, p[2], cz, fz);
      j.cell[0] = (int)cx; j.cell[1] = (int)cy; j.cell[2] = (int)cz;
      for (int c = 0; c < 8; ++c) l4d_red4(G_ref + (size_t)j.idx[c] * 4, j.w[c] * d[0], j.w[c] * d[1], j.w[c] * d[2], j.w[c] * d[3]);
    }
    for (int l = 0; l < 32; ++l) pthread_create(&th[l], nullptr, sv_main, &jobs[l]);
    for (int l = 0; l < 32; ++l) pthread_join(th[l], nullptr);
    pthread_mutex_destroy(&W.run);
    pthread_barrier_destroy(&W.bar);
  }
  return 0;
}
