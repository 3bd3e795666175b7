// nngridsim.cu - TEST INFRASTRUCTURE ONLY (never loaded by the product).
//
// The grid nearest-neighbour search (lidar4d_b200/csrc/l4d_nngrid.cuh) compiled for the CPU: the index is built serially
// with the functions k_nng_geometry / k_nng_count / k_nng_scan / k_nng_scatter call, and every query runs
// nng_query_one, as k_nng_query does on the device, for tests/test_nngrid_hostsim.py.
#include <math.h>
#include <stdint.h>

#include <vector>

#include "../../include/lidar4d_b200.h"
#include "../../lidar4d_b200/csrc/l4d_nngrid.cuh"

// dist[nq], idx[nq] and cand[nq] (records examined per query) for queries q against the cloud xyz[n, 3];
// geo[10] = {dim x, dim y, dim z, cells, budget, indexed points, bits of lo x, lo y, lo z, bits of ih}.  reverse != 0 fills the cells back to front,
// as an atomic cursor may.
extern "C" int ns_query(const float* xyz, uint32_t n, const float* q, uint32_t nq, int reverse, float* dist, int32_t* idx,
                        uint32_t* cand, uint32_t* geo) {
  if (n == 0) return -1;
  const uint32_t budget = l4d_nng_budget(n);
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (uint32_t i = 0; i < n; ++i) {
    const float* p = xyz + 3 * (size_t)i;
    if (!(nng_finite(p[0]) && nng_finite(p[1]) && nng_finite(p[2]))) continue;
    for (int a = 0; a < 3; ++a) { lo[a] = fminf(lo[a], p[a]); hi[a] = fmaxf(hi[a], p[a]); }
  }
  L4DNNGHeader H;
  nng_geometry(lo, hi, budget, &H);
  if (H.cells > budget) return -2;
  std::vector<uint32_t> cell_of(n), start(H.cells + 1, 0), cursor(H.cells);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t c = nng_point_cell(H, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]);
    cell_of[i] = c;
    if (c != 0xffffffffu) {
      if (c >= H.cells) return -3;
      ++start[c + 1];
    }
  }
  for (uint32_t c = 0; c < H.cells; ++c) { start[c + 1] += start[c]; cursor[c] = start[c]; }
  H.n_valid = start[H.cells];
  std::vector<float4> pts(n ? n : 1);
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t i = reverse ? n - 1 - k : k;
    if (cell_of[i] == 0xffffffffu) continue;
    pts[cursor[cell_of[i]]++] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], nng_from_bits(i));
  }
  for (uint32_t j = 0; j < nq; ++j) {
    uint32_t k;
    cand[j] = nng_query_one(H, start.data(), pts.data(), q[3 * (size_t)j], q[3 * (size_t)j + 1], q[3 * (size_t)j + 2], dist + j, &k);
    idx[j] = (int32_t)k;
  }
  geo[0] = H.dim[0]; geo[1] = H.dim[1]; geo[2] = H.dim[2]; geo[3] = H.cells; geo[4] = budget; geo[5] = H.n_valid;
  for (int a = 0; a < 3; ++a) geo[6 + a] = nng_bits(H.lo[a]);
  geo[9] = nng_bits(H.ih);
  return 0;
}

// one axis of the index's arithmetic, for tests that place coordinates on either side of a cell face
extern "C" void ns_axis(float x, float lo, float ih, uint32_t dim, float* u, int32_t* cell) {
  *u = nng_u(x, lo, ih);
  *cell = nng_cell(*u, dim);
}
