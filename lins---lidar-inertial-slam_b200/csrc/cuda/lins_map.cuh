// lins_map.cuh — row F2 of SURVEY.md §8(f): the mapping node's scan-to-map refinement on the device.
//   reference: lins/src/lidar_mapping_node.cpp  cornerOptimization :1351-1461, surfOptimization :1463-1524,
//              LMOptimization :1526-1633 (rows of matA / matB), pointAssociateToMap :594-608
// Split of one iteration:
//   lins_map_knn_kernel   exact 5-NN of every (re-projected) feature point in the map, brute force: the map is
//                         streamed through shared memory in tiles and cut into slices across the grid so that all
//                         SMs work (a few thousand queries alone would fill only ~25 CTAs); every (query, slice)
//                         pair leaves a sorted partial list.  f32 ((dx*dx)+dy*dy)+dz*dz, ascending (distance, index).
//   lins_map_knn_grid_kernel  the same 5-NN through a hashed uniform grid, for every point that can be accepted.
//   lins_map_fit_kernel   merges the partial lists, then per point: line fit (covariance + cv::eigen 3x3) or plane
//                         fit (cv::solve QR 5x3), validity tests, weight, coefficients, the row of matA / matB, and
//                         the f64 block reduction of A^T A (21) and A^T B (6).
//   lins_map_lm_kernel    sums the block partials in a fixed order, rounds to f32, takes the 6x6 LM step and derives
//                         the next pass's sin / cos.  The first pass's sin / cos are evaluated on the host in f32, so
//                         everything the device computes for it is f32 + - * / sqrt, which IEEE fixes bit for bit:
//                         indices, coefficients and masks equal the CPU oracle exactly.
// Every kernel but the brute force serves a table of slots (MapSlot): the lockstep mappers' many, or the one slot of
// lins_gpu_map_set / scan2map / map_associate.
// The small OpenCV kernels (cv::eigen = cyclic Jacobi, cv::solve(DECOMP_QR) = Householder) are restated in
// lins_cv_small.hpp, shared by host and device.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../host/lins_cv_small.hpp"
#include "lins_map_types.cuh"

namespace lins_map {

constexpr int kKnnThreads = 128;
constexpr int kTile = 2048;      // map points per shared-memory tile (32 KB)
constexpr int kFitThreads = 128;
constexpr int kRowAcc = 27;      // 21 (upper triangle of A^T A) + 6 (A^T B)

__device__ __forceinline__ float3 associate_to_map(const float4 pi, const PassConsts& c) {  // :594-608
  const float x1 = c.cYaw * pi.x - c.sYaw * pi.y;
  const float y1 = c.sYaw * pi.x + c.cYaw * pi.y;
  const float z1 = pi.z;
  const float x2 = x1;
  const float y2 = c.cRoll * y1 - c.sRoll * z1;
  const float z2 = c.sRoll * y1 + c.cRoll * z1;
  return make_float3(c.cPitch * x2 + c.sPitch * z2 + c.tX, y2 + c.tY, -c.sPitch * x2 + c.cPitch * z2 + c.tZ);
}

struct Top5 {
  float d[5];
  int i[5];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < 5; ++k) { d[k] = __int_as_float(0x7f800000); i[k] = -1; }
  }
  // strict <: among equal distances the earlier (lower) index stays in front
  __device__ __forceinline__ void insert(float dist, int idx) {
    if (!(dist < d[4])) return;
    d[4] = dist; i[4] = idx;
#pragma unroll
    for (int k = 4; k > 0; --k) {
      if (d[k] < d[k - 1]) { const float td = d[k]; d[k] = d[k - 1]; d[k - 1] = td; const int ti = i[k]; i[k] = i[k - 1]; i[k - 1] = ti; }
    }
  }
};

// grid (query blocks, slices).  part_d / part_i: [n_q][n_slices][5]
__global__ void __launch_bounds__(kKnnThreads) lins_map_knn_kernel(const float4* __restrict__ q, int n_q, const float4* __restrict__ map, int n_map,
                                                                   int slice_len, const PassConsts* __restrict__ pcp, const MapLoopState* __restrict__ st,
                                                                   float* __restrict__ part_d, int* __restrict__ part_i) {
  if (st && st->done) return;  // (the queued tail of a converged scan2map loop)
  const PassConsts pc = *pcp;
  __shared__ float4 tile[kTile];
  const int qi = blockIdx.x * kKnnThreads + threadIdx.x;
  const int slice = blockIdx.y, n_slices = gridDim.y;
  const int m0 = slice * slice_len, m1 = min(n_map, m0 + slice_len);
  float3 s = make_float3(0.f, 0.f, 0.f);
  if (qi < n_q) s = associate_to_map(__ldg(&q[qi]), pc);
  Top5 t;
  t.init();
  for (int base = m0; base < m1; base += kTile) {
    const int cnt = min(kTile, m1 - base);
    __syncthreads();
    for (int j = threadIdx.x; j < cnt; j += kKnnThreads) tile[j] = __ldg(&map[base + j]);
    __syncthreads();
    if (qi < n_q) {
#pragma unroll 4
      for (int j = 0; j < cnt; ++j) {
        const float4 m = tile[j];  // same address for the whole warp: a broadcast
        const float dx = __fsub_rn(s.x, m.x), dy = __fsub_rn(s.y, m.y), dz = __fsub_rn(s.z, m.z);
        const float dist = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (dist < t.d[4]) t.insert(dist, base + j);
      }
    }
  }
  if (qi < n_q) {
    const size_t o = ((size_t)qi * n_slices + slice) * 5;
#pragma unroll
    for (int k = 0; k < 5; ++k) { part_d[o + k] = t.d[k]; part_i[o + k] = t.i[k]; }
  }
}

struct FitOut { float c[4]; bool sel; };

// the body of cornerOptimization for one point (:1360-1458)
__device__ __forceinline__ FitOut corner_fit(const float4* __restrict__ map, const float3 sel, const int ind[5], const float dist[5]) {
  FitOut o;
  o.c[0] = o.c[1] = o.c[2] = o.c[3] = 0.f; o.sel = false;
  if (!(dist[4] < 1.0)) return o;
  float px[5], py[5], pz[5];
  float cx = 0, cy = 0, cz = 0;
#pragma unroll
  for (int j = 0; j < 5; ++j) { const float4 m = __ldg(&map[ind[j]]); px[j] = m.x; py[j] = m.y; pz[j] = m.z; cx += m.x; cy += m.y; cz += m.z; }
  cx /= 5; cy /= 5; cz /= 5;
  float a11 = 0, a12 = 0, a13 = 0, a22 = 0, a23 = 0, a33 = 0;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const float ax = px[j] - cx, ay = py[j] - cy, az = pz[j] - cz;
    a11 += ax * ax; a12 += ax * ay; a13 += ax * az; a22 += ay * ay; a23 += ay * az; a33 += az * az;
  }
  a11 /= 5; a12 /= 5; a13 /= 5; a22 /= 5; a23 /= 5; a33 /= 5;
  float A[9] = {a11, a12, a13, a12, a22, a23, a13, a23, a33}, D[3], V[9];
  lins_cv::jacobi_eigen<3>(A, D, V);
  if (D[0] > 3 * D[1]) {
    const float x0 = sel.x, y0 = sel.y, z0 = sel.z;
    const float x1 = (float)((double)cx + 0.1 * (double)V[0]), y1 = (float)((double)cy + 0.1 * (double)V[1]), z1 = (float)((double)cz + 0.1 * (double)V[2]);
    const float x2 = (float)((double)cx - 0.1 * (double)V[0]), y2 = (float)((double)cy - 0.1 * (double)V[1]), z2 = (float)((double)cz - 0.1 * (double)V[2]);
    const float m11 = (x0 - x1) * (y0 - y2) - (x0 - x2) * (y0 - y1);
    const float m12 = (x0 - x1) * (z0 - z2) - (x0 - x2) * (z0 - z1);
    const float m13 = (y0 - y1) * (z0 - z2) - (y0 - y2) * (z0 - z1);
    const float a012 = sqrtf(m11 * m11 + m12 * m12 + m13 * m13);
    const float l12 = sqrtf((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2) + (z1 - z2) * (z1 - z2));
    const float la = ((y1 - y2) * m11 + (z1 - z2) * m12) / a012 / l12;
    const float lb = -((x1 - x2) * m11 - (z1 - z2) * m13) / a012 / l12;
    const float lc = -((x1 - x2) * m12 + (y1 - y2) * m13) / a012 / l12;
    const float ld2 = a012 / l12;
    const float s = (float)(1 - 0.9 * (double)fabsf(ld2));
    o.c[0] = s * la; o.c[1] = s * lb; o.c[2] = s * lc; o.c[3] = s * ld2;
    o.sel = (double)s > 0.1;
  }
  return o;
}

// the body of surfOptimization for one point (:1471-1521)
__device__ __forceinline__ FitOut surf_fit(const float4* __restrict__ map, const float3 sel, const int ind[5], const float dist[5]) {
  FitOut o;
  o.c[0] = o.c[1] = o.c[2] = o.c[3] = 0.f; o.sel = false;
  if (!(dist[4] < 1.0)) return o;
  float A0[15], B0[5] = {-1.f, -1.f, -1.f, -1.f, -1.f};
  float px[5], py[5], pz[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) { const float4 m = __ldg(&map[ind[j]]); px[j] = m.x; py[j] = m.y; pz[j] = m.z; A0[3 * j] = m.x; A0[3 * j + 1] = m.y; A0[3 * j + 2] = m.z; }
  float pa = 0, pb = 0, pc = 0, pd = 1;
  if (lins_cv::qr_solve<5, 3>(A0, B0)) { pa = B0[0]; pb = B0[1]; pc = B0[2]; }  // a failed cv::solve zeroes its output
  const float ps = sqrtf(pa * pa + pb * pb + pc * pc);
  pa /= ps; pb /= ps; pc /= ps; pd /= ps;
  bool planeValid = true;
#pragma unroll
  for (int j = 0; j < 5; ++j)
    if ((double)fabsf(pa * px[j] + pb * py[j] + pc * pz[j] + pd) > 0.2) planeValid = false;
  if (planeValid) {
    const float pd2 = pa * sel.x + pb * sel.y + pc * sel.z + pd;
    const float s = (float)(1 - 0.9 * (double)fabsf(pd2) / (double)sqrtf(sqrtf(sel.x * sel.x + sel.y * sel.y + sel.z * sel.z)));
    o.c[0] = s * pa; o.c[1] = s * pb; o.c[2] = s * pc; o.c[3] = s * pd2;
    o.sel = (double)s > 0.1;
  }
  return o;
}

// one row of matA / matB (:1549-1593)
__device__ __forceinline__ void lm_row(const float4 po, const float* c, const PassConsts& k, float row[6], float& b) {
  const float srx = k.srx, crx = k.crx, sry = k.sry, cry = k.cry, srz = k.srz, crz = k.crz;
  row[0] = (crx * sry * srz * po.x + crx * crz * sry * po.y - srx * sry * po.z) * c[0] +
           (-srx * srz * po.x - crz * srx * po.y - crx * po.z) * c[1] +
           (crx * cry * srz * po.x + crx * cry * crz * po.y - cry * srx * po.z) * c[2];
  row[1] = ((cry * srx * srz - crz * sry) * po.x + (sry * srz + cry * crz * srx) * po.y + crx * cry * po.z) * c[0] +
           ((-cry * crz - srx * sry * srz) * po.x + (cry * srz - crz * srx * sry) * po.y - crx * sry * po.z) * c[2];
  row[2] = ((crz * srx * sry - cry * srz) * po.x + (-cry * crz - srx * sry * srz) * po.y) * c[0] +
           (crx * crz * po.x - crx * srz * po.y) * c[1] +
           ((sry * srz + cry * crz * srx) * po.x + (crz * sry - cry * srx * srz) * po.y) * c[2];
  row[3] = c[0]; row[4] = c[1]; row[5] = c[2];
  b = -c[3];
}

// One thread per feature point.  partial: [gridDim.x][kRowAcc + 1] (the last entry = selected points of the block).
// Block b serves slot blk_slot[b] (n_sl slots), whose queries q[CORNER ? 0 : 1] start at its block blk[...]; a block
// never straddles two slots, so each slot's partials are those of a run of that slot alone.  part_d / part_i:
// [rows][n_slices][5]
// (n_slices > 1: the brute-force slices of a one-slot table, whose rows are its query indices).  The dense outputs
// (knn_out, coeff_out, mask_out; null: not written) are indexed by the slot's query index.
template <bool CORNER>
__global__ void __launch_bounds__(kFitThreads) lins_map_fit_kernel(int n_slices, const float* __restrict__ part_d,
                                                                   const int* __restrict__ part_i, const PassConsts* __restrict__ pcp,
                                                                   const MapLoopState* __restrict__ st, int32_t* __restrict__ knn_out,
                                                                   float* __restrict__ coeff_out, uint8_t* __restrict__ mask_out,
                                                                   double* __restrict__ partial, const MapSlot* __restrict__ sl, int n_sl,
                                                                   const int* __restrict__ blk_slot) {
  constexpr int K = CORNER ? 0 : 1;
  const int row = blockIdx.x * kFitThreads + threadIdx.x;
  const int slot = n_sl == 1 ? 0 : blk_slot[blockIdx.x];  // (a one-slot table skips the lookup's latency)
  // the slot's record, loop state and constants are loaded before any branch on them, so their latencies overlap
  const MapSlot& v = sl[slot];
  const bool done = st && st[slot].done;
  const PassConsts pc = pcp[slot];
  const float4* __restrict__ q = v.q[K];
  const float4* __restrict__ map = v.map[K];
  const int n_q = v.nq[K], qi = (blockIdx.x - v.blk[K]) * kFitThreads + threadIdx.x;
  if (done) return;
  double acc[kRowAcc];
#pragma unroll
  for (int k = 0; k < kRowAcc; ++k) acc[k] = 0.0;
  int nsel = 0;
  if (qi < n_q) {
    // merge the slices' sorted lists: slices are ascending index ranges, so "strictly smaller displaces" keeps the
    // lower index in front among equal distances.  A list is ascending, so it is left at its first entry that does
    // not beat the current fifth best (most slices contribute nothing).
    Top5 t;
    t.init();
    for (int s = 0; s < n_slices; ++s) {
      const size_t o = ((size_t)row * n_slices + s) * 5;
      for (int k = 0; k < 5; ++k) {
        const int idx = part_i[o + k];
        const float dk = part_d[o + k];
        if (idx < 0 || !(dk < t.d[4])) break;
        t.insert(dk, idx);
      }
    }
    const float4 po = __ldg(&q[qi]);
    const float3 sel = associate_to_map(po, pc);
    const FitOut f = CORNER ? corner_fit(map, sel, t.i, t.d) : surf_fit(map, sel, t.i, t.d);
    if (knn_out) {
#pragma unroll
      for (int k = 0; k < 5; ++k) knn_out[5 * (size_t)qi + k] = t.i[k];
    }
    if (coeff_out) {
#pragma unroll
      for (int k = 0; k < 4; ++k) coeff_out[4 * (size_t)qi + k] = f.c[k];
    }
    if (mask_out) mask_out[qi] = f.sel ? 1 : 0;
    if (f.sel) {
      float row[6], b;
      lm_row(po, f.c, pc, row, b);
      int k = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int c = a; c < 6; ++c) acc[k++] = (double)row[a] * (double)row[c];
#pragma unroll
      for (int a = 0; a < 6; ++a) acc[21 + a] = (double)row[a] * (double)b;
      nsel = 1;
    }
  }
  // fixed-tree block reduction (deterministic)
  __shared__ double wsum[kFitThreads / 32][kRowAcc];
  __shared__ int wcnt[kFitThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kRowAcc; ++k) {
    double v = acc[k];
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    if (lane == 0) wsum[warp][k] = v;
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) nsel += __shfl_xor_sync(0xffffffffu, nsel, m);
  if (lane == 0) wcnt[warp] = nsel;
  __syncthreads();
  if (threadIdx.x < kRowAcc) {
    double v = 0;
    for (int w = 0; w < kFitThreads / 32; ++w) v += wsum[w][threadIdx.x];
    partial[(size_t)blockIdx.x * (kRowAcc + 1) + threadIdx.x] = v;
  }
  if (threadIdx.x == kRowAcc) {
    int c = 0;
    for (int w = 0; w < kFitThreads / 32; ++w) c += wcnt[w];
    partial[(size_t)blockIdx.x * (kRowAcc + 1) + kRowAcc] = (double)c;
  }
}


// =====================================================================================================================
// Reference-scale path (VERDICT r1 item 9): exact 5-NN through a hashed uniform grid + the LM step on the device.
//
// Grid.  The reference accepts a feature point only if its FIFTH neighbour lies within 1 m (pointSearchSqDis[4] < 1.0,
// lidar_mapping_node.cpp:1374, :1481), so the only neighbours that matter are those within 1 m, and every map point
// whose f32 distance is < 1 lies in the 3 x 3 x 3 block of 1 m cells around the query's cell (cells of the exact
// difference: grid_cell, DESIGN.md §4.4).  The grid build bucket-sorts
// the map by hash(cell) (the role of kdtree*FromMap->setInputCloud, :1637-1638); a query warp gives one cell of the
// block to each of 27 lanes (cells that hash to the same bucket are visited once), every lane keeps the five smallest
// (distance, index) keys of its bucket — points of other cells that share the bucket are just extra candidates — and a
// five-round warp minimum merges the lanes.  If the merged fifth distance is < 1, all five are exact (any closer point
// would have been in the block); otherwise the true fifth distance is >= 1 as well and the point is rejected either
// way.  Keys are (f32 distance bits, index), so ties resolve to the lower index exactly like the brute-force scan.
//
// LM loop.  The loop keeps transformTobeMapped, matP / isDegenerate and the report on the device (MapLoopState): per
// iteration the 5-NN kernel, the fit / reduction kernel and a one-warp kernel that sums the block partials in a fixed
// order, takes the 6 x 6 step (LMOptimization :1598-1632, lins_cv_small.hpp) and prepares the next iteration's sin / cos;
// once it sets `done`, the launches still queued return at once.  One D2H and one synchronisation per call.
constexpr float kGridCell = 1.0f;  // >= the 1 m acceptance radius
constexpr int kGridKnnWarps = 4;   // query warps per CTA


// Cell indices are taken as unsigned so that the block's neighbour arithmetic (cx - 1, cx + 1) wraps instead of
// overflowing at a saturated cell; the hash sees the same bits either way.
__device__ __forceinline__ unsigned grid_hash(unsigned ix, unsigned iy, unsigned iz) {
  return (ix * 73856093u) ^ (iy * 19349663u) ^ (iz * 83492791u);
}
// floor(x - ox) of the EXACT difference: f32 operands subtract exactly in f64 unless their exponents are ~29 apart, and
// then the f64 rounding is far below the 2^-25 margin the block rule needs (DESIGN.md §4.4).  An f32 x - ox would round
// near a power of two from the origin and could put a neighbour whose f32 distance is < 1 two cells away.  The
// conversion floors and saturates (NaN -> 0), so far and non-finite coordinates land in the edge cells.
__device__ __forceinline__ void grid_cell(const GridIndex& g, float x, float y, float z, unsigned& ix, unsigned& iy, unsigned& iz) {
  static_assert(kGridCell == 1.0f, "grid_cell assumes 1 m cells");
  ix = (unsigned)__double2int_rd((double)x - (double)g.ox);
  iy = (unsigned)__double2int_rd((double)y - (double)g.oy);
  iz = (unsigned)__double2int_rd((double)z - (double)g.oz);
}
// counting sort of every slot's maps by bucket: count, (host-launched) scan, scatter.  Point i of the n (n_sl slots) is
// point i - m0[k] of slot s's map k, with the slot's grid and its buckets from bucket0[k] on; n counts the maps'
// capacities, and n_dev points at the device-resident number of a map's real points.
struct GridPoint { const float4* map; int i; const int* n_dev; GridIndex g; int b0; };
__device__ __forceinline__ GridPoint grid_point(int i, const MapSlot* sl, int n_sl) {
  int lo = 0, hi = n_sl - 1;  // the last slot whose maps start at or before i
  while (lo < hi) { const int m = (lo + hi + 1) >> 1; if (sl[m].m0[0] <= i) lo = m; else hi = m - 1; }
  const MapSlot& v = sl[lo];
  const int k = i >= v.m0[1];
  return GridPoint{v.map[k], i - v.m0[k], v.n_map[k], v.g[k], v.bucket0[k]};
}
__global__ void lins_grid_count_kernel(int n, int* __restrict__ count, const MapSlot* __restrict__ sl, int n_sl) {
  const int i0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (i0 >= n) return;
  const GridPoint gp = grid_point(i0, sl, n_sl);
  if (gp.i >= *gp.n_dev) return;
  const float4 p = __ldg(&gp.map[gp.i]);
  unsigned ix, iy, iz;
  grid_cell(gp.g, p.x, p.y, p.z, ix, iy, iz);
  atomicAdd(&count[gp.b0 + (grid_hash(ix, iy, iz) & gp.g.mask)], 1);
}
__global__ void lins_grid_scatter_kernel(int n, int* __restrict__ cursor, float4* __restrict__ sorted, const MapSlot* __restrict__ sl, int n_sl) {
  const int i0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (i0 >= n) return;
  const GridPoint gp = grid_point(i0, sl, n_sl);
  if (gp.i >= *gp.n_dev) return;
  const float4 p = __ldg(&gp.map[gp.i]);
  unsigned ix, iy, iz;
  grid_cell(gp.g, p.x, p.y, p.z, ix, iy, iz);
  const int pos = atomicAdd(&cursor[gp.b0 + (grid_hash(ix, iy, iz) & gp.g.mask)], 1);
  sorted[pos] = make_float4(p.x, p.y, p.z, __int_as_float(gp.i));
}

struct Top5K {  // five smallest (distance bits, index) keys, ascending
  unsigned long long k[5];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int j = 0; j < 5; ++j) k[j] = 0xFFFFFFFFFFFFFFFFull;
  }
  __device__ __forceinline__ void insert(unsigned long long key) {
    if (!(key < k[4])) return;
    k[4] = key;
#pragma unroll
    for (int j = 4; j > 0; --j)
      if (k[j] < k[j - 1]) { const unsigned long long t = k[j]; k[j] = k[j - 1]; k[j - 1] = t; }
  }
};

// one warp per query; part_d / part_i: [n_rows][1][5] (a single "slice" for lins_map_fit_kernel).  n_rows rows in
// lins_map_fit_kernel's blocks, row r in block r / kFitThreads of slot blk_slot[that block] (n_sl slots), map `kind` (0
// corner, 1 surf).
__global__ void __launch_bounds__(kGridKnnWarps * 32) lins_map_knn_grid_kernel(int n_rows, const PassConsts* __restrict__ pcp,
                                                                               const MapLoopState* __restrict__ st,
                                                                               float* __restrict__ part_d, int* __restrict__ part_i,
                                                                               const MapSlot* __restrict__ sl, int n_sl, const int* __restrict__ blk_slot,
                                                                               int kind) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kGridKnnWarps + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const int slot = n_sl == 1 ? 0 : blk_slot[row / kFitThreads];  // (a one-slot table skips the lookup's latency)
  // the slot's record, loop state and constants are loaded before any branch on them, so their latencies overlap
  const MapSlot& v = sl[slot];
  const bool done = st && st[slot].done;
  const PassConsts pc = pcp[slot];
  const int qi = row - v.blk[kind] * kFitThreads;
  const float4* __restrict__ q = v.q[kind];
  const GridIndex g = v.g[kind];
  if (done || qi >= v.nq[kind]) return;
  const float3 s = associate_to_map(__ldg(&q[qi]), pc);
  unsigned cx, cy, cz;
  grid_cell(g, s.x, s.y, s.z, cx, cy, cz);
  unsigned b = 0xFFFFFF00u + (unsigned)lane;  // lanes 27..31: a bucket id nobody shares, never scanned
  if (lane < 27) b = grid_hash(cx + lane % 3 - 1u, cy + (lane / 3) % 3 - 1u, cz + lane / 9 - 1u) & g.mask;
  const unsigned same = __match_any_sync(0xffffffffu, b);
  const bool mine = lane < 27 && (__ffs(same) - 1) == lane;  // cells of the block that share a bucket are visited once
  Top5K t;
  t.init();
  if (mine && s.x == s.x) {
    const int p0 = g.start[b], p1 = g.start[b + 1];
    for (int p = p0; p < p1; ++p) {
      const float4 m = __ldg(&g.pts[p]);
      const float dx = __fsub_rn(s.x, m.x), dy = __fsub_rn(s.y, m.y), dz = __fsub_rn(s.z, m.z);
      const float dist = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      // never a NaN or +inf distance, like the brute-force scan
      if (dist < __int_as_float(0x7f800000)) t.insert(((unsigned long long)__float_as_uint(dist) << 32) | (unsigned)__float_as_int(m.w));
    }
  }
  // five rounds: the smallest head among the lanes' ascending lists
  int head = 0;
  const size_t o = (size_t)row * 5;
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    const unsigned long long mykey = head < 5 ? t.k[0] : 0xFFFFFFFFFFFFFFFFull;
    const unsigned hi = (unsigned)(mykey >> 32), lo = (unsigned)mykey;
    const unsigned mhi = __reduce_min_sync(0xffffffffu, hi);
    const unsigned mlo = __reduce_min_sync(0xffffffffu, hi == mhi ? lo : 0xffffffffu);
    if (hi == mhi && lo == mlo && mykey != 0xFFFFFFFFFFFFFFFFull) {  // unique keys: exactly one lane
#pragma unroll
      for (int j = 0; j < 4; ++j) t.k[j] = t.k[j + 1];
      t.k[4] = 0xFFFFFFFFFFFFFFFFull;
      ++head;
    }
    if (lane == 0) {
      const bool none = mhi == 0xffffffffu && mlo == 0xffffffffu;
      part_d[o + r] = none ? __int_as_float(0x7f800000) : __uint_as_float(mhi);
      part_i[o + r] = none ? -1 : (int)mlo;
    }
  }
}

__device__ __forceinline__ void pass_consts_from(const float* T, PassConsts& pc) {  // :579-592, :1527-1532 (f32 like the reference)
  pc.cRoll = (float)cos((double)T[0]); pc.sRoll = (float)sin((double)T[0]);
  pc.cPitch = (float)cos((double)T[1]); pc.sPitch = (float)sin((double)T[1]);
  pc.cYaw = (float)cos((double)T[2]); pc.sYaw = (float)sin((double)T[2]);
  pc.tX = T[3]; pc.tY = T[4]; pc.tZ = T[5];
  pc.srx = pc.sRoll; pc.crx = pc.cRoll; pc.sry = pc.sPitch; pc.cry = pc.cPitch; pc.srz = pc.sYaw; pc.crz = pc.cYaw;
}

// one warp per slot, one block each (the 6 x 6 step itself is one thread): block partials -> matAtA / matAtB (f32), the LM
// step, the next iteration's constants.  Every matrix lives in shared memory (plain dynamically indexed loads / stores).
// Slot s sums its corner blocks [blk[0], blk[0] + nblk[0]) and then its surf blocks, which start at nblocks (the corner
// launch's block count) + blk[1].
__global__ void lins_map_lm_kernel(const double* __restrict__ partial, int nblocks, int iter, MapLoopState* __restrict__ st,
                                   PassConsts* __restrict__ pc_next, const MapSlot* __restrict__ sl) {
  st += blockIdx.x; pc_next += blockIdx.x;
  const MapSlot& m = sl[blockIdx.x];  // (loaded with the done flag)
  const int c0 = m.blk[0], c1 = c0 + m.nblk[0], s0 = nblocks + m.blk[1], s1 = s0 + m.nblk[1];
  if (st->done) return;
  __shared__ double acc[kRowAcc + 1];
  __shared__ float AtA[36], AtB[6], Aw[36], X[6], Ae[36], E[6], V[36], V2[36], Vc[36], Vinv[36], X2[6];
  if (threadIdx.x <= kRowAcc) {  // lane k sums column k of the block partials, in a fixed order: corner blocks, then surf
    double v = 0.0;               // blocks (laserCloudOri's order)
    for (int b = c0; b < c1; ++b) v += partial[(size_t)b * (kRowAcc + 1) + threadIdx.x];
    for (int b = s0; b < s1; ++b) v += partial[(size_t)b * (kRowAcc + 1) + threadIdx.x];
    acc[threadIdx.x] = v;
  }
  __syncwarp();
  if (threadIdx.x != 0) return;
  int k = 0;
  for (int a = 0; a < 6; ++a)
    for (int c = a; c < 6; ++c) { AtA[a * 6 + c] = (float)acc[k]; AtA[c * 6 + a] = (float)acc[k]; ++k; }
  for (int a = 0; a < 6; ++a) AtB[a] = (float)acc[21 + a];
  const int n_sel = (int)acc[kRowAcc];
  st->iters = iter + 1;
  st->n_sel[iter] = n_sel;
  if (n_sel < 50) return;  // LMOptimization returns false before touching the transform (:1535-1537)
  for (int i = 0; i < 36; ++i) Aw[i] = AtA[i];
  for (int i = 0; i < 6; ++i) X[i] = AtB[i];
  if (!lins_cv::qr_solve<6, 6>(Aw, X)) for (int i = 0; i < 6; ++i) X[i] = 0.f;  // a failed cv::solve zeroes matX
  if (iter == 0) {
    for (int i = 0; i < 36; ++i) Ae[i] = AtA[i];
    lins_cv::jacobi_eigen<6>(Ae, E, V);
    for (int i = 0; i < 36; ++i) { V2[i] = V[i]; Vc[i] = V[i]; }
    st->isDegenerate = 0;
    for (int i = 5; i >= 0; --i) {
      if (E[i] < 100.f) { for (int j = 0; j < 6; ++j) V2[i * 6 + j] = 0; st->isDegenerate = 1; }
      else break;
    }
    if (!lins_cv::lu_invert<6>(Vc, Vinv)) for (int i = 0; i < 36; ++i) Vinv[i] = 0.f;
    lins_cv::gemm<6, 6, 6>(Vinv, V2, st->matP);
  }
  if (st->isDegenerate) {
    for (int i = 0; i < 6; ++i) X2[i] = X[i];
    lins_cv::gemm<6, 6, 1>(st->matP, X2, X);
  }
  for (int i = 0; i < 6; ++i) st->T[i] += X[i];
  const float r0 = X[0] * 57.29578f, r1 = X[1] * 57.29578f, r2 = X[2] * 57.29578f;  // pcl::rad2deg(float)
  const float dR = (float)sqrt((double)r0 * (double)r0 + (double)r1 * (double)r1 + (double)r2 * (double)r2);
  const float t0 = X[3] * 100, t1 = X[4] * 100, t2 = X[5] * 100;
  const float dT = (float)sqrt((double)t0 * (double)t0 + (double)t1 * (double)t1 + (double)t2 * (double)t2);
  st->delta_r[iter] = dR; st->delta_t[iter] = dT;
  if (dR < 0.05 && dT < 0.05) { st->converged = 1; st->done = 1; return; }
  pass_consts_from(st->T, *pc_next);
}

}  // namespace lins_map
