// ski.cu -- SKI / KISS-GP kernel-matmul  out = W (T_0 x T_1 x ... x T_{d-1}) W^T V  as a backend of gp_plan (SURVEY.md section 8f row 3,
// BASELINE configs[4]: N = 1e6, d = 3, grid 100^3).
//
// Replaces (reference, paths under /root/reference/gpytorch):
//   Interpolation.interpolate                       utils/interpolation.py:15-167   (Keys cubic convolution, 4 nodes per dimension,
//                                                   one-hot snapping in the first / last grid cell)
//   GridInterpolationKernel.forward / _compute_grid kernels/grid_interpolation_kernel.py:132-213
//   GridKernel.forward (Toeplitz / Kronecker K_uu)  kernels/grid_kernel.py:107-177
//   InterpolatedLinearOperator._matmul, KroneckerProductLinearOperator / ToeplitzLinearOperator._matmul   (linear_operator, absent)
// The interpolation matrix W (4^d non-zeros per row) is never stored expanded: per row and dimension the plan keeps the first
// node index and the 4 one-dimensional weights (16 d + 4 d bytes per row instead of 4^d (8 + 4)); the 4^d products are re-formed
// in registers by the scatter and gather kernels.  The points are bucketed once per data update by the tile of their first
// node, so that a CTA works on the (E + 3)^d grid nodes of one tile in shared memory.  A product is three passes:
//   scatter  U  = W^T V           per tile: shared-memory accumulation, then one red.global.add.v4.f32 per touched node into the
//                                 [M][16] grid block (M = prod G_i; 64 MB at 100^3)
//   modes    U' = (T_0 x ... x T_{d-1}) U   one [G x G] product per dimension on the tensor cores: from the dense factor at
//                                 G <= 128 (the Toeplitz structure saves nothing at G = 100: an FFT of length 2G-2 costs as many
//                                 flops as the direct product), from the factor's generating column t[|a - b|] above, skipping the
//                                 k-chunks where t is exactly zero (O(G band) instead of O(G^2))
//   gather   out = W U'           per tile: node block staged in shared memory, 4^d reads per (row, column group) from there,
//                                 written as the K.V partial block the mBCG finish kernels read (outputscale / noise applied there)
// and the bilinear derivative (hyper-parameter gradients) is d + 1 sweeps of the mode products between two scatters and a dot.
// Prediction on the grid (gp_ski_grid_matmul / gp_ski_interp_matmul, the reference's InterpolatedPredictionStrategy) reuses the
// scatter and the mode products to build grid caches s K_uu W^T V, and interpolates a user grid matrix C [M][t] to the points
// with ski_interp_tiled_kernel, the gather generalised to any t.
// HBM/L2-bound: algorithmic bytes per product (SURVEY.md section 8f) = N 4^d (4 + 8) B as the reference stores W explicitly.
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "gp_common.cuh"
#include "ski_rows.cuh"

namespace gp {

constexpr int SKI_MAXD = 4;
constexpr int SKI_DENSE_G = 128;       // largest grid dimension whose mode product stages its dense factor (ski_mode_kernel)
constexpr int SKI_MAX_G = 131072;      // largest grid dimension (ski_mode_banded_kernel above SKI_DENSE_G)

struct SkiGeom {
  int d;
  int G[SKI_MAXD];
  int64_t stride[SKI_MAXD];   // flat index stride of dimension i (dimension 0 slowest, interpolation.py:157-163)
  float lo[SKI_MAXD], step[SKI_MAXD];
  int64_t M;
};

// Keys (1981) cubic convolution kernel, a = -1/2, in the reference's Horner order (utils/interpolation.py:33-43)
__device__ __forceinline__ float cubic_w(float s) {
  const float u = fabsf(s);
  const float nearv = ((1.5f * u - 2.5f) * u) * u + 1.f;
  const float farv = ((-0.5f * u + 2.5f) * u - 4.f) * u + 2.f;
  return (u < 1.f) ? nearv : farv;     // u in [0, 2]: 1 - clamp(floor(u), 0, 1) selects the branch
}

// its derivative dw/ds = sign(s) (4.5 u^2 - 5 u) for u = |s| < 1, sign(s) (-1.5 u^2 + 5 u - 4) for 1 <= u < 2 (what autograd gives
// through the reference's expression; 0 at s = 0)
__device__ __forceinline__ float cubic_dw(float s) {
  const float u = fabsf(s);
  const float nearv = (4.5f * u - 5.f) * u;
  const float farv = (-1.5f * u + 5.f) * u - 4.f;
  const float v = (u < 1.f) ? nearv : farv;
  return (s < 0.f) ? -v : v;
}

// Interpolation data of coordinate x on one grid axis (first node lo, spacing step, G nodes): returns the first of the 4 nodes
// and their weights w; with DERIV also dw = dw/dx (1 / step per unit of distance; exactly 0 in the one-hot first / last cells,
// as the reference's autograd gives).  ski_interp_kernel and ski_input_grad_tiled_kernel both call this, so they pick the same cell.
template <bool DERIV>
__device__ __forceinline__ int ski_axis_weights(float x, float lo, float step, int G, float (&w)[4], float (&dw)[4]) {
  const float h = fmaxf(step, 1e-10f);
  const float t = (x - lo) / h;
  const float cell = floorf(t);
  const float frac = t - cell;
  int f = (int)cell - 1;                       // left-most of the 4 nodes
#pragma unroll
  for (int j = 0; j < 4; ++j) w[j] = cubic_w(frac + (float)(1 - j));   // distances f+1, f, f-1, f-2
  if (DERIV) {
#pragma unroll
    for (int j = 0; j < 4; ++j) dw[j] = cubic_dw(frac + (float)(1 - j)) / h;
  }
  if (f < 0 || f > G - 4) {
    // first / last cell: the nearest of the first / last 4 nodes gets weight 1 (interpolation.py:84-131)
    const int base = (f < 0) ? 0 : G - 4;
    int best = 0;
    float bd = 3.4e38f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float dj = fabsf(lo + step * (float)(base + j) - x);
      if (dj < bd) { bd = dj; best = j; }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      w[j] = (j == best) ? 1.f : 0.f;
      if (DERIV) dw[j] = 0.f;
    }
    f = base;
  }
  return f;
}

// per row and dimension: first node index and the 4 weights
__global__ void ski_interp_kernel(const float* __restrict__ X, int64_t n, int64_t ldx, SkiGeom g, int* __restrict__ first,
                                  float* __restrict__ wts, int* __restrict__ oob) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  for (int i = 0; i < g.d; ++i) {
    const float x = X[r * ldx + i];
    const float hi = g.lo[i] + g.step[i] * (float)(g.G[i] - 1);
    if (!(x - g.lo[i] >= -1e-7f) || !(x - hi <= 1e-7f)) *oob = 1;   // "Received data that was out of bounds for the specified grid."
    float w[4], unused[4];
    const int f = ski_axis_weights<false>(x, g.lo[i], g.step[i], g.G[i], w, unused);
    first[r * g.d + i] = f;
#pragma unroll
    for (int j = 0; j < 4; ++j) wts[(r * g.d + i) * 4 + j] = w[j];
  }
}

__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---- spatial tiling of the points -------------------------------------------------------------------------------------------------
// W has 4^d non-zeros per row and neighbouring points share most of their grid nodes.  Touching the [M][16] grid block once per
// (point, node) costs 4 GB of L2 atomics / reads per product at BASELINE C5 (1.3 + 0.8 ms of a 2.3 ms product).  Instead the points
// are bucketed ONCE per data update by the tile of their first node (edge E cells per dimension); a CTA then owns a tile, keeps
// the (E + 3)^d nodes the tile's points can touch in shared memory (<= 85 KB), accumulates / reads them there, and exchanges
// each node with the global grid block once per tile: ~25x less L2 traffic.
struct SkiTiles {
  int E[SKI_MAXD];    // tile edge in cells
  int nt[SKI_MAXD];   // tiles per dimension
  int ntiles;
};

template <int D>
__device__ __forceinline__ int ski_tile_of(const int* __restrict__ fr, const SkiTiles& tl) {
  int t = 0;
#pragma unroll
  for (int i = 0; i < D; ++i) t = t * tl.nt[i] + fr[i] / tl.E[i];
  return t;
}

template <int D>
__global__ void ski_tile_count_kernel(const int* __restrict__ first, int64_t n, SkiTiles tl, int* __restrict__ cnt) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) atomicAdd(cnt + ski_tile_of<D>(first + r * D, tl), 1);
}

// exclusive scan of cnt[0..m) into off[0..m] (one CTA; m <= 2^20, once per data update); cnt is reset to 0 for the fill pass
__global__ void __launch_bounds__(1024) ski_tile_scan_kernel(int* __restrict__ cnt, int m, int* __restrict__ off) {
  __shared__ int sh[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < m; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = (i < m) ? cnt[i] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int add = (threadIdx.x >= o) ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += add;
      __syncthreads();
    }
    if (i < m) { off[i] = carry + sh[threadIdx.x] - v; cnt[i] = 0; }
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[1023];
    __syncthreads();
  }
  if (threadIdx.x == 0) off[m] = carry;
}

// bucket fill: sorted copies of the per-point interpolation data + the permutation back to the caller's row order
template <int D>
__global__ void ski_tile_fill_kernel(const int* __restrict__ first, const float* __restrict__ wts, int64_t n, SkiTiles tl,
                                     const int* __restrict__ off, int* __restrict__ cursor, int* __restrict__ perm,
                                     int* __restrict__ first_s, float* __restrict__ wts_s) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int t = ski_tile_of<D>(first + r * D, tl);
  const int64_t pos = off[t] + atomicAdd(cursor + t, 1);
  perm[pos] = (int)r;
#pragma unroll
  for (int i = 0; i < D; ++i) first_s[pos * D + i] = first[r * D + i];
#pragma unroll
  for (int i = 0; i < D * 4; ++i) wts_s[pos * D * 4 + i] = wts[r * D * 4 + i];
}

// geometry of one tile's node block: base node, extent and row-major pitch per dimension (last dimension fastest)
template <int D>
struct SkiBlock {
  int base[D], ext[D], pitch[D];
  int nodes;
};
template <int D>
__device__ __forceinline__ SkiBlock<D> ski_block_of(int tile, const SkiGeom& g, const SkiTiles& tl) {
  SkiBlock<D> b;
  int rem = tile;
#pragma unroll
  for (int i = D - 1; i >= 0; --i) {
    const int tc = rem % tl.nt[i];
    rem /= tl.nt[i];
    b.base[i] = tc * tl.E[i];
    b.ext[i] = min(tl.E[i] + 3, g.G[i] - b.base[i]);
  }
  int pch = 1;
#pragma unroll
  for (int i = D - 1; i >= 0; --i) { b.pitch[i] = pch; pch *= b.ext[i]; }
  b.nodes = pch;
  return b;
}
// Work item wk = (tile, part) of a tiled pass: crowded tiles (few tiles, many points: small grids in low dimension) are shared by
// `parts` CTAs, part taking the sorted points [p0, p1) of its tile.  False when that range is empty.
__device__ __forceinline__ bool ski_work_range(int64_t wk, int parts, const int* __restrict__ off, int& tile, int& p0, int& p1) {
  tile = (int)(wk / parts);
  const int part = (int)(wk % parts);
  const int t0 = off[tile], tn = off[tile + 1] - t0;
  p0 = t0 + (int)((int64_t)tn * part / parts);
  p1 = t0 + (int)((int64_t)tn * (part + 1) / parts);
  return p0 != p1;
}
// A "row" of a tile's node block fixes the coordinates of dimensions 0 .. D-2: block-local node and global flat index of its
// first node (one division chain per row instead of one per element)
struct SkiRowOrigin {
  int node0;
  int64_t idx0;
};
template <int D>
__device__ __forceinline__ SkiRowOrigin ski_row_origin(const SkiBlock<D>& b, const SkiGeom& g, int row) {
  int rem = row, node0 = 0;
  int64_t idx0 = (int64_t)b.base[D - 1] * g.stride[D - 1];
#pragma unroll
  for (int i = D - 2; i >= 0; --i) {
    const int c = rem % b.ext[i];
    rem /= b.ext[i];
    node0 += c * b.pitch[i];
    idx0 += (int64_t)(b.base[i] + c) * g.stride[i];
  }
  return {node0, idx0};
}
// Row-wise traversal of a tile's node block for the exchanges with the global grid block: the lanes cover (last-dimension node,
// column group) pairs of a row, 8 nodes x 4 groups per pass.  fn(local node, global flat index, column group).
template <int D, typename F>
__device__ __forceinline__ void ski_block_rows(const SkiBlock<D>& b, const SkiGeom& g, int warp, int nwarps, int lane, F fn) {
  const int last = b.ext[D - 1];
  const int nrows = b.nodes / last;
  for (int row = warp; row < nrows; row += nwarps) {
    const auto [node0, idx0] = ski_row_origin<D>(b, g, row);
    for (int c = lane >> 2; c < last; c += 8) fn(node0 + c, idx0 + (int64_t)c * g.stride[D - 1], lane & 3);
  }
}

// neighbour q (base-4 digits, dimension 0 most significant) of the warp's current point: block-local node and weight.  The
// point's 4 D weights live one per lane (lane i * 4 + c holds w_i[c]) and are fetched with shuffles: indexing a per-thread
// array with the run-time digit would put it in local memory (3 GB of L2 traffic per product at C5 in the first version).
// fr[i] = first node of the point in dimension i relative to the block.  All 32 lanes must call this together.
template <int D>
__device__ __forceinline__ void ski_local_nnz(const int (&fr)[D], float myw, const SkiBlock<D>& b, int q, int& node, float& w) {
  node = 0;
  w = 1.f;
#pragma unroll
  for (int i = 0; i < D; ++i) {
    const int c = (q >> (2 * (D - 1 - i))) & 3;
    node += (fr[i] + c) * b.pitch[i];
    w *= __shfl_sync(0xffffffffu, myw, i * 4 + c);
  }
}
// Interpolation data of one sorted point as the warp holds it: lane l < 4 D has weight w_{l / 4}[l % 4], lane l < D the first
// node of dimension l.  Loaded one point ahead of its use (the loads are dependent -- perm -> V row -- and a tile's points are
// visited once: without the look-ahead every point costs a full L2 / HBM round trip).
struct SkiPoint {
  float w;
  int f;
};
template <int D>
__device__ __forceinline__ SkiPoint ski_load_point(const int* __restrict__ first_s, const float* __restrict__ wts_s, int64_t p, int lane) {
  SkiPoint pt;
  pt.w = (lane < 4 * D) ? wts_s[p * (4 * D) + lane] : 0.f;
  pt.f = (lane < D) ? first_s[p * D + lane] : 0;
  return pt;
}
template <int D>
__device__ __forceinline__ void ski_point_first(const SkiPoint& pt, const SkiBlock<D>& b, int (&fr)[D]) {
#pragma unroll
  for (int i = 0; i < D; ++i) fr[i] = __shfl_sync(0xffffffffu, pt.f, i) - b.base[i];
}

// U += W^T V: one CTA (4 warps) per (tile, part), node block in shared memory.  Warp w owns column group w (4 of the 16 columns)
// of EVERY node of the block and visits every point of the tile: its lanes are 32 of the point's 4^D neighbours, all distinct
// nodes, so the accumulation is a plain shared-memory read-modify-write -- no atomics (fp32 atomicAdd on shared memory is a
// compare-and-swap loop on this architecture: ATOMS.CAST.SPIN, 250 cycles per add under contention; the version built on it
// took 2.0 ms per product at C5).
constexpr int SKI_SC_THREADS = 128;
template <int D>
__global__ void __launch_bounds__(SKI_SC_THREADS)
ski_scatter_tiled_kernel(const int* __restrict__ first_s, const float* __restrict__ wts_s, const int* __restrict__ perm,
                         const int* __restrict__ off, SkiGeom g, SkiTiles tl, int parts, const float* __restrict__ V16,
                         float* __restrict__ U) {
  constexpr int NNZ = 1 << (2 * D);
  constexpr int NIT = (NNZ + 31) / 32;
  extern __shared__ __align__(16) float blk[];   // [4 column groups][nodes][4]: a warp's 32 lanes (32 nodes, one column group) then
                                                 // spread over all banks; with [nodes][16] they hit 4 banks (16-way conflicts, 1.3 ms)
  const int tid = threadIdx.x, lane = tid & 31, cg = tid >> 5;
  for (int64_t wk = blockIdx.x; wk < (int64_t)tl.ntiles * parts; wk += gridDim.x) {
    int tile, p0, p1;
    if (!ski_work_range(wk, parts, off, tile, p0, p1)) continue;
    const SkiBlock<D> b = ski_block_of<D>(tile, g, tl);
    __syncthreads();
    for (int e = tid; e < b.nodes * 4; e += SKI_SC_THREADS) reinterpret_cast<float4*>(blk)[e] = make_float4(0, 0, 0, 0);
    __syncthreads();
    float* mine = blk + (size_t)cg * b.nodes * 4;   // this warp's plane
    // two-deep look-ahead: point data and V row of p + 1, permutation entry of p + 2
    SkiPoint pt = ski_load_point<D>(first_s, wts_s, p0, lane);
    float4 v = reinterpret_cast<const float4*>(V16 + (int64_t)perm[p0] * TP)[cg];
    int row_n = (p0 + 1 < p1) ? perm[p0 + 1] : 0;
    for (int p = p0; p < p1; ++p) {
      SkiPoint pt_n = pt;
      float4 v_n = v;
      int row_nn = 0;
      if (p + 1 < p1) {
        pt_n = ski_load_point<D>(first_s, wts_s, p + 1, lane);
        v_n = reinterpret_cast<const float4*>(V16 + (int64_t)row_n * TP)[cg];
        if (p + 2 < p1) row_nn = perm[p + 2];
      }
      int fr[D];
      ski_point_first<D>(pt, b, fr);
      int node[NIT];
      float w[NIT];
#pragma unroll
      for (int k = 0; k < NIT; ++k) {
        const int q = lane + 32 * k;
        ski_local_nnz<D>(fr, pt.w, b, q < NNZ ? q : 0, node[k], w[k]);
        if (q >= NNZ) w[k] = 0.f;
      }
      float4 u[NIT];
#pragma unroll
      for (int k = 0; k < NIT; ++k) u[k] = *reinterpret_cast<const float4*>(mine + node[k] * 4);
#pragma unroll
      for (int k = 0; k < NIT; ++k) {
        if (w[k] != 0.f) {   // lanes of one instruction hit distinct nodes; lanes with w = 0 (padding, one-hot edge cells) stay away
          u[k].x = fmaf(w[k], v.x, u[k].x); u[k].y = fmaf(w[k], v.y, u[k].y); u[k].z = fmaf(w[k], v.z, u[k].z); u[k].w = fmaf(w[k], v.w, u[k].w);
          *reinterpret_cast<float4*>(mine + node[k] * 4) = u[k];
        }
      }
      __syncwarp();
      pt = pt_n; v = v_n; row_n = row_nn;
    }
    __syncthreads();
    ski_block_rows<D>(b, g, cg, SKI_SC_THREADS / 32, lane, [&](int node, int64_t idx, int q4) {
      const float4 x = reinterpret_cast<const float4*>(blk)[q4 * b.nodes + node];
      if (x.x != 0.f || x.y != 0.f || x.z != 0.f || x.w != 0.f) red_add_v4(U + idx * TP + q4 * 4, x);
    });
  }
}

// out[perm[p]] = sum_q w_q U[node_q]: the tile's node block is staged in shared memory once; a warp takes every 8th point, its
// lanes = 8 neighbours x 4 column groups
template <int D>
__global__ void __launch_bounds__(256)
ski_gather_tiled_kernel(const int* __restrict__ first_s, const float* __restrict__ wts_s, const int* __restrict__ perm,
                        const int* __restrict__ off, SkiGeom g, SkiTiles tl, int parts, const float* __restrict__ U,
                        float* __restrict__ out) {
  constexpr int NNZ = 1 << (2 * D);
  extern __shared__ __align__(16) float blk[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, cg = lane & 3;
  for (int64_t wk = blockIdx.x; wk < (int64_t)tl.ntiles * parts; wk += gridDim.x) {
    int tile, p0, p1;
    if (!ski_work_range(wk, parts, off, tile, p0, p1)) continue;
    const SkiBlock<D> b = ski_block_of<D>(tile, g, tl);
    __syncthreads();
    ski_block_rows<D>(b, g, warp, 8, lane, [&](int node, int64_t idx, int q4) {
      reinterpret_cast<float4*>(blk)[node * 4 + q4] = __ldg(reinterpret_cast<const float4*>(U + idx * TP) + q4);
    });
    // first point of this warp: loaded while the block is being staged
    SkiPoint pt = {0.f, 0};
    int row = 0;
    if (p0 + warp < p1) { pt = ski_load_point<D>(first_s, wts_s, p0 + warp, lane); row = perm[p0 + warp]; }
    __syncthreads();
    for (int p = p0 + warp; p < p1; p += 8) {
      SkiPoint pt_n = pt;
      int row_n = row;
      if (p + 8 < p1) { pt_n = ski_load_point<D>(first_s, wts_s, p + 8, lane); row_n = perm[p + 8]; }
      int fr[D];
      ski_point_first<D>(pt, b, fr);
      float4 acc = make_float4(0, 0, 0, 0);
#pragma unroll 2
      for (int k = 0; k < (NNZ + 7) / 8; ++k) {        // warp-uniform trip count: the shuffles need all lanes
        const int q = (lane >> 2) + 8 * k;
        int node;
        float w;
        ski_local_nnz<D>(fr, pt.w, b, q < NNZ ? q : 0, node, w);
        if (q >= NNZ) w = 0.f;
        const float4 u = *reinterpret_cast<const float4*>(blk + node * TP + cg * 4);
        acc.x = fmaf(w, u.x, acc.x); acc.y = fmaf(w, u.y, acc.y); acc.z = fmaf(w, u.z, acc.z); acc.w = fmaf(w, u.w, acc.w);
      }
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {   // lanes with the same column group: fixed tree => deterministic
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
      }
      if (lane < 4) reinterpret_cast<float4*>(out + (int64_t)row * TP)[cg] = acc;
      pt = pt_n; row = row_n;
    }
  }
}

// mode product: tensor viewed as [outer][G][inner] (inner includes the 16 columns): out[o][i][x] = sum_k T[i][k] in[o][k][x],
// i.e. per 64-wide slab of the flattened (outer, inner) space one [G x G] . [G x 64] product.  Runs on the tensor cores as a
// 3xTF32 product (T = T_hi + T_lo and B = B_hi + B_lo with round-to-nearest tf32 parts; T_lo B_lo, 2^-22 relative, is dropped):
// fp32-level accuracy at a small multiple of the tf32 rate, so the pass is bound by streaming the grid block, not by FMAs
// (the fp32 CUDA-core version of this kernel took 249 us per pass at G = 100, M = 10^6: 13 TFLOP/s).  Warp-level
// mma.sync.m16n8k8 is the right tool for these skinny products (M = G <= 128 rows, one 64-column slab per CTA step): there is
// no accumulator reuse across slabs for an asynchronous wgmma pipeline to amortise.
constexpr int SKI_MT = 64;          // slab width (positions)
constexpr int SKI_BP = SKI_MT + 8;  // pitch of the staged slab: 72 = 8 mod 32 -> conflict-free B fragments
__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// shared memory: T [GM][TPITCH] fp32 (rows and columns padded with zeros to GM = 16 ceil(G/16), GK = 8 ceil(G/8); TPITCH = GK + 4
// = 12 mod 32 for G = 100: conflict-free A fragments; split into hi / lo when a fragment is loaded), the staged slab as
// B_hi / B_lo [GK][SKI_BP] (split once while staging: seven warps read every value)
__global__ void __launch_bounds__(256)
ski_mode_kernel(const float* __restrict__ T, int G, const float* __restrict__ in, float* __restrict__ out, int64_t inner, int64_t total,
                int64_t nslab) {
  extern __shared__ __align__(16) float smm[];
  const int GM = (G + 15) & ~15, GK = (G + 7) & ~7, TP_ = GK + 4;
  float* Ts = smm;                                                         // [GM][TP_]
  uint32_t* Bh = reinterpret_cast<uint32_t*>(Ts + (size_t)GM * TP_);        // [GK][SKI_BP]
  uint32_t* Bl = Bh + (size_t)GK * SKI_BP;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int r = warp; r < GM; r += 8)
    for (int c = lane; c < TP_; c += 32) Ts[r * TP_ + c] = (r < G && c < G) ? T[r * G + c] : 0.f;
  const int gr = lane >> 2, gc = lane & 3;      // fragment coordinates
  const int nmt = GM / 16, nks = GK / 8;
  const uint32_t inner32 = (uint32_t)inner, total32 = (uint32_t)total;   // the host checks total < 2^31
  const int j4 = tid & 15, kst = tid >> 4;       // staging: this thread's float4 column of the slab, first k row
  for (int64_t slab = blockIdx.x; slab < nslab; slab += gridDim.x) {
    // slab -> 64 consecutive positions q = o * inner + x of the flattened (outer, inner) space, q < total = outer * inner
    const uint32_t q0 = (uint32_t)slab * SKI_MT;
    __syncthreads();
    {
      // 4 consecutive positions share o (inner is a multiple of 16): one division per thread and slab, then a constant stride per k
      const uint32_t q = q0 + (uint32_t)j4 * 4;
      const bool live = q < total32;
      const uint32_t o = live ? q / inner32 : 0u, x = live ? q - o * inner32 : 0u;
      const float* src = in + ((size_t)o * G) * inner + x;
      for (int k = kst; k < GK; k += 16) {
        float4 v = make_float4(0, 0, 0, 0);
        if (live && k < G) v = *reinterpret_cast<const float4*>(src + (size_t)k * inner);
        uint4 h, l;
        h.x = tf32_rna(v.x); h.y = tf32_rna(v.y); h.z = tf32_rna(v.z); h.w = tf32_rna(v.w);
        l.x = tf32_rna(v.x - __uint_as_float(h.x)); l.y = tf32_rna(v.y - __uint_as_float(h.y));
        l.z = tf32_rna(v.z - __uint_as_float(h.z)); l.w = tf32_rna(v.w - __uint_as_float(h.w));
        *reinterpret_cast<uint4*>(&Bh[k * SKI_BP + j4 * 4]) = h;
        *reinterpret_cast<uint4*>(&Bl[k * SKI_BP + j4 * 4]) = l;
      }
    }
    __syncthreads();
    // warp tile: 2 row tiles (32 output rows) x 4 column tiles (32 positions): every B fragment feeds two row tiles, every A
    // fragment four column tiles (one row tile x 8 column tiles per warp needed 1.5 shared-memory loads per MMA)
    const int nh = warp & 1;                       // which half of the slab's 64 positions
    for (int mp = warp >> 1; 2 * mp < nmt; mp += 4) {
      const bool two = 2 * mp + 1 < nmt;
      float acc[2][4][4];
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[m][nt][j] = 0.f;
      const float* tp = Ts + (size_t)(mp * 32 + gr) * TP_ + gc;
      for (int ks = 0; ks < nks; ++ks) {
        const int k0 = ks * 8;
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const float* t2 = tp + (size_t)(two ? m : 0) * 16 * TP_;      // a missing second row tile re-reads the first (discarded)
          const float a[4] = {t2[k0], t2[k0 + 8 * TP_], t2[k0 + 4], t2[k0 + 8 * TP_ + 4]};
#pragma unroll
          for (int j = 0; j < 4; ++j) { ah[m][j] = tf32_rna(a[j]); al[m][j] = tf32_rna(a[j] - __uint_as_float(ah[m][j])); }
        }
        const uint32_t* bh = Bh + (size_t)(k0 + gc) * SKI_BP + nh * 32 + gr;
        const uint32_t* bl = Bl + (size_t)(k0 + gc) * SKI_BP + nh * 32 + gr;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const uint32_t bh0 = bh[nt * 8], bh1 = bh[nt * 8 + 4 * SKI_BP], bl0 = bl[nt * 8], bl1 = bl[nt * 8 + 4 * SKI_BP];
#pragma unroll
          for (int m = 0; m < 2; ++m) {
            mma_tf32_16x8x8(acc[m][nt], al[m], bh0, bh1);   // small terms first
            mma_tf32_16x8x8(acc[m][nt], ah[m], bl0, bl1);
            mma_tf32_16x8x8(acc[m][nt], ah[m], bh0, bh1);
          }
        }
      }
      // C fragment: (row gr, cols 2 gc, 2 gc + 1) and (row gr + 8, same cols) of every 8-column tile
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        if (m == 1 && !two) break;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const uint32_t q = q0 + (uint32_t)(nh * 32 + nt * 8 + 2 * gc);
          if (q < total32) {
            const uint32_t o = q / inner32, x = q - o * inner32;
            const int r0 = mp * 32 + m * 16 + gr;
            float* dst = out + ((size_t)o * G + r0) * inner + x;
            if (r0 < G) *reinterpret_cast<float2*>(dst) = make_float2(acc[m][nt][0], acc[m][nt][1]);
            if (r0 + 8 < G) *reinterpret_cast<float2*>(dst + 8 * (size_t)inner) = make_float2(acc[m][nt][2], acc[m][nt][3]);
          }
        }
      }
    }
  }
}

// Mode product for G > 128 (ski_mode_kernel stages the whole G x G factor, which stops fitting in shared memory there), same
// contract and the same 3xTF32 split on mma.sync.m16n8k8.  T is Toeplitz, T[i][k] = t[|i - k|], and is never stored: a work item
// is (64-position slab, block of SKI_BR output rows), and it loops over the k rows of the mode in chunks of SKI_KC.  Per chunk the
// CTA stages the slab's SKI_KC input rows (split into tf32 hi / lo, as the dense kernel) and the generating window
// w[e] = t[|r0 - k0 - (SKI_KC - 1) + e|], e < SKI_BR + SKI_KC - 1, that holds every entry of the (rows, chunk) tile:
// T[r0 + a][k0 + c] = w[a - c + SKI_KC - 1].  Shared memory is 20 KB whatever G.  Chunks where the tile's entries are all exactly
// 0.0f are skipped: entries at |i - k| >= band are zero (ski_toeplitz_col_kernel writes band on the device), so only chunks that
// meet [r0 - band + 1, r1 + band - 1) run, and a product costs O(G band) per position instead of O(G^2).  Dropping exact zeros
// changes only which zero terms enter the fp32 accumulation.  The next chunk's input rows are loaded into registers while the
// tensor cores work on the current one.
constexpr int SKI_BR = 128;                 // output rows per work item: 4 warp pairs x 32 rows
constexpr int SKI_KC = 32;                  // k rows per chunk: 4 k-steps of 8
constexpr int SKI_WIN = SKI_BR + SKI_KC;    // staged generating window (SKI_BR + SKI_KC - 1 entries used)
__global__ void __launch_bounds__(256, 2)
ski_mode_banded_kernel(const float* __restrict__ t, const int* __restrict__ band, int G, const float* __restrict__ in,
                       float* __restrict__ out, int64_t inner, int64_t total, int64_t nslab) {
  __shared__ __align__(16) uint32_t Bh[SKI_KC * SKI_BP];
  __shared__ __align__(16) uint32_t Bl[SKI_KC * SKI_BP];
  __shared__ uint32_t Wh[SKI_WIN], Wl[SKI_WIN];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gr = lane >> 2, gc = lane & 3;      // fragment coordinates
  const int nh = warp & 1, mp = warp >> 1;      // warp tile: half nh of the slab's 64 positions, rows mp * 32 .. + 32 of the block
  const int j4 = tid & 15, kst = tid >> 4;      // staging: this thread's float4 column of the slab, k rows kst and kst + 16
  const uint32_t inner32 = (uint32_t)inner, total32 = (uint32_t)total;   // the host checks total < 2^31
  const int bw = *band;
  const int nrb = (G + SKI_BR - 1) / SKI_BR;
  for (int64_t wk = blockIdx.x; wk < nslab * nrb; wk += gridDim.x) {
    const int64_t slab = wk / nrb;               // the row blocks of one slab are neighbours: they share input rows in L2
    const int r0 = (int)(wk - slab * nrb) * SKI_BR;
    const int r1 = min(G, r0 + SKI_BR);
    const uint32_t q0 = (uint32_t)slab * SKI_MT;
    const int klo = max(0, r0 - bw + 1), khi = bw > 0 ? min(G, r1 + bw - 1) : 0;   // empty when t is all zero
    // 4 consecutive positions share o (inner is a multiple of 16): one division per thread and work item
    const uint32_t qs = q0 + (uint32_t)j4 * 4;
    const bool live = qs < total32;
    const uint32_t os = live ? qs / inner32 : 0u, xs = live ? qs - os * inner32 : 0u;
    const float* src = in + ((size_t)os * G) * inner + xs;
    auto load = [&](int k0, float4 (&v)[2]) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = k0 + kst + 16 * h;
        v[h] = (live && k < G) ? *reinterpret_cast<const float4*>(src + (size_t)k * inner) : make_float4(0, 0, 0, 0);
      }
    };
    // warp-uniform: this warp's positions or rows lie entirely outside the operand (d = 1 has 16 positions; the last row block)
    const bool work = q0 + (uint32_t)nh * 32 < total32 && r0 + mp * 32 < G;
    float acc[2][4][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[m][nt][j] = 0.f;
    const int kfirst = klo / SKI_KC * SKI_KC;
    float4 pf[2];
    if (kfirst < khi) load(kfirst, pf);
    for (int k0 = kfirst; k0 < khi; k0 += SKI_KC) {
      __syncthreads();                           // the previous chunk's fragments have been read
      for (int e = tid; e < SKI_WIN - 1; e += 256) {
        const int dl = abs(r0 - k0 - (SKI_KC - 1) + e);
        const float v = dl < G ? t[dl] : 0.f;    // dl >= G only pairs a padding row with a padding k (B rows k >= G are zero)
        const uint32_t h = tf32_rna(v);
        Wh[e] = h;
        Wl[e] = tf32_rna(v - __uint_as_float(h));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float4 v = pf[h];
        uint4 hi, lo;
        hi.x = tf32_rna(v.x); hi.y = tf32_rna(v.y); hi.z = tf32_rna(v.z); hi.w = tf32_rna(v.w);
        lo.x = tf32_rna(v.x - __uint_as_float(hi.x)); lo.y = tf32_rna(v.y - __uint_as_float(hi.y));
        lo.z = tf32_rna(v.z - __uint_as_float(hi.z)); lo.w = tf32_rna(v.w - __uint_as_float(hi.w));
        *reinterpret_cast<uint4*>(&Bh[(kst + 16 * h) * SKI_BP + j4 * 4]) = hi;
        *reinterpret_cast<uint4*>(&Bl[(kst + 16 * h) * SKI_BP + j4 * 4]) = lo;
      }
      __syncthreads();
      if (k0 + SKI_KC < khi) load(k0 + SKI_KC, pf);   // in flight during the MMAs below
      if (!work) continue;
#pragma unroll
      for (int ks = 0; ks < SKI_KC / 8; ++ks) {
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          // A fragment (rows gr, gr + 8; columns gc, gc + 4 of the 16 x 8 tile) from the window: lanes read 11 consecutive words
          const int e = mp * 32 + m * 16 + gr - ks * 8 - gc + SKI_KC - 1;
          const int ei[4] = {e, e + 8, e - 4, e + 4};
#pragma unroll
          for (int j = 0; j < 4; ++j) { ah[m][j] = Wh[ei[j]]; al[m][j] = Wl[ei[j]]; }
        }
        const uint32_t* bh = Bh + (size_t)(ks * 8 + gc) * SKI_BP + nh * 32 + gr;
        const uint32_t* bl = Bl + (size_t)(ks * 8 + gc) * SKI_BP + nh * 32 + gr;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          if (q0 + (uint32_t)(nh * 32 + nt * 8) < total32) {   // warp-uniform: position tiles past the operand are left out
            const uint32_t bh0 = bh[nt * 8], bh1 = bh[nt * 8 + 4 * SKI_BP], bl0 = bl[nt * 8], bl1 = bl[nt * 8 + 4 * SKI_BP];
#pragma unroll
            for (int m = 0; m < 2; ++m) {
              mma_tf32_16x8x8(acc[m][nt], al[m], bh0, bh1);   // small terms first
              mma_tf32_16x8x8(acc[m][nt], ah[m], bl0, bl1);
              mma_tf32_16x8x8(acc[m][nt], ah[m], bh0, bh1);
            }
          }
        }
      }
    }
    // every row of the block is written, those whose chunks were all skipped with 0
#pragma unroll
    for (int m = 0; m < 2; ++m) {
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const uint32_t q = q0 + (uint32_t)(nh * 32 + nt * 8 + 2 * gc);
        if (q < total32) {
          const uint32_t o = q / inner32, x = q - o * inner32;
          const int r = r0 + mp * 32 + m * 16 + gr;
          float* dst = out + ((size_t)o * G + r) * inner + x;
          if (r < G) *reinterpret_cast<float2*>(dst) = make_float2(acc[m][nt][0], acc[m][nt][1]);
          if (r + 8 < G) *reinterpret_cast<float2*>(dst + 8 * (size_t)inner) = make_float2(acc[m][nt][2], acc[m][nt][3]);
        }
      }
    }
  }
}

// T_i[a][b] = k_1d(|a - b| step_i / l_i): per-dimension factor of the grid covariance (grid_kernel.py:138-157 evaluates the base
// kernel on every dimension separately, last_dim_is_batch=True).  The dense factor (G <= 128, read by ski_mode_kernel) and the
// generating column (every G) evaluate this one expression, so t[k] == T[a][b] bit for bit for |a - b| = k.
__device__ __forceinline__ float ski_toeplitz_entry(int diff, float step, float inv_ls, int kind, int deriv) {
  const float r = fabsf((float)diff) * step * inv_ls;      // |dx| / l
  float v;
  if (kind == GP_RBF) {
    v = expf(-0.5f * r * r);
    if (deriv) v *= r * r;                                 // l dk/dl = r^2 k  (functions/rbf_covariance.py:20-29)
  } else {
    const float nu2 = (kind == GP_MATERN12) ? 1.f : (kind == GP_MATERN32 ? 3.f : 5.f);
    const float rho = sqrtf(nu2) * r;
    const float ex = expf(-rho);
    if (!deriv) v = (kind == GP_MATERN12) ? ex : (kind == GP_MATERN32 ? (1.f + rho) * ex : (1.f + rho + rho * rho * (1.f / 3.f)) * ex);
    else        v = (kind == GP_MATERN12) ? rho * ex : (kind == GP_MATERN32 ? rho * rho * ex : (1.f + rho) * rho * rho * (1.f / 3.f) * ex);
  }                                                        // l dk/dl = -rho dk/drho  (functions/matern_covariance.py:27-56)
  return v;
}

__global__ void ski_toeplitz_kernel(float* __restrict__ T, int G, float step, float inv_ls, int kind, int deriv) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= G * G) return;
  const int a = e / G, b = e % G;
  T[e] = ski_toeplitz_entry(a - b, step, inv_ls, kind, deriv);
}

// Generating columns t[k] = T[k][0] and dt[k] = l dT[k][0]/dl, k < G, and their band ends: band[0] = 1 + the last k with t[k] != 0
// (0 if none; a NaN counts as non-zero), band[1] the same for dt.  Every entry of T at |a - b| >= band[0] is exactly 0.0f, which
// is what lets ski_mode_banded_kernel skip its k-chunks.  band must be zero before the launch (atomicMax of a fixed set of
// values: the result does not depend on the order).
__global__ void __launch_bounds__(256)
ski_toeplitz_col_kernel(float* __restrict__ t, float* __restrict__ dt, int G, float step, float inv_ls, int kind, int* __restrict__ band) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  float v = 0.f, dv = 0.f;
  if (k < G) {
    v = ski_toeplitz_entry(k, step, inv_ls, kind, 0);
    dv = ski_toeplitz_entry(k, step, inv_ls, kind, 1);
    t[k] = v;
    dt[k] = dv;
  }
  const unsigned e0 = __reduce_max_sync(0xffffffffu, (k < G && !(v == 0.f)) ? (unsigned)k + 1u : 0u);
  const unsigned e1 = __reduce_max_sync(0xffffffffu, (k < G && !(dv == 0.f)) ? (unsigned)k + 1u : 0u);
  if ((threadIdx.x & 31) == 0) {
    if (e0) atomicMax(band, (int)e0);
    if (e1) atomicMax(band + 1, (int)e1);
  }
}

// <a, b> over n floats -> one fp64 partial per CTA (fixed order inside the CTA and on the host: reproducible)
__global__ void __launch_bounds__(256) ski_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n4,
                                                      double* __restrict__ part) {
  __shared__ double sh[256];
  double acc = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (int64_t)gridDim.x * 256) {
    const float4 x = reinterpret_cast<const float4*>(a)[i], y = reinterpret_cast<const float4*>(b)[i];
    acc += (double)x.x * y.x + (double)x.y * y.y + (double)x.z * y.z + (double)x.w * y.w;
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}

static size_t ski_mode_smem(int G) {
  const size_t GM = (G + 15) & ~15, GK = (G + 7) & ~7;
  return sizeof(float) * (GM * (GK + 4) + 2 * GK * SKI_BP);
}

// fn(std::integral_constant<int, D>()) for D = d: the passes are compiled once per dimension 1 .. SKI_MAXD
template <typename F>
static int ski_with_d(int d, F&& fn) {
  switch (d) {
    case 1: return fn(std::integral_constant<int, 1>());
    case 2: return fn(std::integral_constant<int, 2>());
    case 3: return fn(std::integral_constant<int, 3>());
    case 4: return fn(std::integral_constant<int, 4>());
  }
  set_error("SKI backend supports 1 <= d <= 4 (d=%d)", d);
  return GP_E_SHAPE;
}

static SkiGeom ski_geom(const gp_ski_state* s, int d) {
  SkiGeom g;
  g.d = d;
  g.M = 1;
  for (int i = d - 1; i >= 0; --i) { g.G[i] = s->G[i]; g.lo[i] = s->lo[i]; g.step[i] = s->step[i]; g.stride[i] = g.M; g.M *= s->G[i]; }
  return g;
}

static SkiTiles ski_tiles_of(const gp_ski_state* s, int d) {
  SkiTiles tl;
  tl.ntiles = s->ntiles;
  for (int i = 0; i < SKI_MAXD; ++i) { tl.E[i] = i < d ? s->tile_edge[i] : 1; tl.nt[i] = i < d ? s->tile_num[i] : 1; }
  return tl;
}

// bucket the points by tile (counting sort on the device): once per data update
static int ski_bucket_points(gp_plan* p, const SkiGeom& g) {
  gp_ski_state* s = p->ski;
  cudaStream_t st = p->stream;
  const int d = g.d;
  const int64_t n = p->n1;
  GP_REQUIRE(n < ((int64_t)1 << 31), GP_E_SHAPE, "SKI: n too large");
  // (E + 3)^d nodes x 64 B of shared memory per CTA: 4 / 23 / 22 / 40 KB -> 5 to 8 CTAs per SM hide the dependent
  // shared-memory read-modify-write chain of the scatter and the per-point loads (E = 8 at d = 3 -- 85 KB, 2 CTAs per SM -- was 3x slower)
  static const int edge_by_d[SKI_MAXD + 1] = {0, 64, 16, 4, 2};
  int64_t nt = 1;
  for (int i = 0; i < d; ++i) {
    s->tile_edge[i] = edge_by_d[d];
    s->tile_num[i] = std::max(1, (int)cdiv(g.G[i] - 3, s->tile_edge[i]));
    nt *= s->tile_num[i];
  }
  GP_REQUIRE(nt <= (1 << 20), GP_E_SHAPE, "SKI: %lld point tiles (grid too fine for d=%d)", (long long)nt, d);
  s->ntiles = (int)nt;
  const SkiTiles tl = ski_tiles_of(s, d);
  GP_CHECK(s->tile_cnt.ensure(sizeof(int) * nt));
  GP_CHECK(s->tile_off.ensure(sizeof(int) * (nt + 1)));
  GP_CHECK(s->perm.ensure(sizeof(int) * n));
  GP_CHECK(s->first_s.ensure(sizeof(int) * n * d));
  GP_CHECK(s->wts_s.ensure(sizeof(float) * n * d * 4));
  GP_CUDA(cudaMemsetAsync(s->tile_cnt.p, 0, sizeof(int) * nt, st));
  const unsigned gb = (unsigned)cdiv(n, 256);
  int* cnt = s->tile_cnt.as<int>();
  int* off = s->tile_off.as<int>();
  GP_CHECK(ski_with_d(d, [&](auto D) {
    ski_tile_count_kernel<D><<<gb, 256, 0, st>>>(s->first.as<int>(), n, tl, cnt);
    ski_tile_scan_kernel<<<1, 1024, 0, st>>>(cnt, (int)nt, off);
    ski_tile_fill_kernel<D><<<gb, 256, 0, st>>>(s->first.as<int>(), s->wts.as<float>(), n, tl, off, cnt, s->perm.as<int>(),
                                                s->first_s.as<int>(), s->wts_s.as<float>());
    return GP_OK;
  }));
  p->launches += 3;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

constexpr int SKI_TILE_SMEM = 96 * 1024;   // dynamic shared memory the tiled kernels opt in to
constexpr int SKI_IP_CW = 32;              // columns per chunk of the interpolation and input-gradient passes

// Launch shape of the tiled passes (scatter, gather, interpolation, input gradient): one CTA per (tile, part) work item, parts =
// CTAs per tile at ~256 points each on average (no host read-back of the real counts: the split only balances load), at most 16
// CTAs per SM striding over the work items; a CTA stages the nodes of its tile's block in shared memory.
struct SkiPass {
  SkiGeom g;
  SkiTiles tl;
  int parts;
  unsigned grid;
  size_t nodes;   // nodes of the largest tile block
};
template <int D>
static int ski_tiled_pass(gp_plan* p, SkiPass* ps) {
  const gp_ski_state* s = p->ski;
  ps->g = ski_geom(s, D);
  ps->tl = ski_tiles_of(s, D);
  const int64_t avg = p->n1 / std::max(1, s->ntiles);
  ps->parts = (int)std::min<int64_t>(1024, std::max<int64_t>(1, cdiv(avg, 256)));
  ps->grid = (unsigned)std::min<int64_t>((int64_t)ps->tl.ntiles * ps->parts, 16 * (int64_t)p->n_sm);
  ps->nodes = 1;
  for (int i = 0; i < D; ++i) ps->nodes *= (size_t)std::min(s->tile_edge[i] + 3, s->G[i]);
  // the widest staging: SKI_IP_CW floats per node (the scatter and gather stage TP)
  GP_REQUIRE(ps->nodes * SKI_IP_CW * sizeof(float) <= (size_t)SKI_TILE_SMEM, GP_E_SHAPE,
             "SKI: tile block of %zu nodes does not fit in shared memory", ps->nodes);
  // the interpolation and input-gradient kernels (below) opt in where they are launched
  GP_CHECK(opt_in_smem<ski_scatter_tiled_kernel<D>>(p->device, SKI_TILE_SMEM));
  GP_CHECK(opt_in_smem<ski_gather_tiled_kernel<D>>(p->device, SKI_TILE_SMEM));
  return GP_OK;
}

int ski_pack(gp_plan* p) {
  gp_ski_state* s = p->ski;
  GP_REQUIRE(s != nullptr, GP_E_STATE, "SKI grid not set");
  GP_REQUIRE(p->same && p->row_begin == 0 && p->row_count == p->n1, GP_E_SHAPE, "the SKI backend needs a square, unsharded operator");
  cudaStream_t st = p->stream;
  const int d = p->d;
  const int64_t n = p->n1;
  const SkiGeom g = ski_geom(s, d);
  s->M = g.M;
  GP_CHECK(s->first.ensure(sizeof(int) * n * d));
  GP_CHECK(s->wts.ensure(sizeof(float) * n * d * 4));
  GP_CHECK(s->gridA.ensure(sizeof(float) * g.M * TP));
  GP_CHECK(s->gridB.ensure(sizeof(float) * g.M * TP));
  GP_CHECK(s->flag.ensure(64));
  GP_CHECK(p->mean.ensure(sizeof(float) * (d + 4)));
  p->xbad = reinterpret_cast<int*>(p->mean.as<float>() + d);
  GP_CUDA(cudaMemsetAsync(p->xbad, 0, sizeof(int), st));
  GP_CUDA(cudaMemsetAsync(s->flag.p, 0, sizeof(int), st));
  ski_interp_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(p->X1, n, p->ld1, g, s->first.as<int>(), s->wts.as<float>(), s->flag.as<int>());
  p->launches++;
  GP_CHECK(ski_bucket_points(p, g));
  // dense factors for the dimensions ski_mode_kernel runs (G <= SKI_DENSE_G), generating columns and band ends for every dimension
  size_t toff = 0, coff = 0;
  for (int i = 0; i < d; ++i) {
    if (s->G[i] <= SKI_DENSE_G) toff += (size_t)s->G[i] * s->G[i];
    coff += (size_t)s->G[i];
  }
  GP_CHECK(s->T.ensure(sizeof(float) * toff));
  GP_CHECK(s->dT.ensure(sizeof(float) * toff));   // l_i dT_i/dl_i: the factors of the hyper-parameter gradients
  GP_CHECK(s->tcol.ensure(sizeof(float) * coff));
  GP_CHECK(s->dtcol.ensure(sizeof(float) * coff));
  GP_CHECK(s->band.ensure(sizeof(int) * 2 * SKI_MAXD));
  GP_CUDA(cudaMemsetAsync(s->band.p, 0, sizeof(int) * 2 * SKI_MAXD, st));
  toff = 0;
  coff = 0;
  for (int i = 0; i < d; ++i) {
    const float l = (p->ls.size() == 1) ? p->ls[0] : p->ls[i];
    if (s->G[i] <= SKI_DENSE_G) {
      ski_toeplitz_kernel<<<(unsigned)cdiv((int64_t)s->G[i] * s->G[i], 256), 256, 0, st>>>(s->T.as<float>() + toff, s->G[i], s->step[i], 1.f / l, p->kind, 0);
      ski_toeplitz_kernel<<<(unsigned)cdiv((int64_t)s->G[i] * s->G[i], 256), 256, 0, st>>>(s->dT.as<float>() + toff, s->G[i], s->step[i], 1.f / l, p->kind, 1);
      p->launches += 2;
      toff += (size_t)s->G[i] * s->G[i];
    }
    ski_toeplitz_col_kernel<<<(unsigned)cdiv(s->G[i], 256), 256, 0, st>>>(s->tcol.as<float>() + coff, s->dtcol.as<float>() + coff, s->G[i],
                                                                         s->step[i], 1.f / l, p->kind, s->band.as<int>() + 2 * i);
    p->launches++;
    coff += (size_t)s->G[i];
  }
  int h_oob = 0;
  GP_CUDA(cudaMemcpyAsync(&h_oob, s->flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  GP_CUDA(cudaStreamSynchronize(st));
  GP_REQUIRE(!h_oob, GP_E_SHAPE, "Received data that was out of bounds for the specified grid.");
  // geometry of the K.V partial block: one "split", rows padded like the dense backends
  p->nsplit = 1;
  p->nparts = 1;
  p->rows_pad = cdiv(p->row_count, 2 * TILE_I) * 2 * TILE_I;
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// d mode products  *out = (F_0 x ... x F_{d-1}) in,  F_i = dT_i for i == dt_dim and T_i otherwise (dt_dim = -1: K_uu).  Product i
// writes bufs[i & 1]; `in` may be buf1 (overwritten after the first product), and *out is the buffer of the last product.
// A dimension with G <= SKI_DENSE_G runs ski_mode_kernel on its dense factor, a larger one ski_mode_banded_kernel on its
// generating column.
static int ski_mode_products(gp_plan* p, const SkiGeom& g, const float* in, float* buf0, float* buf1, int dt_dim, float** out) {
  const gp_ski_state* s = p->ski;
  GP_CHECK(opt_in_smem<ski_mode_kernel>(p->device, 160 * 1024));
  float* bufs[2] = {buf0, buf1};
  const float* cur = in;
  size_t toff = 0, coff = 0;
  for (int i = 0; i < g.d; ++i) {
    const int G = g.G[i];
    const int64_t inner = g.stride[i] * TP;                // elements after mode i (incl. the 16 columns)
    const int64_t total = g.M / G * TP;                    // positions of the flattened (outer, inner) space
    const int64_t nslab = cdiv(total, SKI_MT);
    GP_REQUIRE(total < ((int64_t)1 << 31), GP_E_SHAPE, "SKI: grid block too large");
    if (G <= SKI_DENSE_G) {
      const float* F = (i == dt_dim ? s->dT : s->T).as<float>() + toff;
      ski_mode_kernel<<<(unsigned)std::min<int64_t>(nslab, 2 * p->n_sm), 256, ski_mode_smem(G), p->stream>>>(F, G, cur, bufs[i & 1], inner, total, nslab);
      toff += (size_t)G * G;
    } else {
      const float* F = (i == dt_dim ? s->dtcol : s->tcol).as<float>() + coff;
      const int* band = s->band.as<int>() + 2 * i + (i == dt_dim ? 1 : 0);
      const int64_t items = nslab * cdiv(G, SKI_BR);
      ski_mode_banded_kernel<<<(unsigned)std::min<int64_t>(items, 4 * p->n_sm), 256, 0, p->stream>>>(F, band, G, cur, bufs[i & 1], inner, total, nslab);
    }
    cur = bufs[i & 1];
    coff += (size_t)G;
  }
  p->launches += g.d;
  *out = bufs[(g.d - 1) & 1];
  return GP_OK;
}

// scatter + d mode products: *grid_out = (T_0 x ... x T_{d-1}) W^T V16, a [M][16] block (gridA or gridB)
template <int D>
static int ski_grid_apply(gp_plan* p, const SkiPass& ps, const float* V16, float** grid_out) {
  gp_ski_state* s = p->ski;
  float* A = s->gridA.as<float>();
  GP_CUDA(cudaMemsetAsync(A, 0, sizeof(float) * ps.g.M * TP, p->stream));
  ski_scatter_tiled_kernel<D><<<ps.grid, SKI_SC_THREADS, ps.nodes * TP * sizeof(float), p->stream>>>(
      s->first_s.as<int>(), s->wts_s.as<float>(), s->perm.as<int>(), s->tile_off.as<int>(), ps.g, ps.tl, ps.parts, V16, A);
  p->launches++;
  GP_CHECK(ski_mode_products(p, ps.g, A, s->gridB.as<float>(), A, -1, grid_out));
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

template <int D>
static int ski_matmul_d(gp_plan* p, const float* V16, float* OUT16) {
  gp_ski_state* s = p->ski;
  SkiPass ps;
  GP_CHECK(ski_tiled_pass<D>(p, &ps));
  float* cur = nullptr;
  GP_CHECK(ski_grid_apply<D>(p, ps, V16, &cur));
  ski_gather_tiled_kernel<D><<<ps.grid, 256, ps.nodes * TP * sizeof(float), p->stream>>>(
      s->first_s.as<int>(), s->wts_s.as<float>(), s->perm.as<int>(), s->tile_off.as<int>(), ps.g, ps.tl, ps.parts, cur, OUT16);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// Bilinear derivative of the interpolated operator (the reference reaches it through InterpolatedLinearOperator._bilinear_derivative
// -> the grid kernel's Toeplitz columns -> autograd, kernels/grid_kernel.py:138-177):
//   sum_ij (L_i . R_j) d(K_ski)_ij / d theta = < A, dK_uu/d theta B >,   A = W^T L, B = W^T R   (grid blocks [M][16]),
//   dK_uu / d l_i = (1 / l_i) T_0 x ... x (l_i dT_i/dl_i) x ... x T_{d-1}.
// total[0] += <A, K_uu B> (d/d outputscale), total[1 + i] += <A, (.. dT_i ..) B>: d + 1 sweeps of d mode products each.
template <int D>
static int ski_bilinear_d(gp_plan* p, const float* L16, const float* R16, double* total) {
  gp_ski_state* s = p->ski;
  cudaStream_t st = p->stream;
  constexpr int DOT_BLOCKS = 296;
  SkiPass ps;
  GP_CHECK(ski_tiled_pass<D>(p, &ps));
  const SkiGeom& g = ps.g;
  const size_t tsm = ps.nodes * TP * sizeof(float);
  GP_CHECK(s->gridC.ensure(sizeof(float) * g.M * TP));
  GP_CHECK(s->gridD.ensure(sizeof(float) * g.M * TP));
  GP_CHECK(p->misc.ensure(sizeof(double) * DOT_BLOCKS * (D + 1)));
  float* A = s->gridC.as<float>();
  float* B = s->gridD.as<float>();
  double* part = p->misc.as<double>();
  GP_CUDA(cudaMemsetAsync(A, 0, sizeof(float) * g.M * TP, st));
  GP_CUDA(cudaMemsetAsync(B, 0, sizeof(float) * g.M * TP, st));
  ski_scatter_tiled_kernel<D><<<ps.grid, SKI_SC_THREADS, tsm, st>>>(s->first_s.as<int>(), s->wts_s.as<float>(), s->perm.as<int>(), s->tile_off.as<int>(), g, ps.tl, ps.parts, L16, A);
  ski_scatter_tiled_kernel<D><<<ps.grid, SKI_SC_THREADS, tsm, st>>>(s->first_s.as<int>(), s->wts_s.as<float>(), s->perm.as<int>(), s->tile_off.as<int>(), g, ps.tl, ps.parts, R16, B);
  p->launches += 2;
  for (int term = 0; term <= D; ++term) {          // term 0: K_uu ; term 1 + i: derivative factor in dimension i
    float* cur = nullptr;
    GP_CHECK(ski_mode_products(p, g, B, s->gridA.as<float>(), s->gridB.as<float>(), term - 1, &cur));
    ski_dot_kernel<<<DOT_BLOCKS, 256, 0, st>>>(A, cur, g.M * TP / 4, part + (size_t)term * DOT_BLOCKS);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  std::vector<double> h((size_t)DOT_BLOCKS * (D + 1));
  GP_CUDA(cudaMemcpyAsync(h.data(), part, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, st));
  GP_CUDA(cudaStreamSynchronize(st));
  for (int term = 0; term <= D; ++term) {
    double acc = 0.0;
    for (int b = 0; b < DOT_BLOCKS; ++b) acc += h[(size_t)term * DOT_BLOCKS + b];
    total[term] += acc;
  }
  return GP_OK;
}

int ski_bilinear(gp_plan* p, const float* L16, const float* R16, double* total) {
  return ski_with_d(p->d, [&](auto D) { return ski_bilinear_d<D>(p, L16, R16, total); });
}

// partial[0][r][:] = (W K_uu W^T V16)[r][:]   (outputscale / noise are applied by the finish kernels)
int ski_kmv_partials(gp_plan* p, const float* V16, const int* done_flag) {
  (void)done_flag;   // the products of a finished mBCG are cheap no-ops for the dense kernels; here they simply run
  return ski_with_d(p->d, [&](auto D) { return ski_matmul_d<D>(p, V16, p->partial.as<float>()); });
}

// ---- single entries (ski_rows.cuh): the diagonal, requested rows and the pivoted Cholesky (pivchol.cu) ----------------------------
int ski_rows_args(const gp_plan* p, SkiRows* s) {
  const gp_ski_state* k = p->ski;
  GP_REQUIRE(k != nullptr && k->tcol.p != nullptr, GP_E_STATE, "SKI grid not packed");
  s->d = p->d;
  int off = 0;
  for (int i = 0; i < 4; ++i) {
    const bool live = i < p->d;
    s->G[i] = live ? k->G[i] : 0;
    s->coff[i] = off;
    s->uoff[i] = off;
    if (live) off += k->G[i];
  }
  s->usum = off;
  s->staged = off <= SKI_U_MAX;
  s->os = p->outputscale;
  s->tc = k->tcol.as<float>();
  s->first = k->first.as<int>();
  s->wts = k->wts.as<float>();
  return GP_OK;
}

__global__ void ski_kdiag_kernel(const SkiRows s, int64_t n, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ski_diag_entry(s, i);
}

// OUT[r][j] = K_ski(idx[r], j): blockIdx.y = r, u of row idx[r] staged by every CTA of the row
__global__ void __launch_bounds__(256)
ski_krows_kernel(const SkiRows s, const int64_t* __restrict__ idx, int64_t n, float* __restrict__ out, int64_t ldo) {
  __shared__ float u[SKI_U_MAX];
  const int64_t i = idx[blockIdx.y];
  if (i < 0 || i >= n) {   // out-of-range row index (CTA-uniform): NaN row, as the dense row extraction, instead of an out-of-bounds read
    const int64_t jj = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (jj < n) out[(int64_t)blockIdx.y * ldo + jj] = __int_as_float(0x7fc00000);
    return;
  }
  ski_stage_u(s, i, u, threadIdx.x, 256);
  __syncthreads();
  const int64_t j = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (j < n) out[(int64_t)blockIdx.y * ldo + j] = ski_entry(s, u, i, j);
}

// per-CTA fp64 partial sums of the diagonal (fixed order in the CTA and on the host: reproducible)
__global__ void __launch_bounds__(256) ski_diag_sum_kernel(const SkiRows s, int64_t n, double* __restrict__ part) {
  __shared__ double sh[256];
  double acc = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) acc += (double)ski_diag_entry(s, i);
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}

int ski_kdiag(gp_plan* p, float* OUT) {
  SkiRows s;
  GP_CHECK(ski_rows_args(p, &s));
  ski_kdiag_kernel<<<(unsigned)cdiv(p->n1, 256), 256, 0, p->stream>>>(s, p->n1, OUT);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int ski_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "SKI row extraction takes at most 65535 rows per call (got %lld)", (long long)m);
  SkiRows s;
  GP_CHECK(ski_rows_args(p, &s));
  ski_krows_kernel<<<dim3((unsigned)cdiv(p->n1, 256), (unsigned)m), 256, 0, p->stream>>>(s, idx, p->n1, OUT, ldo);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int ski_diag_sum(gp_plan* p, double* out) {
  SkiRows s;
  GP_CHECK(ski_rows_args(p, &s));
  const int gs = (int)std::max<int64_t>(1, std::min<int64_t>(cdiv(p->n1, 256), 2 * (int64_t)p->n_sm));
  GP_CHECK(p->misc.ensure(sizeof(double) * gs));
  ski_diag_sum_kernel<<<gs, 256, 0, p->stream>>>(s, p->n1, p->misc.as<double>());
  p->launches++;
  GP_CUDA(cudaGetLastError());
  std::vector<double> h(gs);
  GP_CUDA(cudaMemcpyAsync(h.data(), p->misc.p, sizeof(double) * gs, cudaMemcpyDeviceToHost, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));
  double acc = 0.0;
  for (int b = 0; b < gs; ++b) acc += h[b];
  *out = acc;
  return GP_OK;
}

// ---- prediction on the grid (gp_ski_grid_matmul / gp_ski_interp_matmul) ----------------------------------------------------------
// The reference's InterpolatedPredictionStrategy (models/exact_prediction_strategies.py:481-827) keeps its mean and LOVE caches on
// the grid, c = s K_uu W^T alpha and C = s K_uu W^T R, and predicts with one interpolation W* c / W* C per call: O(4^d t) per test
// point, independent of the training-set size.

// OUT[r][c] = s U[r][c] for c < tc: the [M][16] grid block of one column chunk into the caller's [M][ldo] matrix
__global__ void ski_grid_export_kernel(const float* __restrict__ U, int64_t M, int tc, float s, float* __restrict__ out, int64_t ldo) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M * tc) return;
  const int64_t r = e / tc;
  const int c = (int)(e - r * tc);
  out[r * ldo + c] = s * U[r * TP + c];
}

// OUT[:, 0:tc] = s K_uu W^T V[:, 0:tc] for one chunk of tc <= 16 columns (staged in p->V16), OUT a [M][ldo] grid matrix
template <int D>
static int ski_grid_block(gp_plan* p, const SkiPass& ps, const float* V, int64_t ldv, int tc, float* OUT, int64_t ldo) {
  float* cur = nullptr;
  GP_CHECK(to_v16(p, V, ldv, tc, p->n1, p->V16.as<float>()));
  GP_CHECK(ski_grid_apply<D>(p, ps, p->V16.as<float>(), &cur));
  ski_grid_export_kernel<<<(unsigned)cdiv(ps.g.M * tc, 256), 256, 0, p->stream>>>(cur, ps.g.M, tc, p->outputscale, OUT, ldo);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// sum_q w_q C[node_q] for one point and column in the fixed separable order  sum_a w_0[a] (sum_b w_1[b] (... C[...])):
// b points at the point's first node, pitch[k] is the distance of neighbouring nodes of dimension k (in floats)
template <int D, int K>
struct SkiInterpSum {
  static __device__ __forceinline__ float run(const float* b, const float4 (&w)[D], const int (&pitch)[D]) {
    float s = w[K].x * SkiInterpSum<D, K + 1>::run(b, w, pitch);
    s = fmaf(w[K].y, SkiInterpSum<D, K + 1>::run(b + pitch[K], w, pitch), s);
    s = fmaf(w[K].z, SkiInterpSum<D, K + 1>::run(b + 2 * pitch[K], w, pitch), s);
    s = fmaf(w[K].w, SkiInterpSum<D, K + 1>::run(b + 3 * pitch[K], w, pitch), s);
    return s;
  }
};
template <int D>
struct SkiInterpSum<D, D> {
  static __device__ __forceinline__ float run(const float* b, const float4 (&)[D], const int (&)[D]) { return *b; }
};

// OUT[perm[p]][c] = sum_q w_q C[node_q][c] for the tc <= 32 columns of one chunk (C and OUT offset to the chunk by the caller).
// One CTA per (tile, part), as the gather: the tile's (E + 3)^D node block of the chunk is staged in shared memory as [node][LP],
// LP = tc rounded up to a power of two (44 KB at d = 3, LP = 32), then every lane owns one (point, column) pair: LP lanes per point
// read consecutive columns of a node, 32 / LP points per warp -- so a single column (the mean) keeps all 32 lanes busy on 32
// points.  The point's 4 D weights sit in registers; no atomics and no cross-lane sums, so repeated calls are bit-identical
// whatever ldc / ldo.  Staged with float4 loads when the chunk is full and 16-byte aligned (vec).
constexpr int SKI_IP_THREADS = 256;
template <int D>
__global__ void __launch_bounds__(SKI_IP_THREADS)
ski_interp_tiled_kernel(const int* __restrict__ first_s, const float* __restrict__ wts_s, const int* __restrict__ perm,
                        const int* __restrict__ off, SkiGeom g, SkiTiles tl, int parts, const float* __restrict__ C, int64_t ldc,
                        int tc, int lp_log2, int vec, float* __restrict__ out, int64_t ldo) {
  extern __shared__ __align__(16) float blk[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int col = lane & ((1 << lp_log2) - 1);
  const int slot = (tid >> lp_log2);                    // this lane's point slot in the CTA
  const int nslot = SKI_IP_THREADS >> lp_log2;
  const int gshift = vec ? lp_log2 - 2 : lp_log2;        // log2 of the staged column groups per node (float4 or float)
  for (int64_t wk = blockIdx.x; wk < (int64_t)tl.ntiles * parts; wk += gridDim.x) {
    int tile, p0, p1;
    if (!ski_work_range(wk, parts, off, tile, p0, p1)) continue;
    const SkiBlock<D> b = ski_block_of<D>(tile, g, tl);
    __syncthreads();
    // staging, row by row as ski_block_rows: the lanes cover (last-dimension node, column group) pairs of a row
    const int last = b.ext[D - 1];
    const int nrows = b.nodes / last;
    for (int row = warp; row < nrows; row += SKI_IP_THREADS / 32) {
      const auto [node0, idx0] = ski_row_origin<D>(b, g, row);
      for (int e = lane; e < (last << gshift); e += 32) {
        const int c = e >> gshift, q = e & ((1 << gshift) - 1);
        const float* src = C + (idx0 + (int64_t)c * g.stride[D - 1]) * ldc;
        float* dst = blk + ((size_t)(node0 + c) << lp_log2);
        if (vec) reinterpret_cast<float4*>(dst)[q] = __ldg(reinterpret_cast<const float4*>(src) + q);
        else dst[q] = (q < tc) ? __ldg(src + q) : 0.f;
      }
    }
    __syncthreads();
    if (col < tc) {
      int pitch[D];
#pragma unroll
      for (int i = 0; i < D; ++i) pitch[i] = b.pitch[i] << lp_log2;
      for (int p = p0 + slot; p < p1; p += nslot) {
        float4 w[D];
        int node = 0;
#pragma unroll
        for (int i = 0; i < D; ++i) {
          node += (first_s[(int64_t)p * D + i] - b.base[i]) * b.pitch[i];
          w[i] = reinterpret_cast<const float4*>(wts_s)[(int64_t)p * D + i];
        }
        const float v = SkiInterpSum<D, 0>::run(blk + ((size_t)node << lp_log2) + col, w, pitch);
        out[(int64_t)perm[p] * ldo + col] = v;
      }
    }
  }
}

template <int D>
static int ski_grid_matmul_d(gp_plan* p, const float* V, int64_t ldv, int t, float* OUT, int64_t ldo) {
  SkiPass ps;
  GP_CHECK(ski_tiled_pass<D>(p, &ps));
  GP_CHECK(p->V16.ensure(sizeof(float) * p->n1 * TP));
  for (int c0 = 0; c0 < t; c0 += TP) GP_CHECK(ski_grid_block<D>(p, ps, V + c0, ldv, std::min(TP, t - c0), OUT + c0, ldo));
  return GP_OK;
}

template <int D>
static int ski_interp_matmul_d(gp_plan* p, const float* C, int64_t ldc, int t, float* OUT, int64_t ldo) {
  const gp_ski_state* s = p->ski;
  SkiPass ps;
  GP_CHECK(ski_tiled_pass<D>(p, &ps));
  GP_CHECK(opt_in_smem<ski_interp_tiled_kernel<D>>(p->device, SKI_TILE_SMEM));
  for (int c0 = 0; c0 < t; c0 += SKI_IP_CW) {
    const int tc = std::min(SKI_IP_CW, t - c0);
    int lg = 0;
    while ((1 << lg) < tc) ++lg;
    const int vec = tc == (1 << lg) && tc >= 4 && ldc % 4 == 0 && (reinterpret_cast<uintptr_t>(C + c0) & 15) == 0;
    ski_interp_tiled_kernel<D><<<ps.grid, SKI_IP_THREADS, ps.nodes * (sizeof(float) << lg), p->stream>>>(
        s->first_s.as<int>(), s->wts_s.as<float>(), s->perm.as<int>(), s->tile_off.as<int>(), ps.g, ps.tl, ps.parts, C + c0, ldc, tc,
        lg, vec, OUT + c0, ldo);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// ---- input gradient (gp_ski_input_grad: deep kernel learning through a KISS-GP operator) -------------------------------------------
// F = sum_i L_i . (K_ski R)_i with K_ski = s W K_uu W^T.  Row i of W depends on x_i alone, so
//   dF/dx_ik = sum_c [ L_ic (d_k W_i . B_R)_c + R_ic (d_k W_i . B_L)_c ],   B_R = s K_uu W^T R,  B_L = s K_uu W^T L   ([M][t] grid blocks)
// where d_k W_i is row i's 4^D tensor-product weights with the dimension-k factor replaced by dw_k (ski_axis_weights<true>).
// One CTA per (tile, part), as ski_interp_tiled_kernel: the tile's node block of one column chunk [B_R | B_L] (2 tc <= 32 columns,
// padded to LP = a power of two) is staged in shared memory; a lane owns one (point, column) pair, forms the D derivative-weighted
// sums in the fixed separable order and multiplies each by its paired coefficient (L_ic for a B_R column, R_ic for a B_L column).
// The LP lanes of a point reduce with a fixed xor-shuffle tree; chunk c0 > 0 adds to what the previous chunk wrote (same stream,
// fixed order).  The pass has no atomics; B_R / B_L come from the product's scatter, whose per-tile red.add order varies, so
// repeated calls agree to the rounding of those sums.  The plan keeps no cell fractions, so the weights and
// their derivatives are recomputed from the plan's inputs X by the helper that packed them.
template <int D>
__global__ void __launch_bounds__(SKI_IP_THREADS)
ski_input_grad_tiled_kernel(const int* __restrict__ first_s, const int* __restrict__ perm, const int* __restrict__ off, SkiGeom g,
                            SkiTiles tl, int parts, const float* __restrict__ X, int64_t ldx, const float* __restrict__ BR,
                            const float* __restrict__ BL, int tc, int lp_log2, const float* __restrict__ L, int64_t ldl,
                            const float* __restrict__ R, int64_t ldr, int accumulate, float* __restrict__ DX, int64_t lddx) {
  extern __shared__ __align__(16) float blk[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int lp = 1 << lp_log2;
  const int col = lane & (lp - 1);
  const int ppw = 32 >> lp_log2;                          // points per warp and step
  const int pstep = (SKI_IP_THREADS / 32) * ppw;
  for (int64_t wk = blockIdx.x; wk < (int64_t)tl.ntiles * parts; wk += gridDim.x) {
    int tile, p0, p1;
    if (!ski_work_range(wk, parts, off, tile, p0, p1)) continue;
    const SkiBlock<D> b = ski_block_of<D>(tile, g, tl);
    __syncthreads();
    const int last = b.ext[D - 1];
    const int nrows = b.nodes / last;
    for (int row = warp; row < nrows; row += SKI_IP_THREADS / 32) {
      const auto [node0, idx0] = ski_row_origin<D>(b, g, row);
      for (int e = lane; e < (last << lp_log2); e += 32) {
        const int c = e >> lp_log2, q = e & (lp - 1);
        const int64_t gi = (idx0 + (int64_t)c * g.stride[D - 1]) * TP;
        blk[((size_t)(node0 + c) << lp_log2) + q] = (q < tc) ? __ldg(BR + gi + q) : (q < 2 * tc ? __ldg(BL + gi + q - tc) : 0.f);
      }
    }
    __syncthreads();
    int pitch[D];
#pragma unroll
    for (int i = 0; i < D; ++i) pitch[i] = b.pitch[i] << lp_log2;
    // warp-uniform trip count: the reduction shuffles need every lane
    for (int pb = p0 + warp * ppw; pb < p1; pb += pstep) {
      const int p = pb + (lane >> lp_log2);
      const bool live = p < p1;
      float gk[D];
#pragma unroll
      for (int k = 0; k < D; ++k) gk[k] = 0.f;
      int row = 0;
      if (live) {
        row = perm[p];
        float4 w[D], dw[D];
        int node = 0;
#pragma unroll
        for (int i = 0; i < D; ++i) {
          float a[4], da[4];
          ski_axis_weights<true>(X[(int64_t)row * ldx + i], g.lo[i], g.step[i], g.G[i], a, da);
          w[i] = make_float4(a[0], a[1], a[2], a[3]);
          dw[i] = make_float4(da[0], da[1], da[2], da[3]);
          node += (first_s[(int64_t)p * D + i] - b.base[i]) * b.pitch[i];
        }
        if (col < 2 * tc) {
          const float coef = (col < tc) ? L[(int64_t)row * ldl + col] : R[(int64_t)row * ldr + (col - tc)];
          const float* base = blk + ((size_t)node << lp_log2) + col;
#pragma unroll
          for (int k = 0; k < D; ++k) {
            float4 wk[D];
#pragma unroll
            for (int i = 0; i < D; ++i) wk[i] = (i == k) ? dw[i] : w[i];
            gk[k] = coef * SkiInterpSum<D, 0>::run(base, wk, pitch);
          }
        }
      }
      for (int o = 1; o < lp; o <<= 1) {
#pragma unroll
        for (int k = 0; k < D; ++k) gk[k] += __shfl_xor_sync(0xffffffffu, gk[k], o);
      }
      if (live && col == 0) {
        float* dst = DX + (int64_t)row * lddx;
#pragma unroll
        for (int k = 0; k < D; ++k) dst[k] = accumulate ? dst[k] + gk[k] : gk[k];
      }
    }
  }
}

template <int D>
static int ski_input_grad_d(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, float* DX, int64_t lddx) {
  gp_ski_state* s = p->ski;
  SkiPass ps;
  GP_CHECK(ski_tiled_pass<D>(p, &ps));
  GP_CHECK(opt_in_smem<ski_input_grad_tiled_kernel<D>>(p->device, SKI_TILE_SMEM));
  // B_R / B_L of one 16-column chunk live in the bilinear derivative's grid blocks (allocated by the hyper-parameter backward)
  GP_CHECK(p->V16.ensure(sizeof(float) * p->n1 * TP));
  GP_CHECK(s->gridC.ensure(sizeof(float) * ps.g.M * TP));
  GP_CHECK(s->gridD.ensure(sizeof(float) * ps.g.M * TP));
  float* BR = s->gridC.as<float>();
  float* BL = s->gridD.as<float>();
  for (int c0 = 0; c0 < t; c0 += TP) {
    const int tc = std::min(TP, t - c0);
    GP_CHECK(ski_grid_block<D>(p, ps, R + c0, ldr, tc, BR, TP));
    GP_CHECK(ski_grid_block<D>(p, ps, L + c0, ldl, tc, BL, TP));
    int lg = 1;
    while ((1 << lg) < 2 * tc) ++lg;
    ski_input_grad_tiled_kernel<D><<<ps.grid, SKI_IP_THREADS, ps.nodes * (sizeof(float) << lg), p->stream>>>(
        s->first_s.as<int>(), s->perm.as<int>(), s->tile_off.as<int>(), ps.g, ps.tl, ps.parts, p->X1, p->ld1, BR, BL, tc, lg,
        L + c0, ldl, R + c0, ldr, c0 > 0, DX, lddx);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// the arguments both calls share: a packed, unsharded SKI plan; t >= 1 columns, leading dimensions >= t
static int ski_predict_check(gp_plan* p, int t, int64_t ld_in, int64_t ld_out, const char* what) {
  GP_REQUIRE(p != nullptr && p->data_set && p->hypers_set, GP_E_STATE, "%s: plan not ready (set_data + set_ski + set_hypers)", what);
  GP_REQUIRE(p->backend == GP_BACKEND_SKI && p->ski != nullptr, GP_E_STATE, "%s needs a SKI plan (gp_plan_set_ski)", what);
  GP_REQUIRE(!(p->comm && p->comm->world > 1) && p->row_begin == 0 && p->row_count == p->n1, GP_E_SHAPE,
             "%s is not available on row-sharded plans", what);
  GP_REQUIRE(t >= 1 && ld_in >= t && ld_out >= t, GP_E_SHAPE, "%s: bad shape t=%d, leading dimensions %lld / %lld", what, t,
             (long long)ld_in, (long long)ld_out);
  GP_REQUIRE(p->ski->tcol.p != nullptr && p->ski->perm.p != nullptr, GP_E_STATE, "%s: SKI grid not packed", what);
  GP_CUDA(cudaSetDevice(p->device));
  return GP_OK;
}

}  // namespace gp

using namespace gp;

// GridInterpolationKernel(base_kernel, grid_size, num_dims, grid_bounds): grid_lo = first node, grid_step = node spacing
// (utils/grid.py:142-180 create_grid: linspace(lo - step, hi + step, size) per dimension)
extern "C" int gp_plan_set_ski(gp_plan* p, const int* grid_sizes, const float* grid_lo, const float* grid_step, int d) {
  GP_REQUIRE(p != nullptr && p->data_set, GP_E_STATE, "set_data must precede set_ski");
  GP_CHECK(refuse_settings(p, CALL_SET_SKI));
  GP_REQUIRE(d == p->d && d >= 1 && d <= SKI_MAXD, GP_E_SHAPE, "SKI: grid dimension %d does not match the data (d=%d, max %d)", d, p->d, SKI_MAXD);
  int64_t M = 1;
  bool large = false;
  for (int i = 0; i < d; ++i) {
    GP_REQUIRE(grid_sizes[i] >= 4 && grid_sizes[i] <= SKI_MAX_G && grid_step[i] > 0.f, GP_E_SHAPE,
               "SKI: grid size %d (dim %d) must be in [4, %d]", grid_sizes[i], i, SKI_MAX_G);
    M = std::min<int64_t>(M * grid_sizes[i], (int64_t)1 << 40);   // saturated: 4 dimensions of 2^17 would overflow
    large |= grid_sizes[i] > SKI_DENSE_G;
  }
  // the mode kernels index the [M][16] grid block's positions in 32 bits; grids within [4, 128]^d keep the limits they always had
  // (the per-mode check in ski_mode_products)
  GP_REQUIRE(!large || M * TP < ((int64_t)1 << 31), GP_E_SHAPE, "SKI: grid of %lld nodes too large (M * 16 must be below 2^31)",
             (long long)M);
  if (!p->ski) p->ski = new gp_ski_state();
  for (int i = 0; i < d; ++i) { p->ski->G[i] = grid_sizes[i]; p->ski->lo[i] = grid_lo[i]; p->ski->step[i] = grid_step[i]; }
  p->backend_req = GP_BACKEND_SKI;
  p->backend = GP_BACKEND_SKI;
  if (p->hypers_set) return pack_inputs(p);
  return GP_OK;
}

extern "C" int gp_ski_grid_matmul(gp_plan* p, const float* V, int64_t ldv, int t, float* OUT, int64_t ldo) {
  GP_CHECK(ski_predict_check(p, t, ldv, ldo, "gp_ski_grid_matmul"));
  return ski_with_d(p->d, [&](auto D) { return ski_grid_matmul_d<D>(p, V, ldv, t, OUT, ldo); });
}

extern "C" int gp_ski_input_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, float* DX, int64_t lddx) {
  GP_CHECK(ski_predict_check(p, t, ldl, ldr, "gp_ski_input_grad"));
  GP_CHECK(refuse_settings(p, CALL_SKI_INPUT_GRAD));
  GP_REQUIRE(L && R && DX && lddx >= p->d, GP_E_SHAPE, "gp_ski_input_grad: bad output (leading dimension %lld, d=%d)", (long long)lddx, p->d);
  return ski_with_d(p->d, [&](auto D) { return ski_input_grad_d<D>(p, L, ldl, R, ldr, t, DX, lddx); });
}

extern "C" int gp_ski_interp_matmul(gp_plan* p, const float* C, int64_t ldc, int t, float* OUT, int64_t ldo) {
  GP_CHECK(ski_predict_check(p, t, ldc, ldo, "gp_ski_interp_matmul"));
  return ski_with_d(p->d, [&](auto D) { return ski_interp_matmul_d<D>(p, C, ldc, t, OUT, ldo); });
}
