// compact.cu -- the compact-support backend (GP_BACKEND_COMPACT): piecewise polynomial kernels (R&W eq. 4.21, the reference's
// kernels/piecewise_polynomial_kernel.py), k = (1 - r)_+^(j+q) poly_q(r), r = |(x - x') / l|, which is exactly zero for r >= 1.
//
// Once per gp_plan_set_data each side's points are put in Morton order of their raw inputs (a stable device radix sort, so the
// order does not depend on the lengthscales) and grouped into row tiles of PP_TI and column tiles of PP_TJ sorted points, each with
// the bounding box of its raw coordinates.  Once per hyper-parameter update the rows are packed as (x - mean) / l in sorted order and
// every row tile gets the CSR list of the column tiles whose boxes, scaled by 1 / l, are closer than 1 (in fp64: the squared gap is
// a lower bound of r^2 for every pair of the two tiles, so no pair with r < 1 is dropped).  A pair with r >= 1 inside a listed tile
// pair contributes an exact 0 through max(0, 1 - r), so the sparse K.V is the dense fp32 evaluation up to summation order.
//
// K.V: one CTA per (row tile, slot); slot k of a row tile walks entries [k chunk, (k + 1) chunk) of its list and writes the usual
// partial[slot][row][16], rows stored back through the permutation, so the finish, mBCG, MINRES, Lanczos and SLQ kernels run
// unchanged.  Every (row tile, slot) writes its rows, zeros where the list is shorter.  No atomics: repeated calls are bit-identical.
// Rows, the diagonal and the pivoted Cholesky read the caller-ordered packed rows Z2 through cov_from_arg<PP_K> (kmv_simt.cu,
// pivchol.cu).
#include <limits.h>

#include <algorithm>
#include <cub/cub.cuh>

#include "gp_common.cuh"
#include "simt_pass.cuh"

namespace gp {

// keep a tile pair while its squared box gap (fp64) is below this; the slack above 1 only adds tile pairs
constexpr double PP_REACH2 = 1.0 + 1.0 / 1048576.0;

CovParam pp_param(int q, int d) {
  const int j = d / 2 + q + 1;
  const double J = j;
  double c1 = 0.0, c2 = 0.0, c3 = 0.0;
  if (q == 1) {
    c1 = J + 1.0;
  } else if (q == 2) {
    c1 = J + 2.0;
    c2 = (J + 4.0 * J + 3.0) / 3.0;   // the reference module's coefficient; R&W eq. 4.21 has (j^2 + 4 j + 3) / 3 (DESIGN 4.24)
  } else if (q == 3) {
    c1 = J + 3.0;
    c2 = (6.0 * J * J + 36.0 * J + 45.0) / 15.0;
    c3 = (J * J * J + 9.0 * J * J + 23.0 * J + 15.0) / 15.0;
  }
  CovParam cp{};
  cp.pp_e = j + q;
  cp.pp_c1 = (float)c1;
  cp.pp_c2 = (float)c2;
  cp.pp_c3 = (float)c3;
  return cp;
}

// bits per dimension of the Morton key: bits * d <= 60
__host__ __device__ inline int pp_key_bits(int d) { return std::min(20, 60 / d); }

// per-dimension lo / hi of the finite raw inputs (one CTA per dimension): lohi[c] = lo, lohi[d + c] = hi
__global__ void pp_lohi_kernel(const float* __restrict__ X, int64_t n, int64_t ld, float* __restrict__ lohi) {
  const int c = blockIdx.x, d = gridDim.x;
  __shared__ float slo[256], shi[256];
  float lo = INFINITY, hi = -INFINITY;
  for (int64_t r = threadIdx.x; r < n; r += blockDim.x) {
    const float v = X[r * ld + c];
    if (isfinite(v)) {
      lo = fminf(lo, v);
      hi = fmaxf(hi, v);
    }
  }
  slo[threadIdx.x] = lo;
  shi[threadIdx.x] = hi;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      slo[threadIdx.x] = fminf(slo[threadIdx.x], slo[threadIdx.x + s]);
      shi[threadIdx.x] = fmaxf(shi[threadIdx.x], shi[threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    lohi[c] = slo[0];
    lohi[d + c] = shi[0];
  }
}

// Morton key of every point: cell_c = floor((x_c - lo_c) / (hi_c - lo_c) 2^bits) (clamped; 0 for a non-finite coordinate, so a
// NaN cannot break the sort), bit b of dimension c at key bit b d + c.  Explicitly rounded fp64 steps: the same keys in numpy.
__global__ void pp_key_kernel(const float* __restrict__ X, int64_t n, int64_t ld, int d, int bits, const float* __restrict__ lohi,
                              unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long top = (1ull << bits) - 1ull;
  const double cells = (double)(1ull << bits);
  unsigned long long key = 0ull;
  for (int c = 0; c < d; ++c) {
    const float v = X[i * ld + c];
    const double lo = lohi[c], hi = lohi[d + c];
    unsigned long long cell = 0ull;
    if (isfinite(v) && hi > lo) {
      const double t = __dmul_rn(__ddiv_rn(__dsub_rn((double)v, lo), __dsub_rn(hi, lo)), cells);
      cell = t >= cells ? top : (unsigned long long)t;
    }
    for (int b = 0; b < bits; ++b) key |= ((cell >> b) & 1ull) << (b * d + c);
  }
  keys[i] = key;
  vals[i] = (int)i;
}

// raw bounding box of every tile of `tile` sorted points: box[t][0][c] = lo, box[t][1][c] = hi (non-finite values ignored)
__global__ void pp_box_kernel(const float* __restrict__ X, int64_t ld, int d, const int* __restrict__ perm, int64_t n, int tile,
                              int64_t ntile, float* __restrict__ box) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ntile * d) return;
  const int64_t t = idx / d;
  const int c = (int)(idx % d);
  float lo = INFINITY, hi = -INFINITY;
  const int64_t e = min(n, (t + 1) * tile);
  for (int64_t r = t * tile; r < e; ++r) {
    const float v = X[(int64_t)perm[r] * ld + c];
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  box[(t * 2) * d + c] = lo;
  box[(t * 2 + 1) * d + c] = hi;
}

// packed rows in sorted order: Zs[s] = Z[perm[s]]
__global__ void pp_gather_kernel(const float* __restrict__ Z, const int* __restrict__ perm, int64_t n, int DP, float* __restrict__ Zs) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * DP) return;
  const int64_t s = idx / DP;
  Zs[idx] = Z[(int64_t)perm[s] * DP + idx % DP];
}

// whether row tile box a and column tile box b may hold a pair with r < 1: sum_c (gap_c / l_c)^2 < PP_REACH2, gap_c = max(0,
// lo_b - hi_a, lo_a - hi_b) in fp64 (a difference of two fp32 values), explicitly rounded in dimension order
__device__ __forceinline__ bool pp_reach(const float* __restrict__ a, const float* __restrict__ b, const double* __restrict__ ls, int d) {
  double s = 0.0;
  for (int c = 0; c < d; ++c) {
    const double g = fmax(fmax(__dsub_rn((double)b[c], (double)a[d + c]), __dsub_rn((double)a[c], (double)b[d + c])), 0.0);
    const double u = __ddiv_rn(g, ls[c]);
    s = __dadd_rn(s, __dmul_rn(u, u));
  }
  return s < PP_REACH2;
}

// one CTA per row tile: how many column tiles are within reach
__global__ void pp_count_kernel(const float* __restrict__ box1, const float* __restrict__ box2, int64_t ntile_j, int d,
                                const double* __restrict__ ls, int* __restrict__ cnt) {
  const int64_t it = blockIdx.x;
  const float* a = box1 + it * 2 * d;
  int k = 0;
  for (int64_t jt = threadIdx.x; jt < ntile_j; jt += blockDim.x) k += pp_reach(a, box2 + jt * 2 * d, ls, d) ? 1 : 0;
  typedef cub::BlockReduce<int, 256> Reduce;
  __shared__ typename Reduce::TempStorage tmp;
  const int tot = Reduce(tmp).Sum(k);
  if (threadIdx.x == 0) cnt[it] = tot;
}

// one CTA per row tile: its column tiles within reach, ascending
__global__ void pp_fill_kernel(const float* __restrict__ box1, const float* __restrict__ box2, int64_t ntile_j, int d,
                               const double* __restrict__ ls, const int64_t* __restrict__ rowptr, int* __restrict__ cols) {
  const int64_t it = blockIdx.x;
  const float* a = box1 + it * 2 * d;
  typedef cub::BlockScan<int, 256> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int64_t base;
  if (threadIdx.x == 0) base = rowptr[it];
  __syncthreads();
  for (int64_t j0 = 0; j0 < ntile_j; j0 += blockDim.x) {
    const int64_t jt = j0 + threadIdx.x;
    const int keep = (jt < ntile_j && pp_reach(a, box2 + jt * 2 * d, ls, d)) ? 1 : 0;
    int pos, tot;
    Scan(tmp).ExclusiveSum(keep, pos, tot);
    if (keep) cols[base + pos] = (int)jt;
    __syncthreads();
    if (threadIdx.x == 0) base += tot;
    __syncthreads();
  }
}

struct PpSched {
  const float* Zs1;
  const float* Zs2;
  const int* perm1;
  const int* perm2;
  const int64_t* rowptr;
  const int* cols;
  int chunk;
  int64_t n1, n2;
};

// stage column tile jt: its sorted packed rows and the 16 columns of B (caller's order, gathered through perm2); zero beyond n2
template <int DP>
__device__ __forceinline__ void pp_stage(const PpSched& s, int64_t jt, const float* __restrict__ B, float (*zj)[DP], float (*bj)[TP]) {
  const int64_t j0 = jt * PP_TJ;
  const int nj = (int)min((int64_t)PP_TJ, s.n2 - j0);
  for (int e = threadIdx.x; e < PP_TJ * DP / 4; e += PP_TI) {
    const int jj = e / (DP / 4);
    reinterpret_cast<float4*>(&zj[0][0])[e] =
        jj < nj ? reinterpret_cast<const float4*>(s.Zs2 + j0 * DP)[e] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int e = threadIdx.x; e < PP_TJ * TP / 4; e += PP_TI) {
    const int jj = e / (TP / 4), q = e % (TP / 4);
    reinterpret_cast<float4*>(&bj[0][0])[e] =
        jj < nj ? reinterpret_cast<const float4*>(B + (int64_t)s.perm2[j0 + jj] * TP)[q] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// grid (ntile_i, nparts), PP_TI threads, one sorted row each
template <int DP>
__global__ void __launch_bounds__(PP_TI)
pp_kmv_kernel(PpSched s, const float* __restrict__ V16, float* __restrict__ partial, int64_t rows_pad, CovParam cp,
              const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  __shared__ __align__(16) float zj[PP_TJ][DP];
  __shared__ __align__(16) float vj[PP_TJ][TP];
  const int64_t it = blockIdx.x, slot = blockIdx.y;
  const int64_t i = it * PP_TI + threadIdx.x;
  const bool rv = i < s.n1;
  float zi[DP];
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? s.Zs1[i * DP + c] : 0.f;
  float acc[TP];
#pragma unroll
  for (int c = 0; c < TP; ++c) acc[c] = 0.f;
  const int64_t b = s.rowptr[it] + slot * s.chunk, e = min(s.rowptr[it + 1], b + s.chunk);
  for (int64_t l = b; l < e; ++l) {
    __syncthreads();
    pp_stage<DP>(s, s.cols[l], V16, zj, vj);
    __syncthreads();
#pragma unroll 4
    for (int jj = 0; jj < PP_TJ; ++jj) {
      float r2 = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        const float df = zi[c] - zj[jj][c];
        r2 = fmaf(df, df, r2);
      }
      const float k = pp_k(sqrtf(r2), cp);
#pragma unroll
      for (int c = 0; c < TP; ++c) acc[c] = fmaf(k, vj[jj][c], acc[c]);
    }
  }
  if (rv) {
    float4* dst = reinterpret_cast<float4*>(partial + (slot * rows_pad + s.perm1[i]) * TP);
#pragma unroll
    for (int q = 0; q < 4; ++q) dst[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
  }
}

// Bilinear gradient over the same units: gout[unit][0] = sum w k, then ARD: gout[unit][1 + c] = sum w (-k'(r)) dz_c^2 / r, else
// gout[unit][1] = sum w (-k'(r)) r, with w = L_i . R_j.  fp32 within one column tile, fp64 across tiles and in the CTA reduction.
template <int DP, bool ARD>
__global__ void __maxnreg__(168)   // the ARD variant holds d fp64 and d fp32 accumulators per thread
pp_bilinear_kernel(PpSched s, const float* __restrict__ L16, const float* __restrict__ R16, CovParam cp, int d,
                   double* __restrict__ gout, int gstride) {
  __shared__ __align__(16) float zj[PP_TJ][DP];
  __shared__ __align__(16) float rj[PP_TJ][TP];
  constexpr int NG = ARD ? DP : 1;
  const int64_t it = blockIdx.x, slot = blockIdx.y;
  const int64_t i = it * PP_TI + threadIdx.x;
  const bool rv = i < s.n1;
  float zi[DP], li[TP];
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? s.Zs1[i * DP + c] : 0.f;
  const int64_t ui = rv ? (int64_t)s.perm1[i] : 0;
#pragma unroll
  for (int c = 0; c < TP; ++c) li[c] = rv ? L16[ui * TP + c] : 0.f;
  double hk = 0.0, hl[NG];
#pragma unroll
  for (int c = 0; c < NG; ++c) hl[c] = 0.0;
  const int64_t b = s.rowptr[it] + slot * s.chunk, e = min(s.rowptr[it + 1], b + s.chunk);
  for (int64_t l = b; l < e; ++l) {
    __syncthreads();
    pp_stage<DP>(s, s.cols[l], R16, zj, rj);
    __syncthreads();
    float gk = 0.f, gl[NG];
#pragma unroll
    for (int c = 0; c < NG; ++c) gl[c] = 0.f;
    for (int jj = 0; jj < PP_TJ; ++jj) {
      float w = 0.f;
#pragma unroll
      for (int c = 0; c < TP; ++c) w = fmaf(li[c], rj[jj][c], w);
      float df2[DP], r2 = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        const float df = zi[c] - zj[jj][c];
        df2[c] = df * df;
        r2 += df2[c];
      }
      const float r = sqrtf(r2);
      gk = fmaf(w, pp_k(r, cp), gk);
      const float g = w * pp_mdk(r, cp);
      if (ARD) {
        const float gs = r > 0.f ? g / r : 0.f;   // dz_c^2 / r <= r: bounded, and 0 at r = 0 (the diagonal, duplicate points)
#pragma unroll
        for (int c = 0; c < NG; ++c) gl[c] = fmaf(gs, df2[c], gl[c]);
      } else {
        gl[0] = fmaf(g, r, gl[0]);
      }
    }
    hk += (double)gk;
#pragma unroll
    for (int c = 0; c < NG; ++c) hl[c] += (double)gl[c];
  }
  __shared__ double red[PP_TI];
  const int nout = 1 + (ARD ? d : 1);
  const int64_t unit = slot * gridDim.x + it;
#pragma unroll
  for (int o = 0; o < 1 + NG; ++o) {   // unrolled: every accumulator is read at a compile-time index (no local memory)
    if (o >= nout) break;
    const double v = o == 0 ? hk : hl[o > 0 ? o - 1 : 0];
    __syncthreads();
    block_sum_store<PP_TI>(red, v, gout + unit * gstride + o);
  }
}

static PpSched pp_sched(gp_plan* p) {
  const gp_compact_state* c = p->compact;
  const float* Zs1 = p->same ? c->Zs2.as<float>() : c->Zs1.as<float>();
  const int* perm2 = p->same ? c->perm1.as<int>() : c->perm2.as<int>();
  return PpSched{Zs1, c->Zs2.as<float>(), c->perm1.as<int>(), perm2, c->rowptr.as<int64_t>(), c->cols.as<int>(), c->chunk, p->n1, p->n2};
}

// Morton order of n points X (stable: equal keys keep their input order) -> perm [n] int32
static int pp_sort_side(gp_plan* p, const float* X, int64_t n, int64_t ld, gp::DevBuf& perm) {
  gp_compact_state* c = p->compact;
  cudaStream_t st = p->stream;
  const int d = p->d, bits = pp_key_bits(d);
  GP_CHECK(c->lohi.ensure(sizeof(float) * 2 * d));
  pp_lohi_kernel<<<d, 256, 0, st>>>(X, n, ld, c->lohi.as<float>());
  size_t tb = 0;
  GP_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                          (const int*)nullptr, (int*)nullptr, (int)n, 0, bits * d, st));
  const size_t kb = sizeof(unsigned long long) * (size_t)n, vb = (sizeof(int) * (size_t)n + 255) / 256 * 256;
  GP_CHECK(c->sortbuf.ensure(2 * kb + vb + tb));
  char* base = c->sortbuf.as<char>();
  unsigned long long* kin = reinterpret_cast<unsigned long long*>(base);
  unsigned long long* kout = reinterpret_cast<unsigned long long*>(base + kb);
  int* vin = reinterpret_cast<int*>(base + 2 * kb);
  GP_CHECK(perm.ensure(sizeof(int) * (size_t)n));
  pp_key_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(X, n, ld, d, bits, c->lohi.as<float>(), kin, vin);
  GP_CUDA(cub::DeviceRadixSort::SortPairs(base + 2 * kb + vb, tb, kin, kout, vin, perm.as<int>(), (int)n, 0, bits * d, st));
  p->launches += 3;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

static int pp_boxes(gp_plan* p, const float* X, int64_t ld, const int* perm, int64_t n, int tile, int64_t ntile, gp::DevBuf& box) {
  const int d = p->d;
  GP_CHECK(box.ensure(sizeof(float) * 2 * d * (size_t)ntile));
  pp_box_kernel<<<(unsigned)cdiv(ntile * d, 128), 128, 0, p->stream>>>(X, ld, d, perm, n, tile, ntile, box.as<float>());
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int compact_pack(gp_plan* p) {
  gp_compact_state* c = p->compact;
  GP_REQUIRE(p->d >= 1 && p->d <= PP_DMAX, GP_E_SHAPE, "a piecewise polynomial kernel takes 1 <= d <= %d input columns (d=%d)",
             PP_DMAX, p->d);
  GP_REQUIRE(p->row_begin == 0 && p->row_count == p->n1, GP_E_STATE,
             "the piecewise polynomial backend needs every row on one rank; this plan is row-sharded");
  GP_REQUIRE(p->n1 < INT_MAX && p->n2 < INT_MAX, GP_E_SHAPE, "the piecewise polynomial backend takes fewer than 2^31 points per side");
  cudaStream_t st = p->stream;
  const int d = p->d, DP = p->DP;
  const float* X2 = p->same ? p->X1 : p->X2;
  const int64_t ld2 = p->same ? p->ld1 : p->ld2;
  c->ntile_i = cdiv(p->n1, PP_TI);
  c->ntile_j = cdiv(p->n2, PP_TJ);
  if (c->order_stale) {
    GP_CHECK(pp_sort_side(p, p->X1, p->n1, p->ld1, c->perm1));
    if (!p->same) GP_CHECK(pp_sort_side(p, X2, p->n2, ld2, c->perm2));
    const int* perm2 = p->same ? c->perm1.as<int>() : c->perm2.as<int>();
    GP_CHECK(pp_boxes(p, p->X1, p->ld1, c->perm1.as<int>(), p->n1, PP_TI, c->ntile_i, c->box1));
    GP_CHECK(pp_boxes(p, X2, ld2, perm2, p->n2, PP_TJ, c->ntile_j, c->box2));
    c->order_stale = false;
  }
  // the packed rows in sorted order
  GP_CHECK(c->Zs2.ensure(sizeof(float) * (size_t)p->n2 * DP));
  pp_gather_kernel<<<(unsigned)cdiv(p->n2 * DP, 256), 256, 0, st>>>(p->Z2.as<float>(), p->same ? c->perm1.as<int>() : c->perm2.as<int>(),
                                                                   p->n2, DP, c->Zs2.as<float>());
  p->launches++;
  if (!p->same) {
    GP_CHECK(c->Zs1.ensure(sizeof(float) * (size_t)p->n1 * DP));
    pp_gather_kernel<<<(unsigned)cdiv(p->n1 * DP, 256), 256, 0, st>>>(p->Z1.as<float>(), c->perm1.as<int>(), p->n1, DP, c->Zs1.as<float>());
    p->launches++;
  }
  // the tile-pair lists for these lengthscales
  std::vector<double> ls(d);
  for (int k = 0; k < d; ++k) ls[k] = (double)(p->ls.size() == 1 ? p->ls[0] : p->ls[k]);
  const int64_t nti = c->ntile_i, ntj = c->ntile_j;
  GP_CHECK(c->lsd.ensure(sizeof(double) * d));
  GP_CHECK(c->cnt.ensure(sizeof(int) * (size_t)nti));
  GP_CHECK(c->rowptr.ensure(sizeof(int64_t) * (size_t)(nti + 1)));
  GP_CUDA(cudaMemcpyAsync(c->lsd.p, ls.data(), sizeof(double) * d, cudaMemcpyHostToDevice, st));
  pp_count_kernel<<<(unsigned)nti, 256, 0, st>>>(c->box1.as<float>(), c->box2.as<float>(), ntj, d, c->lsd.as<double>(), c->cnt.as<int>());
  p->launches++;
  std::vector<int> cnt(nti);
  GP_CUDA(cudaMemcpyAsync(cnt.data(), c->cnt.p, sizeof(int) * nti, cudaMemcpyDeviceToHost, st));
  GP_CUDA(cudaStreamSynchronize(st));
  std::vector<int64_t> rowptr(nti + 1, 0);
  int64_t lmax = 0;
  for (int64_t t = 0; t < nti; ++t) {
    rowptr[t + 1] = rowptr[t] + cnt[t];
    lmax = std::max<int64_t>(lmax, cnt[t]);
  }
  c->pairs = rowptr[nti];
  GP_CHECK(c->cols.ensure(sizeof(int) * (size_t)std::max<int64_t>(1, c->pairs)));
  GP_CUDA(cudaMemcpyAsync(c->rowptr.p, rowptr.data(), sizeof(int64_t) * (nti + 1), cudaMemcpyHostToDevice, st));
  pp_fill_kernel<<<(unsigned)nti, 256, 0, st>>>(c->box1.as<float>(), c->box2.as<float>(), ntj, d, c->lsd.as<double>(),
                                                c->rowptr.as<int64_t>(), c->cols.as<int>());
  p->launches++;
  // slots: enough (row tile, slot) units for about four CTAs per SM, and no unit longer than twice the mean list (at least 8
  // column tiles), at most PP_MAX_SLOTS
  const int64_t mean = cdiv(std::max<int64_t>(c->pairs, 1), nti);
  const int64_t occ = cdiv(4 * (int64_t)p->n_sm, nti);
  int64_t chunk = std::max<int64_t>(1, cdiv(lmax, occ));
  chunk = std::min<int64_t>(chunk, std::max<int64_t>(8, 2 * mean));
  chunk = std::max<int64_t>(chunk, cdiv(std::max<int64_t>(lmax, 1), PP_MAX_SLOTS));
  c->chunk = (int)chunk;
  p->nsplit = p->nparts = (int)std::max<int64_t>(1, cdiv(lmax, chunk));
  GP_CUDA(cudaStreamSynchronize(st));   // rowptr is a stack-lifetime vector
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int compact_kmv_partials(gp_plan* p, const float* V16, const int* done_flag) {
  const PpSched s = pp_sched(p);
  const dim3 grid((unsigned)p->compact->ntile_i, (unsigned)p->nparts);
  const CovParam cp = cov_param(p);
  float* part = partial_ptr(p);
  switch (p->DP) {
    case 4: pp_kmv_kernel<4><<<grid, PP_TI, 0, p->stream>>>(s, V16, part, p->rows_pad, cp, done_flag); break;
    case 8: pp_kmv_kernel<8><<<grid, PP_TI, 0, p->stream>>>(s, V16, part, p->rows_pad, cp, done_flag); break;
    case 12: pp_kmv_kernel<12><<<grid, PP_TI, 0, p->stream>>>(s, V16, part, p->rows_pad, cp, done_flag); break;
    case 16: pp_kmv_kernel<16><<<grid, PP_TI, 0, p->stream>>>(s, V16, part, p->rows_pad, cp, done_flag); break;
    default: set_error("piecewise polynomial K.V: unsupported DP=%d", p->DP); return GP_E_SHAPE;
  }
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

template <bool ARD>
static int pp_bilinear_launch(gp_plan* p, const PpSched& s, const float* L16, const float* R16, double* gout, int gstride) {
  const dim3 grid((unsigned)p->compact->ntile_i, (unsigned)p->nparts);
  const CovParam cp = cov_param(p);
  switch (p->DP) {
    case 4: pp_bilinear_kernel<4, ARD><<<grid, PP_TI, 0, p->stream>>>(s, L16, R16, cp, p->d, gout, gstride); break;
    case 8: pp_bilinear_kernel<8, ARD><<<grid, PP_TI, 0, p->stream>>>(s, L16, R16, cp, p->d, gout, gstride); break;
    case 12: pp_bilinear_kernel<12, ARD><<<grid, PP_TI, 0, p->stream>>>(s, L16, R16, cp, p->d, gout, gstride); break;
    case 16: pp_bilinear_kernel<16, ARD><<<grid, PP_TI, 0, p->stream>>>(s, L16, R16, cp, p->d, gout, gstride); break;
    default: set_error("piecewise polynomial gradient: unsupported DP=%d", p->DP); return GP_E_SHAPE;
  }
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int compact_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  const bool ard = p->ls.size() > 1;
  const int nout = 1 + (ard ? p->d : 1);
  const PpSched sc = pp_sched(p);
  std::vector<double> total;
  GP_CHECK(bilinear_sweep(p, L, ldl, R, ldr, s, p->n1, p->compact->ntile_i * p->nparts, nout,
                          [&](const float* L16, const float* R16, double* gout) -> int {
                            return ard ? pp_bilinear_launch<true>(p, sc, L16, R16, gout, nout) : pp_bilinear_launch<false>(p, sc, L16, R16, gout, nout);
                          }, total));
  // dk/dl_c = -k'(r) dz_c^2 / (r l_c); one lengthscale: -k'(r) r / l.  Both times S
  *grad_os = total[0];
  if (ard)
    for (int c = 0; c < p->d; ++c) grad_ls[c] = p->outputscale * total[1 + c] / (double)p->ls[c];
  else
    grad_ls[0] = p->outputscale * total[1] / (double)p->ls[0];
  return GP_OK;
}

int refuse_compact(const gp_plan* p, const char* call) {
  if (p == nullptr || p->compact == nullptr) return GP_OK;
  set_error("%s: the plan runs the compact-support backend of a piecewise polynomial kernel (gp_plan_set_hypers_pp), which takes no "
            "other operator setting", call);
  return GP_E_STATE;
}

void compact_release(gp_plan* p) {
  gp_compact_state* c = p->compact;
  if (c == nullptr) return;
  gp::DevBuf* bufs[] = {&c->perm1, &c->perm2, &c->box1, &c->box2, &c->Zs1, &c->Zs2, &c->rowptr, &c->cols, &c->cnt,
                        &c->sortbuf, &c->lohi, &c->lsd};
  for (auto* b : bufs) b->release();
  delete c;
  p->compact = nullptr;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_hypers_pp(gp_plan* p, int q, const float* lengthscale, int n_ls, float outputscale, float noise) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(q >= 0 && q <= 3, GP_E_SHAPE, "q expected to be 0, 1, 2 or 3 (q=%d)", q);
  GP_REQUIRE(lengthscale && n_ls >= 1, GP_E_SHAPE, "lengthscale missing");
  GP_REQUIRE(!p->data_set || n_ls == 1 || n_ls == p->d, GP_E_SHAPE, "lengthscale count %d does not match d=%d", n_ls, p->d);
  for (int i = 0; i < n_ls; ++i)
    GP_REQUIRE(lengthscale[i] > 0.f && isfinite(lengthscale[i]), GP_E_SHAPE, "lengthscale[%d]=%g must be positive", i, lengthscale[i]);
  GP_REQUIRE(outputscale > 0.f && noise >= 0.f, GP_E_SHAPE, "outputscale must be > 0 and noise >= 0");
  // a plain plan only (a low-rank correction aside; an RQ or polynomial kind is replaced, as gp_plan_set_hypers replaces a kind)
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE,
             "gp_plan_set_hypers_pp takes a plain plan, and this one runs the SKI backend (gp_plan_set_ski)");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "gp_plan_set_hypers_pp takes a plain plan, and this one is a kernel sum");
  GP_REQUIRE((plan_settings(p) & ~(PS_LOWRANK | PS_RQ | PS_POLY)) == 0, GP_E_STATE,
             "gp_plan_set_hypers_pp takes a plain plan (a low-rank correction aside), and this one carries another operator setting");
  GP_REQUIRE(!(p->comm && p->comm->world > 1) && (!p->data_set || (p->row_begin == 0 && p->row_count == p->n1)), GP_E_STATE,
             "gp_plan_set_hypers_pp takes every row on one rank, and this plan is row-sharded");
  GP_CUDA(cudaSetDevice(p->device));
  // all or nothing, as gp_plan_set_hypers_rq: a failed pack restores the previous hyper-parameters (and packing)
  const bool fresh = p->compact == nullptr;
  if (fresh) p->compact = new gp_compact_state();
  const int old_kind = p->kind, old_q = p->compact->q;
  const std::vector<float> old_ls = p->ls;
  const float old_os = p->outputscale, old_noise = p->noise;
  const bool old_set = p->hypers_set;
  p->kind = GP_PPOLY;
  p->compact->q = q;
  p->ls.assign(lengthscale, lengthscale + n_ls);
  p->outputscale = outputscale;
  p->noise = noise;
  p->hypers_set = true;
  if (!p->data_set) return GP_OK;
  const int st = pack_inputs(p);
  if (st != GP_OK) {
    p->kind = old_kind;
    p->ls = old_ls;
    p->outputscale = old_os;
    p->noise = old_noise;
    p->hypers_set = old_set;
    if (fresh) compact_release(p);
    else p->compact->q = old_q;
    if (old_set) pack_inputs(p);   // the previous packing; the error reported is the first one
  }
  return st;
}

extern "C" int gp_plan_tile_pairs(gp_plan* p, int64_t* evaluated, int64_t* total) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(p->compact != nullptr && p->data_set && p->hypers_set, GP_E_STATE,
             "gp_plan_tile_pairs: the plan does not run the compact-support backend (gp_plan_set_hypers_pp), or is not packed");
  if (evaluated) *evaluated = p->compact->pairs;
  if (total) *total = p->compact->ntile_i * p->compact->ntile_j;
  return GP_OK;
}
