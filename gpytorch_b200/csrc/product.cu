// product.cu -- kernel products  K = S prod_f k_f  (ProductKernel, reference kernels/kernel.py:547-551, :634-690: the
// reference evaluates every factor densely and multiplies the N x N matrices).  A sum splits into one launch per term; a product
// does not, so it has fused kernels of its own that form prod_f k_f per pair in registers.
//
// The parent plan (backend GP_BACKEND_PRODUCT) owns no packed inputs: it holds the workspaces (partial slots, packed V tiles, CG
// state), the noise, the combined scale S = prod_f s_f (in gp_plan::outputscale, applied by the usual finish kernels) and the OR of
// the factors' non-finite-input flags.  The factors are complete plain plans over the same rows that keep their own packed inputs
// (their lengthscales / active dimensions differ); the kernels here read those arrays directly.
//
// One exponential per pair: in the packed units every covariance is poly(rho) 2^e (cov_poly_exp, gp_common.cuh), so
// prod_f k_f = (prod_f poly_f) ex2(sum_f e_f) costs one ex2 whatever the number of factors, plus one sqrt per Matern factor.
//
//   product_tc_kernel    two tensor-core factors, KP_a + KP_b <= 128: the one warp-specialised wgmma pipeline of kmv_tc.cu, run
//                        with a second GEMM1 operand (the factors' own packed tiles; S_a into s, S_b into the registers that
//                        hold P_hi afterwards) and the product covariance in the epilogue.  It and its launcher live in kmv_tc.cu.
//   product_simt_kernel  2 to 4 factors of a total padded width <= 128 on CUDA cores: the structure of kmv_simt_kernel with the
//                        factors' packed rows staged back to back, direct differences per factor, exact a_f = 0 on the diagonal.
//   product_bilinear_kernel  one pass over the pairs for every factor's lengthscale gradient and dF/dS (fp32, fp64 block partials).
#include <string.h>

#include <algorithm>

#include "gp_common.cuh"

namespace gp {

// ---- the factors as a kernel argument (indexed with compile-time constants only) ------------------------------------------
struct ProdFactors {
  int n;
  const float* Z1[4];   // packed rows of the row side / the column side, [.][DP[f]]
  const float* Z2[4];
  int DP[4];
  int rbf[4];
  CovPoly c[4];
};

// chunk q (4 floats) of the staged row belongs to the factor whose chunk range contains it: ends b[f] = sum_{g <= f} DP[g] / 4
struct ProdBounds {
  int b[4];
};
__device__ __forceinline__ ProdBounds prod_bounds(const ProdFactors& pf) {
  ProdBounds pb;
  int e = 0;
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    if (f < pf.n) e += pf.DP[f] >> 2;
    pb.b[f] = e;
  }
  return pb;
}

// row i of every factor's row side, back to back, zero beyond the last factor
template <int DPT>
__device__ __forceinline__ void prod_load_row(const ProdFactors& pf, const ProdBounds& pb, int64_t i, bool valid, float (&zi)[DPT]) {
#pragma unroll
  for (int q = 0; q < DPT / 4; ++q) {
    const float* src = nullptr;
    if (q < pb.b[0]) src = pf.Z1[0] + i * pf.DP[0] + 4 * q;
    else if (q < pb.b[1]) src = pf.Z1[1] + i * pf.DP[1] + 4 * (q - pb.b[0]);
    else if (q < pb.b[2]) src = pf.Z1[2] + i * pf.DP[2] + 4 * (q - pb.b[1]);
    else if (q < pb.b[3]) src = pf.Z1[3] + i * pf.DP[3] + 4 * (q - pb.b[2]);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (valid && src) v = *reinterpret_cast<const float4*>(src);
    zi[4 * q] = v.x; zi[4 * q + 1] = v.y; zi[4 * q + 2] = v.z; zi[4 * q + 3] = v.w;
  }
}

// columns [j0, j0 + nj) of every factor's column side into zj[SIMT_TJ][DPT] (rows >= nj zero)
template <int DPT>
__device__ __forceinline__ void prod_stage_cols(const ProdFactors& pf, const ProdBounds& pb, int64_t j0, int nj, float* zj, int tid) {
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    if (f < pf.n) {
      const int dp = pf.DP[f], off = 4 * (f ? pb.b[f - 1] : 0);
      const float* src = pf.Z2[f] + j0 * dp;
      for (int e = tid; e < SIMT_TJ * dp; e += SIMT_TI) {
        const int jj = e / dp, c = e - jj * dp;
        zj[jj * DPT + off + c] = (jj < nj) ? src[e] : 0.f;
      }
    }
  }
}

// per-factor squared distances of the staged row jj: sq[f] = |z_i,f - z_j,f|^2 (df2: the squared differences, column by column)
template <int DPT, bool KEEP>
__device__ __forceinline__ void prod_sqdist(const ProdBounds& pb, const float (&zi)[DPT], const float* zrow, float (&sq)[4], float* df2) {
  sq[0] = sq[1] = sq[2] = sq[3] = 0.f;
#pragma unroll
  for (int q = 0; q < DPT / 4; ++q) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float df = zi[4 * q + k] - zrow[4 * q + k];
      if (KEEP) df2[4 * q + k] = df * df;
      t = fmaf(df, df, t);
    }
    if (q < pb.b[0]) sq[0] += t;
    else if (q < pb.b[1]) sq[1] += t;
    else if (q < pb.b[2]) sq[2] += t;
    else sq[3] += t;
  }
}

// ---- (a) CUDA-core product kernel: grid (row blocks, nsplit); 128 threads, one output row each; partial[split][row][16] ----
template <int DPT>
__global__ void __launch_bounds__(SIMT_TI)
product_simt_kernel(const ProdFactors pf, const float* __restrict__ V16, float* __restrict__ partial, int64_t n1, int64_t n2,
                    int64_t rows_pad, int64_t cols_per_split, int same, int64_t row_begin, const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  __shared__ __align__(16) float zj[SIMT_TJ * DPT];
  __shared__ __align__(16) float vj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int split = blockIdx.y;
  const int64_t j_begin = (int64_t)split * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const ProdBounds pb = prod_bounds(pf);
  float zi[DPT];
  prod_load_row<DPT>(pf, pb, i, i < n1, zi);
  for (int e = tid; e < SIMT_TJ * DPT; e += SIMT_TI) zj[e] = 0.f;   // the padding columns beyond the last factor stay zero
  float acc[TP];
#pragma unroll
  for (int c = 0; c < TP; ++c) acc[c] = 0.f;
  const int64_t gi = i + row_begin;

  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    prod_stage_cols<DPT>(pf, pb, j0, nj, zj, tid);
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) (&vj[0][0])[e] = (e / TP < nj) ? V16[j0 * TP + e] : 0.f;
    __syncthreads();
#pragma unroll 2
    for (int jj = 0; jj < SIMT_TJ; ++jj) {
      float sq[4];
      prod_sqdist<DPT, false>(pb, zi, zj + jj * DPT, sq, nullptr);
      const bool dg = same && (j0 + jj) == gi;   // exact diagonal: every factor's argument is 0 (kernel.py:44-45)
      float poly = 1.f, e = 0.f;
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        if (f < pf.n) {
          float pl, ef;
          cov_poly_exp<true>(pf.rbf[f] != 0, pf.c[f], dg ? 0.f : -0.5f * sq[f], &pl, &ef);
          poly *= pl;
          e += ef;
        }
      }
      const float k = poly * ex2_approx(e);
#pragma unroll
      for (int c = 0; c < TP; ++c) acc[c] = fmaf(k, vj[jj][c], acc[c]);
    }
  }
  if (i < rows_pad) {
    float4* dst = reinterpret_cast<float4*>(partial + ((int64_t)split * rows_pad + i) * TP);
#pragma unroll
    for (int q = 0; q < 4; ++q) dst[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
  }
}

// ---- bilinear derivative of a product: one pass for every factor ---------------------------------------------------------------
//   gout[block][0]      = sum_ij w_ij prod_f k_f                                          (-> dF/dS)
//   gout[block][1 + c]  = sum_ij w_ij (prod_{g != f} k_g) g_f (z_ic - z_jc)^2 / |dz_f|^2  for staged column c of factor f
// (g_f = l dk_f/dl; a scalar-lengthscale factor sums its columns on the host, which gives sum w prod_{g != f} k_g g_f)
template <int DPT>
__global__ void __launch_bounds__(SIMT_TI)
product_bilinear_kernel(const ProdFactors pf, const float* __restrict__ L16, const float* __restrict__ R16, int64_t n1, int64_t n2,
                        int64_t cols_per_split, int same, int64_t row_begin, double* __restrict__ gout) {
  __shared__ __align__(16) float zj[SIMT_TJ * DPT];
  __shared__ __align__(16) float rj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int64_t j_begin = (int64_t)blockIdx.y * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const bool rv = i < n1;
  const ProdBounds pb = prod_bounds(pf);
  float zi[DPT], li[TP];
  prod_load_row<DPT>(pf, pb, i, rv, zi);
#pragma unroll
  for (int c = 0; c < TP; ++c) li[c] = rv ? L16[i * TP + c] : 0.f;
  for (int e = tid; e < SIMT_TJ * DPT; e += SIMT_TI) zj[e] = 0.f;
  float gk = 0.f, gl[DPT];
#pragma unroll
  for (int c = 0; c < DPT; ++c) gl[c] = 0.f;
  const int64_t gi = i + row_begin;
  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    prod_stage_cols<DPT>(pf, pb, j0, nj, zj, tid);
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) (&rj[0][0])[e] = (e / TP < nj) ? R16[j0 * TP + e] : 0.f;
    __syncthreads();
    for (int jj = 0; jj < nj; ++jj) {
      float w = 0.f;
#pragma unroll
      for (int c = 0; c < TP; ++c) w = fmaf(li[c], rj[jj][c], w);
      float sq[4], df2[DPT];
      prod_sqdist<DPT, true>(pb, zi, zj + jj * DPT, sq, df2);
      const bool dg = same && (j0 + jj) == gi;
      float pl[4], gp[4], e = 0.f;
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        pl[f] = 1.f;
        gp[f] = 0.f;
        if (f < pf.n) {
          float ef;
          dcov_poly_exp(pf.rbf[f] != 0, pf.c[f], dg ? 0.f : -0.5f * sq[f], &pl[f], &gp[f], &ef);
          e += ef;
        }
      }
      const float wE = w * ex2_approx(e);
      gk = fmaf(wE, pl[0] * pl[1] * pl[2] * pl[3], gk);
      // factor f: w (prod_{g != f} poly_g) gpoly_f E / |dz_f|^2, spread over its columns by their squared differences
      float gs[4];
      gs[0] = sq[0] > 0.f ? wE * gp[0] * pl[1] * pl[2] * pl[3] / sq[0] : 0.f;
      gs[1] = sq[1] > 0.f ? wE * pl[0] * gp[1] * pl[2] * pl[3] / sq[1] : 0.f;
      gs[2] = sq[2] > 0.f ? wE * pl[0] * pl[1] * gp[2] * pl[3] / sq[2] : 0.f;
      gs[3] = sq[3] > 0.f ? wE * pl[0] * pl[1] * pl[2] * gp[3] / sq[3] : 0.f;
#pragma unroll
      for (int q = 0; q < DPT / 4; ++q) {
        const float g = q < pb.b[0] ? gs[0] : q < pb.b[1] ? gs[1] : q < pb.b[2] ? gs[2] : gs[3];
#pragma unroll
        for (int k = 0; k < 4; ++k) gl[4 * q + k] = fmaf(g, df2[4 * q + k], gl[4 * q + k]);
      }
    }
  }
  // block reduction in double
  __shared__ double red[SIMT_TI];
  const int64_t blk = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
  for (int o = 0; o < 1 + DPT; ++o) {
    float v = (o == 0) ? gk : 0.f;
    if (o > 0) {
#pragma unroll
      for (int c = 0; c < DPT; ++c)
        if (c == o - 1) v = gl[c];
    }
    __syncthreads();
    red[tid] = (double)v;
    __syncthreads();
    for (int sft = SIMT_TI / 2; sft > 0; sft >>= 1) {
      if (tid < sft) red[tid] += red[tid + sft];
      __syncthreads();
    }
    if (tid == 0) gout[blk * (1 + DPT) + o] = red[0];
  }
}

// ---- small kernels ---------------------------------------------------------------------------------------------------------------
__global__ void product_or_flags_kernel(const int* f0, const int* f1, const int* f2, const int* f3, int* out) {
  *out = (*f0 | *f1 | (f2 ? *f2 : 0) | (f3 ? *f3 : 0)) ? 1 : 0;
}

__global__ void product_mul_rows_kernel(const float* __restrict__ src, int64_t n, float* __restrict__ OUT, int64_t ldo) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) OUT[blockIdx.y * ldo + j] *= src[blockIdx.y * n + j];
}

// ---- host ----------------------------------------------------------------------------------------------------------------------
static int round_dpt(int w) {
  const int opts[] = {8, 12, 16, 24, 32, 48, 64, 96, 128};
  for (int o : opts)
    if (w <= o) return o;
  return -1;
}

static ProdFactors prod_factors(const gp_plan* p) {
  ProdFactors pf;
  memset(&pf, 0, sizeof(pf));
  pf.n = (int)p->factors.size();
  for (int f = 0; f < pf.n; ++f) {
    const gp_plan* q = p->factors[f];
    pf.Z2[f] = q->Z2.as<float>();
    pf.Z1[f] = q->same ? q->Z2.as<float>() + q->row_begin * q->DP : q->Z1.as<float>();
    pf.DP[f] = q->DP;
    pf.rbf[f] = q->kind == GP_RBF;
    pf.c[f] = cov_poly_of(q->kind);
  }
  return pf;
}

int product_pack(gp_plan* p) {
  const int nf = (int)p->factors.size();
  GP_REQUIRE(nf >= 2 && nf <= 4, GP_E_SHAPE, "a kernel product takes 2 to 4 factors");
  GP_REQUIRE(p->row_begin == 0 && p->row_count == p->n1 && !(p->comm && p->comm->world > 1), GP_E_SHAPE,
             "kernel product: a row-sharded plan is not available");
  p->backend = GP_BACKEND_PRODUCT;
  p->rows_pad = cdiv(p->row_count, 2 * TILE_I) * 2 * TILE_I;
  p->ntile_i = p->rows_pad / TILE_I;
  p->ntile_j = cdiv(p->n2, TILE_J);
  int dp = 0, kp = 0;
  bool all_tc = true;
  float S = 1.f;
  for (int f = 0; f < nf; ++f) {
    const gp_plan* q = p->factors[f];
    GP_REQUIRE(q && q != p && q->data_set && q->hypers_set, GP_E_STATE, "kernel product: every factor needs set_data + set_hypers");
    GP_REQUIRE(q->backend == GP_BACKEND_TCGEN05 || q->backend == GP_BACKEND_SIMT, GP_E_SHAPE,
               "kernel product: a factor must be a plain kernel plan (not SKI, not a sum, not a product, not multitask, not derivative)");
    GP_CHECK(refuse_settings(q, CALL_PRODUCT_FACTOR_REFRESH));
    GP_CHECK(refuse_compact(q, "a kernel product's factor"));
    GP_REQUIRE(q->row_begin == 0 && q->row_count == q->n1 && !(q->comm && q->comm->world > 1), GP_E_SHAPE,
               "kernel product: a row-sharded factor is not available");
    GP_REQUIRE(q->n1 == p->n1 && q->n2 == p->n2 && q->same == p->same, GP_E_SHAPE,
               "kernel product: factor shape %lld x %lld differs from the product's %lld x %lld", (long long)q->n1, (long long)q->n2,
               (long long)p->n1, (long long)p->n2);
    GP_REQUIRE(q->device == p->device && q->stream == p->stream, GP_E_STATE, "kernel product: factors must live on the product's device and stream");
    GP_REQUIRE(q->rows_pad == p->rows_pad, GP_E_STATE, "kernel product: row padding mismatch");
    dp += q->DP;
    kp += q->KP;
    all_tc = all_tc && q->backend == GP_BACKEND_TCGEN05;
    S *= q->outputscale;
    p->fac_gen[f] = q->pack_gen;
  }
  p->prod_tc = nf == 2 && all_tc && kp <= KP_MAX;
  GP_REQUIRE(p->prod_tc || dp <= 128, GP_E_SHAPE, "kernel product: total padded input width %d > 128 is not supported", dp);
  p->DP = dp;
  p->KP = kp;
  p->outputscale = S;   // the finish kernels scale the unscaled product by S
  choose_splits(p, p->prod_tc);   // for the product's own unit cost, not inherited from a factor
  p->nparts = p->nsplit;
  GP_CHECK(p->mean.ensure(sizeof(int) * 4));
  p->xbad = p->mean.as<int>();
  product_or_flags_kernel<<<1, 1, 0, p->stream>>>(p->factors[0]->xbad, p->factors[1]->xbad, nf > 2 ? p->factors[2]->xbad : nullptr,
                                                  nf > 3 ? p->factors[3]->xbad : nullptr, p->xbad);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  if (p->prod_tc) GP_CHECK(p->Vtiles.ensure(sizeof(float) * p->ntile_j * V_TILE_FLOATS));
  return GP_OK;
}

int product_refresh(gp_plan* p) {
  GP_REQUIRE(p->factors.size() >= 2, GP_E_STATE, "kernel product: no factors set (gp_plan_set_product)");
  for (size_t f = 0; f < p->factors.size(); ++f)
    if (p->factors[f]->pack_gen != p->fac_gen[f]) return product_pack(p);
  return GP_OK;
}

// the tensor-core kernel reads the plan's packed V tiles (pack_v_tiles by the caller), the CUDA-core kernel the fp32 rows V16
int product_kmv_launch(gp_plan* p, const float* V16, const int* done_flag) {
  GP_CHECK(product_refresh(p));
  if (p->prod_tc) return product_tc_launch(p, done_flag);
  GP_REQUIRE(V16 != nullptr, GP_E_STATE, "kernel product: fp32 rows of V needed for the CUDA-core kernel");
  const ProdFactors pf = prod_factors(p);
  dim3 grid((unsigned)cdiv(p->row_count, SIMT_TI), (unsigned)p->nsplit);
  const int64_t cps = p->tiles_per_split * SIMT_TJ;
#define GP_PROD_SIMT_CASE(D)                                                                                                      \
  case D:                                                                                                                         \
    product_simt_kernel<D><<<grid, SIMT_TI, 0, p->stream>>>(pf, V16, p->partial.as<float>(), p->row_count, p->n2, p->rows_pad, cps, \
                                                            p->same ? 1 : 0, p->row_begin, done_flag);                            \
    break;
  switch (round_dpt(p->DP)) {
    GP_PROD_SIMT_CASE(8) GP_PROD_SIMT_CASE(12) GP_PROD_SIMT_CASE(16) GP_PROD_SIMT_CASE(24) GP_PROD_SIMT_CASE(32)
    GP_PROD_SIMT_CASE(48) GP_PROD_SIMT_CASE(64) GP_PROD_SIMT_CASE(96) GP_PROD_SIMT_CASE(128)
  }
#undef GP_PROD_SIMT_CASE
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// rows of the product: factor 0 writes OUT (its outputscale included), every later factor writes scratch rows that are multiplied
// in; a factor with non-finite inputs returns NaN rows
int product_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "rows of a kernel product: at most 65535 rows per call (m=%lld)", (long long)m);
  GP_CHECK(product_refresh(p));
  GP_CHECK(gp_krows(p->factors[0], idx, m, OUT, ldo));
  GP_CHECK(p->misc.ensure(sizeof(float) * (size_t)m * p->n2));
  for (size_t f = 1; f < p->factors.size(); ++f) {
    GP_CHECK(gp_krows(p->factors[f], idx, m, p->misc.as<float>(), p->n2));
    product_mul_rows_kernel<<<dim3((unsigned)cdiv(p->n2, 256), (unsigned)m), 256, 0, p->stream>>>(p->misc.as<float>(), p->n2, OUT, ldo);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int product_kdiag_cross(gp_plan* p, float* OUT) {
  GP_CHECK(gp_kdiag(p->factors[0], OUT));
  GP_CHECK(p->misc.ensure(sizeof(float) * (size_t)p->n1));
  for (size_t f = 1; f < p->factors.size(); ++f) {
    GP_CHECK(gp_kdiag(p->factors[f], p->misc.as<float>()));
    product_mul_rows_kernel<<<dim3((unsigned)cdiv(p->n1, 256), 1), 256, 0, p->stream>>>(p->misc.as<float>(), p->n1, OUT, p->n1);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int product_bilinear_grad(gp_plan* p, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  GP_CHECK(product_refresh(p));
  GP_REQUIRE(p->DP <= 64, GP_E_SHAPE, "bilinear gradient of a kernel product supports a total padded input width <= 64 (got %d)", p->DP);
  const int DPT = round_dpt(p->DP), nout = 1 + DPT;
  const ProdFactors pf = prod_factors(p);
  dim3 grid;
  int64_t cps;
  bilinear_split(p, p->n2, &grid, &cps);
  const int64_t nblk = (int64_t)grid.x * grid.y;
  GP_CHECK(p->misc.ensure(sizeof(double) * (nblk * nout + nout)));
  GP_CHECK(p->misc2.ensure(sizeof(float) * p->row_count * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * p->n2 * TP));
  double* gout = p->misc.as<double>();
  double* gsum = gout + nblk * nout;
  std::vector<double> total(nout, 0.0), h(nout);
  for (int c0 = 0; c0 < s; c0 += TP) {
    const int tc = std::min(TP, s - c0);
    GP_CHECK(to_v16(p, Lf + c0, ldl, tc, p->row_count, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, Rt + c0, ldr, tc, p->n2, p->misc3.as<float>()));
#define GP_PROD_BL_CASE(D)                                                                                                          \
  case D:                                                                                                                           \
    product_bilinear_kernel<D><<<grid, SIMT_TI, 0, p->stream>>>(pf, p->misc2.as<float>(), p->misc3.as<float>(), p->row_count, p->n2, \
                                                                cps, p->same ? 1 : 0, p->row_begin, gout);                          \
    break;
    switch (DPT) { GP_PROD_BL_CASE(8) GP_PROD_BL_CASE(12) GP_PROD_BL_CASE(16) GP_PROD_BL_CASE(24) GP_PROD_BL_CASE(32) GP_PROD_BL_CASE(48) GP_PROD_BL_CASE(64) }
#undef GP_PROD_BL_CASE
    p->launches++;
    GP_CUDA(cudaGetLastError());
    GP_CHECK(sum_partials_double(p, gout, nblk, nout, nout, gsum));
    GP_CUDA(cudaMemcpyAsync(h.data(), gsum, sizeof(double) * nout, cudaMemcpyDeviceToHost, p->stream));
    GP_CUDA(cudaStreamSynchronize(p->stream));
    for (int o = 0; o < nout; ++o) total[o] += h[o];
  }
  // dF/dS = sum w prod k ; d/dl_f: S times the factor's column sums over its lengthscale(s)
  *grad_os = total[0];
  int off = 1, g = 0;
  for (const gp_plan* q : p->factors) {
    if (q->ls.size() > 1) {
      for (int c = 0; c < q->d; ++c) grad_ls[g++] = (double)p->outputscale * total[off + c] / (double)q->ls[c];
    } else {
      double sum = 0.0;
      for (int c = 0; c < q->DP; ++c) sum += total[off + c];
      grad_ls[g++] = (double)p->outputscale * sum / (double)q->ls[0];
    }
    off += q->DP;
  }
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_product(gp_plan* p, gp_plan* const* factors, int n_factors) {
  GP_REQUIRE(p && p->data_set, GP_E_STATE, "kernel product: call gp_plan_set_data on the product first");
  GP_REQUIRE(p->ski == nullptr, GP_E_STATE, "a SKI plan cannot become a kernel product");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel-sum plan cannot become a kernel product");
  GP_CHECK(refuse_settings(p, CALL_SET_PRODUCT));
  GP_CHECK(refuse_compact(p, "gp_plan_set_product"));
  GP_CUDA(cudaSetDevice(p->device));
  if (factors == nullptr || n_factors == 0) {   // back to a plain plan
    if (p->backend_req != GP_BACKEND_PRODUCT) return GP_OK;
    p->factors.clear();
    p->prod_tc = false;
    p->backend_req = GP_BACKEND_AUTO;
    p->backend = GP_BACKEND_SIMT;
    return p->hypers_set ? pack_inputs(p) : GP_OK;
  }
  GP_REQUIRE(n_factors >= 2 && n_factors <= 4, GP_E_SHAPE, "a kernel product takes 2 to 4 factors (got %d)", n_factors);
  for (int f = 0; f < n_factors; ++f) {
    GP_REQUIRE(factors[f] != nullptr && factors[f] != p, GP_E_STATE, "kernel product: factor %d is null or the product itself", f);
    GP_CHECK(refuse_settings(factors[f], CALL_PRODUCT_FACTOR));
    GP_CHECK(refuse_compact(factors[f], "gp_plan_set_product (a factor)"));
  }
  p->factors.assign(factors, factors + n_factors);
  p->backend_req = GP_BACKEND_PRODUCT;
  p->backend = GP_BACKEND_PRODUCT;
  return p->hypers_set ? product_pack(p) : GP_OK;   // without hyper-parameters (the noise) yet: packed by gp_plan_set_hypers
}
