// additive.cu -- additive GPs: a sum of D univariate kernels and their interaction terms up to degree M (Duvenaud et al.; the
// reference builds them as ScaleKernel(RBFKernel(batch_shape=[D], ard_num_dims=1)) over X.mT.unsqueeze(-1), then .sum(dim=-3) or
// utils/sum_interaction_terms.py, both dense).  Per pair, with c_i = s_i k_i(x_i, x'_i) over column i of X:
//
//   K(x, x') = sum_{m=1}^{M} e_m(c_1, .., c_D),   e_m the elementary symmetric polynomial of degree m.
//
// The reference forms sum_m e_m by Newton-Girard from the power sums p_k = sum_i c_i^k, whose alternating signs cancel badly in
// fp32.  Here e is built by the positive recurrence e_m <- e_m + c_i e_{m-1} (m = M .. 1, e_0 = 1): M FMAs per component on
// non-negative terms, so every partial sum is a sum of positive products and the relative error of K stays O(D M u).  The square
// diagonal is the constant sum_m e_m(s_1 .. s_D).
//
// The plan is a plain SIMT plan over d = D columns with D ARD lengthscales: pack.cu's Z = (x - mean) sqrt(C) / l_i already holds
// every component's packed coordinate, so a_i = -0.5 (z_i - z'_i)^2 and k_i = poly(rho_i) 2^{e_i} (cov_poly_exp).  The difference
// of a row with itself is exactly 0, so the diagonal of a square operator gets a_i = 0 without a test.
//
//   additive_kmv_kernel       K.V on CUDA cores, partial[split][row][16] like kmv_simt_kernel (finish kernels: scale 1).  D ex2 per
//                             pair make it MUFU-bound, which tensor cores would not relieve.  M <= 4 compiled as template cases,
//                             5 <= M <= 8 through the generic recurrence of ADD_MMAX degrees.
//   additive_krows_kernel / additive_kdiag_cross_kernel   rows and the diagonal of a cross operator
//   additive_bilinear_kernel  one pass over the pairs for the D lengthscale and D component-scale gradients
#include <math.h>
#include <string.h>

#include <algorithm>

#include "gp_common.cuh"

namespace gp {

constexpr int ADD_G = 8;   // components whose gradients one CTA of the bilinear kernel accumulates (blockIdx.z = group)

AddHyp additive_hyp(const gp_plan* p) {
  AddHyp h;
  memset(&h, 0, sizeof(h));
  h.D = (int)p->add_s.size();
  h.M = p->add_M;
  for (int c = 0; c < h.D; ++c) h.s[c] = p->add_s[c];
  h.rbf = p->kind == GP_RBF;
  h.cp = cov_poly_of(p->kind);
  return h;
}

// ---- K.V: grid (row blocks, nsplit); 128 threads, one output row each -------------------------------------------------------
// (a minimum of 4 CTAs per SM leaves up to 128 registers; without it ptxas spills 8 bytes in some instantiations at 56-72)
template <bool RBF, int MT, int DP>
__global__ void __launch_bounds__(SIMT_TI, 4)
additive_kmv_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ V16,
                    float* __restrict__ partial, int64_t n1, int64_t n2, int64_t rows_pad, int64_t cols_per_split, const AddHyp h,
                    const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  __shared__ __align__(16) float zj[SIMT_TJ][DP];
  __shared__ __align__(16) float vj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int split = blockIdx.y;
  const int64_t j_begin = (int64_t)split * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const int M = MT < ADD_MMAX ? MT : h.M;
  float zi[DP];
  const bool rv = i < n1;
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? Z1[i * DP + c] : 0.f;
  float acc[TP];
#pragma unroll
  for (int c = 0; c < TP; ++c) acc[c] = 0.f;

  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < SIMT_TJ * DP; e += SIMT_TI) (&zj[0][0])[e] = (e / DP < nj) ? Z2[j0 * DP + e] : 0.f;
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) (&vj[0][0])[e] = (e / TP < nj) ? V16[j0 * TP + e] : 0.f;
    __syncthreads();
#pragma unroll 2
    for (int jj = 0; jj < SIMT_TJ; ++jj) {
      float e[MT + 1];
      e[0] = 1.f;
#pragma unroll
      for (int m = 1; m <= MT; ++m) e[m] = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c)
        if (c < h.D) esym_push<MT>(e, h.s[c] * add_comp<RBF>(h.cp, zi[c] - zj[jj][c]), M);
      const float k = esym_total<MT>(e, M);
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

// ---- rows: OUT[r][j] = K(x1[idx[r]], x2[j]); NaN rows for an index out of range or non-finite inputs (as krows_kernel) ------
template <bool RBF>
__global__ void additive_krows_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int DP, const int64_t* __restrict__ idx,
                                      int64_t n1_local, int64_t n2, const AddHyp h, float* __restrict__ OUT, int64_t ldo,
                                      const int* __restrict__ xbad) {
  __shared__ float zi[ADD_DMAX];
  const int64_t r = blockIdx.y;
  const int64_t i = idx[r];
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 0 || i >= n1_local || *xbad) {
    if (j < n2) OUT[r * ldo + j] = __int_as_float(0x7fc00000);
    return;
  }
  for (int c = threadIdx.x; c < h.D; c += blockDim.x) zi[c] = Z1[i * DP + c];
  __syncthreads();
  if (j >= n2) return;
  OUT[r * ldo + j] = add_pair<RBF>(h, zi, Z2 + j * DP);
}

// diagonal of a cross operator (n1 == n2): OUT[i] = K(x1_i, x2_i)
template <bool RBF>
__global__ void additive_kdiag_cross_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int DP, int64_t n, const AddHyp h,
                                            float* __restrict__ OUT, const int* __restrict__ xbad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  OUT[i] = *xbad ? __int_as_float(0x7fc00000) : add_pair<RBF>(h, Z1 + i * DP, Z2 + i * DP);
}

// diagonal of a square operator: the constant sum_m e_m(s), NaN for non-finite inputs
__global__ void additive_fill_kernel(float* __restrict__ OUT, int64_t n, float v, const int* __restrict__ xbad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) OUT[i] = *xbad ? __int_as_float(0x7fc00000) : v;
}

// ---- bilinear derivative: grid (row blocks, column splits, component groups of ADD_G) ---------------------------------------
// With w_ij = L_i . R_j, dK/dc_q = sum_{m=1}^{M} e_{m-1}(c without c_q) and l dk_q/dl = gpoly_q 2^{e_q} (dcov_poly_exp):
//   gout[block][g * 2G + q]      = sum_ij w_ij dK/dc_q s_q gpoly_q 2^{e_q}   (host: / l_q -> dF/dl_q)
//   gout[block][g * 2G + G + q]  = sum_ij w_ij dK/dc_q k_q                   (dF/ds_q)
// for the components q of group g = blockIdx.z.  e is formed in fp64 and the leave-one-out values by e^{-q}_j = e_j - c_q e^{-q}_{j-1}:
// dK/dc_q >= 1 (its e_0 term), so the subtraction's absolute error, fp64 rounding times sum_j e_j, is small against it.
template <bool RBF, int DP>
__global__ void __launch_bounds__(SIMT_TI)
additive_bilinear_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ L16,
                         const float* __restrict__ R16, int64_t n1, int64_t n2, int64_t cols_per_split, const AddHyp h,
                         double* __restrict__ gout, int gstride) {
  __shared__ __align__(16) float zj[SIMT_TJ][DP];
  __shared__ __align__(16) float rj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int grp = blockIdx.z;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int64_t j_begin = (int64_t)blockIdx.y * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const bool rv = i < n1;
  float zi[DP], li[TP];
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? Z1[i * DP + c] : 0.f;
#pragma unroll
  for (int c = 0; c < TP; ++c) li[c] = rv ? L16[i * TP + c] : 0.f;
  float gl[ADD_G], gs[ADD_G];
#pragma unroll
  for (int q = 0; q < ADD_G; ++q) gl[q] = gs[q] = 0.f;
  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < SIMT_TJ * DP; e += SIMT_TI) (&zj[0][0])[e] = (e / DP < nj) ? Z2[j0 * DP + e] : 0.f;
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) (&rj[0][0])[e] = (e / TP < nj) ? R16[j0 * TP + e] : 0.f;
    __syncthreads();
    for (int jj = 0; jj < nj; ++jj) {
      float w = 0.f;
#pragma unroll
      for (int c = 0; c < TP; ++c) w = fmaf(li[c], rj[jj][c], w);
      double e[ADD_MMAX + 1];
      e[0] = 1.0;
#pragma unroll
      for (int m = 1; m <= ADD_MMAX; ++m) e[m] = 0.0;
      float cq[ADD_G], kq[ADD_G], gq[ADD_G];
#pragma unroll
      for (int q = 0; q < ADD_G; ++q) cq[q] = kq[q] = gq[q] = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        if (c < h.D) {
          const float df = zi[c] - zj[jj][c];
          float pl, gp, ex;
          dcov_poly_exp(RBF, h.cp, -0.5f * (df * df), &pl, &gp, &ex);
          const float E = ex2_approx(ex);
          const float k = pl * E;
          const float ci = h.s[c] * k;
          esym_push<ADD_MMAX>(e, (double)ci, h.M);
          if (c / ADD_G == grp) {   // c % ADD_G is a compile-time index: the group's values stay in registers
            cq[c % ADD_G] = ci;
            kq[c % ADD_G] = k;
            gq[c % ADD_G] = h.s[c] * gp * E;
          }
        }
      }
#pragma unroll
      for (int q = 0; q < ADD_G; ++q) {
        double lo = 1.0, dk = 1.0;   // e^{-q}_0 and the running sum_{m=1}^{M} e^{-q}_{m-1}
#pragma unroll
        for (int m = 1; m < ADD_MMAX; ++m) {
          if (m < h.M) {
            lo = e[m] - (double)cq[q] * lo;
            dk += lo;
          }
        }
        const float wd = w * (float)dk;
        gl[q] = fmaf(wd, gq[q], gl[q]);
        gs[q] = fmaf(wd, kq[q], gs[q]);
      }
    }
  }
  __shared__ double red[SIMT_TI];
  const int64_t blk = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
#pragma unroll
  for (int o = 0; o < 2 * ADD_G; ++o) {
    __syncthreads();
    red[tid] = (double)(o < ADD_G ? gl[o] : gs[o - ADD_G]);
    __syncthreads();
    for (int sft = SIMT_TI / 2; sft > 0; sft >>= 1) {
      if (tid < sft) red[tid] += red[tid + sft];
      __syncthreads();
    }
    if (tid == 0) gout[blk * gstride + grp * 2 * ADD_G + o] = red[0];
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------------------
int additive_pack(gp_plan* p) {
  const int D = (int)p->add_s.size();
  GP_REQUIRE(p->d == D, GP_E_SHAPE, "additive plan: %d component scales for data of d=%d columns (one component per column)", D, p->d);
  GP_REQUIRE((int)p->ls.size() == D, GP_E_SHAPE,
             "additive plan: gp_plan_set_hypers must give one lengthscale per component (%d), got %d", D, (int)p->ls.size());
  GP_REQUIRE(p->backend == GP_BACKEND_SIMT, GP_E_STATE, "additive plan: the packing did not select the CUDA-core layout");
  // sum_{m=1}^{M} e_m(s) in fp64 by the same recurrence
  double e[ADD_MMAX + 1] = {1.0};
  for (int c = 0; c < D; ++c)
    for (int m = p->add_M; m >= 1; --m) e[m] += (double)p->add_s[c] * e[m - 1];
  double k = 0.0;
  for (int m = 1; m <= p->add_M; ++m) k += e[m];
  p->add_diag = k;
  return GP_OK;
}

static const float* add_z1(const gp_plan* p) { return p->same ? p->Z2.as<float>() + p->row_begin * p->DP : p->Z1.as<float>(); }

template <bool RBF, int MT>
static int add_kmv_dp(gp_plan* p, const AddHyp& h, const float* V16, const int* done_flag) {
  dim3 grid((unsigned)cdiv(p->row_count, SIMT_TI), (unsigned)p->nsplit);
  const int64_t cps = p->tiles_per_split * SIMT_TJ;
#define GP_ADD_CASE(DPV)                                                                                                           \
  case DPV:                                                                                                                        \
    additive_kmv_kernel<RBF, MT, DPV><<<grid, SIMT_TI, 0, p->stream>>>(add_z1(p), p->Z2.as<float>(), V16, partial_ptr(p), p->row_count, \
                                                                       p->n2, p->rows_pad, cps, h, done_flag);                     \
    break;
  switch (p->DP) {
    GP_ADD_CASE(4) GP_ADD_CASE(8) GP_ADD_CASE(12) GP_ADD_CASE(16) GP_ADD_CASE(24) GP_ADD_CASE(32)
    default:
      set_error("additive plan: unsupported padded width %d", p->DP);
      return GP_E_SHAPE;
  }
#undef GP_ADD_CASE
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

template <bool RBF>
static int add_kmv_m(gp_plan* p, const AddHyp& h, const float* V16, const int* done_flag) {
  switch (h.M) {
    case 1: return add_kmv_dp<RBF, 1>(p, h, V16, done_flag);
    case 2: return add_kmv_dp<RBF, 2>(p, h, V16, done_flag);
    case 3: return add_kmv_dp<RBF, 3>(p, h, V16, done_flag);
    case 4: return add_kmv_dp<RBF, 4>(p, h, V16, done_flag);
    default: return add_kmv_dp<RBF, ADD_MMAX>(p, h, V16, done_flag);
  }
}

int additive_kmv_launch(gp_plan* p, const float* V16, const int* done_flag) {
  GP_REQUIRE(V16 != nullptr, GP_E_STATE, "additive plan: fp32 rows of V needed");
  const AddHyp h = additive_hyp(p);
  return h.rbf ? add_kmv_m<true>(p, h, V16, done_flag) : add_kmv_m<false>(p, h, V16, done_flag);
}

int additive_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "rows of an additive plan: at most 65535 rows per call (m=%lld)", (long long)m);
  const AddHyp h = additive_hyp(p);
  dim3 grid((unsigned)cdiv(p->n2, 256), (unsigned)m);
  if (h.rbf) additive_krows_kernel<true><<<grid, 256, 0, p->stream>>>(add_z1(p), p->Z2.as<float>(), p->DP, idx, p->row_count, p->n2, h, OUT, ldo, p->xbad);
  else additive_krows_kernel<false><<<grid, 256, 0, p->stream>>>(add_z1(p), p->Z2.as<float>(), p->DP, idx, p->row_count, p->n2, h, OUT, ldo, p->xbad);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int additive_kdiag(gp_plan* p, float* OUT) {
  if (p->same) {
    additive_fill_kernel<<<(unsigned)cdiv(p->row_count, 256), 256, 0, p->stream>>>(OUT, p->row_count, (float)p->add_diag, p->xbad);
  } else {
    GP_REQUIRE(p->n1 == p->n2, GP_E_SHAPE, "diagonal of a %lld x %lld cross-covariance is undefined (kernel(x1, x2, diag=True) needs equal sizes)",
               (long long)p->n1, (long long)p->n2);
    const AddHyp h = additive_hyp(p);
    const unsigned g = (unsigned)cdiv(p->n1, 256);
    if (h.rbf) additive_kdiag_cross_kernel<true><<<g, 256, 0, p->stream>>>(p->Z1.as<float>(), p->Z2.as<float>(), p->DP, p->n1, h, OUT, p->xbad);
    else additive_kdiag_cross_kernel<false><<<g, 256, 0, p->stream>>>(p->Z1.as<float>(), p->Z2.as<float>(), p->DP, p->n1, h, OUT, p->xbad);
  }
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

template <bool RBF>
static int add_bilinear_launch(gp_plan* p, const AddHyp& h, dim3 grid, int64_t cps, const float* L16, const float* R16, double* gout, int gstride) {
#define GP_ADD_BL_CASE(DPV)                                                                                                      \
  case DPV:                                                                                                                      \
    additive_bilinear_kernel<RBF, DPV><<<grid, SIMT_TI, 0, p->stream>>>(add_z1(p), p->Z2.as<float>(), L16, R16, p->row_count, p->n2, \
                                                                        cps, h, gout, gstride);                                  \
    break;
  switch (p->DP) {
    GP_ADD_BL_CASE(4) GP_ADD_BL_CASE(8) GP_ADD_BL_CASE(12) GP_ADD_BL_CASE(16) GP_ADD_BL_CASE(24) GP_ADD_BL_CASE(32)
    default:
      set_error("additive plan: unsupported padded width %d", p->DP);
      return GP_E_SHAPE;
  }
#undef GP_ADD_BL_CASE
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// grad_ls[c] = dF/dl_c, grad_os[c] = dF/ds_c for the D components (grad_os holds D doubles on an additive plan)
int additive_bilinear_grad(gp_plan* p, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  const AddHyp h = additive_hyp(p);
  const int ngrp = (int)cdiv(h.D, ADD_G), nout = ngrp * 2 * ADD_G;
  dim3 grid;
  int64_t cps;
  bilinear_split(p, p->n2, &grid, &cps);
  const int64_t nblk = (int64_t)grid.x * grid.y;
  grid.z = (unsigned)ngrp;
  GP_CHECK(p->misc.ensure(sizeof(double) * (nblk * nout + nout)));
  GP_CHECK(p->misc2.ensure(sizeof(float) * p->row_count * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * p->n2 * TP));
  double* gout = p->misc.as<double>();
  double* gsum = gout + nblk * nout;
  std::vector<double> total(nout, 0.0), hbuf(nout);
  for (int c0 = 0; c0 < s; c0 += TP) {
    const int tc = std::min(TP, s - c0);
    GP_CHECK(to_v16(p, Lf + c0, ldl, tc, p->row_count, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, Rt + c0, ldr, tc, p->n2, p->misc3.as<float>()));
    GP_CHECK(h.rbf ? add_bilinear_launch<true>(p, h, grid, cps, p->misc2.as<float>(), p->misc3.as<float>(), gout, nout)
                   : add_bilinear_launch<false>(p, h, grid, cps, p->misc2.as<float>(), p->misc3.as<float>(), gout, nout));
    GP_CHECK(sum_partials_double(p, gout, nblk, nout, nout, gsum));
    GP_CUDA(cudaMemcpyAsync(hbuf.data(), gsum, sizeof(double) * nout, cudaMemcpyDeviceToHost, p->stream));
    GP_CUDA(cudaStreamSynchronize(p->stream));
    for (int o = 0; o < nout; ++o) total[o] += hbuf[o];
  }
  for (int c = 0; c < h.D; ++c) {
    const int base = (c / ADD_G) * 2 * ADD_G + c % ADD_G;
    grad_ls[c] = total[base] / (double)p->ls[c];
    grad_os[c] = total[base + ADD_G];
  }
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_additive(gp_plan* p, int max_degree, const float* comp_scale, int n_comp) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  if (comp_scale == nullptr || n_comp == 0) {   // back to a plain plan
    if (p->add_M == 0) return GP_OK;
    p->add_M = 0;
    p->add_s.clear();
    return (p->data_set && p->hypers_set) ? pack_inputs(p) : GP_OK;
  }
  GP_REQUIRE(p->data_set, GP_E_STATE, "additive plan: call gp_plan_set_data first");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "a SKI plan cannot become an additive plan");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel-sum plan cannot become an additive plan");
  GP_CHECK(refuse_settings(p, CALL_SET_ADDITIVE));
  GP_CHECK(refuse_compact(p, "gp_plan_set_additive"));
  GP_REQUIRE(p->row_begin == 0 && p->row_count == p->n1 && !(p->comm && p->comm->world > 1), GP_E_SHAPE,
             "an additive plan is not available on a row-sharded plan");
  GP_REQUIRE(n_comp >= 1 && n_comp <= ADD_DMAX, GP_E_SHAPE, "an additive plan takes 1 to %d components (got %d)", ADD_DMAX, n_comp);
  GP_REQUIRE(n_comp == p->d, GP_E_SHAPE, "additive plan: %d components for data of d=%d columns (one component per column)", n_comp, p->d);
  GP_REQUIRE(max_degree >= 1 && max_degree <= ADD_MMAX, GP_E_SHAPE, "additive plan: max_degree=%d not in [1, %d]", max_degree, ADD_MMAX);
  for (int c = 0; c < n_comp; ++c)
    GP_REQUIRE(comp_scale[c] > 0.f && isfinite(comp_scale[c]), GP_E_SHAPE, "additive plan: component scale[%d]=%g must be positive", c,
               comp_scale[c]);
  GP_CUDA(cudaSetDevice(p->device));
  p->add_M = std::min(max_degree, n_comp);   // e_m = 0 for m > D
  p->add_s.assign(comp_scale, comp_scale + n_comp);
  return p->hypers_set ? pack_inputs(p) : GP_OK;
}
