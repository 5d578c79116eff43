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
//   AddEntry                  rows and the diagonal of a cross operator on the shared row kernels (simt_pass.cuh)
//   additive_bilinear_kernel  one pass over the pairs for the D lengthscale and D component-scale gradients
#include <math.h>
#include <string.h>

#include <algorithm>

#include "gp_common.cuh"
#include "simt_pass.cuh"

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

// ---- rows and the diagonal of a cross operator: K(x1_i, x2_j) from two packed rows -----------------------------------------
template <bool RBF>
struct AddEntry {
  static constexpr bool XBAD = true;
  const float* Z1;
  const float* Z2;
  int64_t ld;   // DP (64-bit: ptxas then keeps both kernels at or below the registers of their former per-family copies)
  AddHyp h;
  __host__ __device__ int width() const { return h.D; }
  __device__ __forceinline__ float entry(const float* za, const float* zb, int64_t, int64_t) const { return add_pair<RBF>(h, za, zb); }
};

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
    block_sum_store<SIMT_TI>(red, (double)(o < ADD_G ? gl[o] : gs[o - ADD_G]), gout + blk * gstride + grp * 2 * ADD_G + o);
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
  const bool ok = with_width<4, 8, 12, 16, 24, 32>(p->DP, [&](auto w) {
    additive_kmv_kernel<RBF, MT, decltype(w)::value><<<grid, SIMT_TI, 0, p->stream>>>(add_z1(p), p->Z2.as<float>(), V16, partial_ptr(p),
                                                                                      p->row_count, p->n2, p->rows_pad, cps, h, done_flag);
  });
  if (!ok) {
    set_error("additive plan: unsupported padded width %d", p->DP);
    return GP_E_SHAPE;
  }
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
  if (h.rbf) return launch_krows(p, AddEntry<true>{add_z1(p), p->Z2.as<float>(), p->DP, h}, idx, m, OUT, ldo);
  return launch_krows(p, AddEntry<false>{add_z1(p), p->Z2.as<float>(), p->DP, h}, idx, m, OUT, ldo);
}

// square: the constant sum_m e_m(s); cross: per pair.  NaN for non-finite inputs
int additive_kdiag(gp_plan* p, float* OUT) {
  const AddHyp h = additive_hyp(p);
  const float v = (float)p->add_diag;
  if (h.rbf) return launch_kdiag(p, OUT, &v, AddEntry<true>{p->Z1.as<float>(), p->Z2.as<float>(), p->DP, h});
  return launch_kdiag(p, OUT, &v, AddEntry<false>{p->Z1.as<float>(), p->Z2.as<float>(), p->DP, h});
}

template <bool RBF>
static int add_bilinear_launch(gp_plan* p, const AddHyp& h, dim3 grid, int64_t cps, const float* L16, const float* R16, double* gout, int gstride) {
  const bool ok = with_width<4, 8, 12, 16, 24, 32>(p->DP, [&](auto w) {
    additive_bilinear_kernel<RBF, decltype(w)::value><<<grid, SIMT_TI, 0, p->stream>>>(add_z1(p), p->Z2.as<float>(), L16, R16,
                                                                                       p->row_count, p->n2, cps, h, gout, gstride);
  });
  if (!ok) {
    set_error("additive plan: unsupported padded width %d", p->DP);
    return GP_E_SHAPE;
  }
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
  std::vector<double> total;
  GP_CHECK(bilinear_sweep(p, Lf, ldl, Rt, ldr, s, p->row_count, nblk, nout, [&](const float* L16, const float* R16, double* gout) -> int {
    return h.rbf ? add_bilinear_launch<true>(p, h, grid, cps, L16, R16, gout, nout) : add_bilinear_launch<false>(p, h, grid, cps, L16, R16, gout, nout);
  }, total));
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
