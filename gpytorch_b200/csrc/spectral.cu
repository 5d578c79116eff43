// spectral.cu -- spectral mixture (SM) kernels (Wilson & Adams 2013; the reference's kernels/spectral_mixture_kernel.py, which
// builds dense [Q, n, m, d] temporaries).  For tau = x - x' over d dimensions, Q components with weights w_q, means mu_qd and
// scales v_qd, and the plan's outputscale S:
//
//   K(x, x') = S prod_d sum_q w_q exp(-2 pi^2 v_qd^2 tau_d^2) cos(2 pi mu_qd tau_d)
//
// -- the reference sums the components of every dimension before it takes the product over the dimensions; for d = 1 this is the
// familiar S sum_q w_q exp(..) cos(..).  The square diagonal is the constant S (sum_q w_q)^d.
//
// Packing (spectral_pack).  One row of W = pad4(d + Q d) floats per point: the fp32 inputs x_c themselves, then per (q, c) the
// reduced phase p_qc(x) = mu_qc x_c - floor(mu_qc x_c + 1/2) in [-1/2, 1/2), formed in fp64 from the fp32 x and mu (their product
// is exact in fp64) and rounded once to fp32.  Then cos(2 pi mu tau) = cos(2 pi (p - p')) for the exact inputs, and the argument
// of the cosine stays in (-2 pi, 2 pi) whatever |x|: the reference's fp32 argument 2 pi (mu x - mu x') carries an absolute error
// of order u |mu x|, which reaches 1e-2 rad at x ~ 1e5.  tau_c = x_c - x'_c is formed in fp32 from the raw inputs, so its error is
// relative (u |tau|) and the exponent's error does not grow with |x| either (mean-centring would add u |x - mean| to each side).
//
//   spectral_kmv_kernel        K.V on CUDA cores into partial[split][row][16] (the finish kernels apply S).  Per pair: d
//                              differences, Q d exponents (one FMUL each, beta_qd = -2 pi^2 v_qd^2 log2 e in the argument struct),
//                              Q d ex2 and Q d cos of the reduced phase difference, Q d FMAs into the d mixtures, d - 1 products and
//                              16 FMAs.  2 Q d MUFU operations per pair make it bound by the special-function unit; tensor cores
//                              would not change that count.  Template cases: d exact (1 .. 8), Q up to QM in {1, 4, min(16, 32/d)}.
//   SmEntry                    rows and the diagonal of a cross operator (runtime Q, d) on the shared row kernels (simt_pass.cuh)
//   spectral_bilinear_kernel   one pass over the pairs for the Q (1 + 2d) parameter gradients and dF/dS; fp64 accumulators,
//                              components in groups of sm_gq(d) on blockIdx.z, a fixed-order block reduction (no atomics)
#include <math.h>
#include <string.h>

#include <algorithm>

#include "gp_common.cuh"
#include "simt_pass.cuh"

namespace gp {

constexpr float SM_TWO_PI = 6.2831853071795865f;

// components whose gradients one CTA of the bilinear kernel accumulates: (1 + 2d) fp64 sums each, at most 17 such sums per thread,
// which with the dF/dS sum makes at most 18 accumulators (d = 8)
__host__ __device__ constexpr int sm_gq(int D) { return (1 + 2 * D) * 4 <= 17 ? 4 : ((1 + 2 * D) * 2 <= 17 ? 2 : 1); }
// packed row width of (D, Q)
__host__ __device__ constexpr int sm_width(int D, int Q) { return ((D + Q * D) + 3) / 4 * 4; }

SmHyp spectral_hyp(const gp_plan* p) {
  SmHyp h;
  memset(&h, 0, sizeof(h));
  h.Q = p->sm_Q;
  h.d = p->d;
  h.S = p->outputscale;
  for (int q = 0; q < h.Q; ++q) h.w[q] = p->sm_w[q];
  for (int k = 0; k < h.Q * h.d; ++k) {
    const double v = p->sm_v[k];
    h.beta[k] = (float)(-2.0 * M_PI * M_PI * v * v * 1.4426950408889634);
  }
  return h;
}

// ---- packing: one thread per point ---------------------------------------------------------------------------------------------
__global__ void spectral_pack_kernel(const float* __restrict__ X, int64_t n, int64_t ld, int d, int Q, int W,
                                     const float* __restrict__ mu, float* __restrict__ P, int* __restrict__ xbad) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  float* row = P + r * W;
  bool bad = false;
  for (int c = 0; c < d; ++c) {
    const float x = X[r * ld + c];
    bad |= !(fabsf(x) <= 3.402823466e38f);
    row[c] = x;
  }
  for (int k = 0; k < Q * d; ++k) {
    const double t = (double)mu[k] * (double)X[r * ld + k % d];   // exact: 24 + 24 significant bits
    row[d + k] = (float)(t - floor(t + 0.5));
  }
  for (int k = d + Q * d; k < W; ++k) row[k] = 0.f;
  if (bad) *xbad = 1;
}

// ---- K.V: grid (row blocks, nsplit); 128 threads, one output row each -------------------------------------------------------
template <int D, int QM>
__global__ void __launch_bounds__(SIMT_TI, 4)
spectral_kmv_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int W, const float* __restrict__ V16,
                    float* __restrict__ partial, int64_t n1, int64_t n2, int64_t rows_pad, int64_t cols_per_split, const SmHyp h,
                    const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  constexpr int WT = sm_width(D, QM);
  __shared__ __align__(16) float zj[SIMT_TJ][WT];
  __shared__ __align__(16) float vj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int split = blockIdx.y;
  const int64_t j_begin = (int64_t)split * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const int Q = h.Q;
  const bool rv = i < n1;
  float xi[D], pi[QM * D];
#pragma unroll
  for (int c = 0; c < D; ++c) xi[c] = rv ? Z1[i * W + c] : 0.f;
#pragma unroll
  for (int k = 0; k < QM * D; ++k) pi[k] = (rv && k < Q * D) ? Z1[i * W + D + k] : 0.f;
  float acc[TP];
#pragma unroll
  for (int c = 0; c < TP; ++c) acc[c] = 0.f;

  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < SIMT_TJ * W; e += SIMT_TI) {
      const int r = e / W;
      zj[r][e - r * W] = r < nj ? Z2[j0 * W + e] : 0.f;
    }
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) (&vj[0][0])[e] = (e / TP < nj) ? V16[j0 * TP + e] : 0.f;
    __syncthreads();
#pragma unroll 2
    for (int jj = 0; jj < SIMT_TJ; ++jj) {
      float k = 1.f;
#pragma unroll
      for (int c = 0; c < D; ++c) {
        const float t = xi[c] - zj[jj][c];
        const float t2 = t * t;
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < QM; ++q) {
          if (q < Q) {
            const float e = ex2_approx(h.beta[q * D + c] * t2);
            const float cs = __cosf(SM_TWO_PI * (pi[q * D + c] - zj[jj][D + q * D + c]));
            s = fmaf(h.w[q], e * cs, s);
          }
        }
        k *= s;
      }
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

// ---- rows and the diagonal of a cross operator: K(x1_i, x2_j) from two packed rows (runtime Q, d) ---------------------------
struct SmEntry {
  static constexpr bool XBAD = true;
  const float* Z1;
  const float* Z2;
  int ld;   // W
  SmHyp h;
  __host__ __device__ int width() const { return ld; }
  __device__ __forceinline__ float entry(const float* za, const float* zb, int64_t, int64_t) const { return sm_pair(h, za, zb); }
};

// ---- bilinear derivative: grid (row blocks, column splits, component groups of GQ = sm_gq(D)) -------------------------------
// With g = L_i . R_j, the mixtures s_c = sum_q w_q e_qc cos_qc and P_c = prod_{c' != c} s_c' (prefix and suffix products, no
// division), per group g = blockIdx.z and its components q = g GQ + k:
//   out[0]                    = sum g prod_c s_c                          (dF/dS)
//   out[1 + k]                = sum g sum_c P_c e_qc cos_qc               (dF/dw_q / S)
//   out[1 + GQ + k D + c]     = sum g P_c e_qc sin_qc tau_c               (dF/dmu_qc / (-2 pi S w_q))
//   out[1 + GQ + GQ D + k D + c] = sum g P_c e_qc cos_qc tau_c^2          (dF/dv_qc / (-4 pi^2 S w_q v_qc))
// Every pair term is formed in fp32 and added to an fp64 accumulator.
// (with __launch_bounds__(SIMT_TI) ptxas keeps <4, 1> at 80 registers and spills 8 bytes; an explicit cap of 255 does not)
template <int D, int QM>
__global__ void __maxnreg__(255)
spectral_bilinear_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int W, const float* __restrict__ L16,
                         const float* __restrict__ R16, int64_t n1, int64_t n2, int64_t cols_per_split, const SmHyp h,
                         double* __restrict__ gout, int gstride) {
  constexpr int GQ = sm_gq(D);
  constexpr int NO = 1 + GQ * (1 + 2 * D);
  constexpr int WT = sm_width(D, QM);
  __shared__ __align__(16) float zj[SIMT_TJ][WT];
  __shared__ __align__(16) float rj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int grp = blockIdx.z;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int64_t j_begin = (int64_t)blockIdx.y * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const int Q = h.Q;
  const bool rv = i < n1;
  float xi[D], pi[QM * D], li[TP];
#pragma unroll
  for (int c = 0; c < D; ++c) xi[c] = rv ? Z1[i * W + c] : 0.f;
#pragma unroll
  for (int k = 0; k < QM * D; ++k) pi[k] = (rv && k < Q * D) ? Z1[i * W + D + k] : 0.f;
#pragma unroll
  for (int c = 0; c < TP; ++c) li[c] = rv ? L16[i * TP + c] : 0.f;
  double acc[NO];
#pragma unroll
  for (int o = 0; o < NO; ++o) acc[o] = 0.0;
  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < SIMT_TJ * W; e += SIMT_TI) {
      const int r = e / W;
      zj[r][e - r * W] = r < nj ? Z2[j0 * W + e] : 0.f;
    }
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) (&rj[0][0])[e] = (e / TP < nj) ? R16[j0 * TP + e] : 0.f;
    __syncthreads();
    for (int jj = 0; jj < nj; ++jj) {
      float g = 0.f;
#pragma unroll
      for (int c = 0; c < TP; ++c) g = fmaf(li[c], rj[jj][c], g);
      float tau[D], s[D], ge[GQ][D], gc[GQ][D], gs[GQ][D];
#pragma unroll
      for (int k = 0; k < GQ; ++k)
#pragma unroll
        for (int c = 0; c < D; ++c) ge[k][c] = gc[k][c] = gs[k][c] = 0.f;
#pragma unroll
      for (int c = 0; c < D; ++c) {
        tau[c] = xi[c] - zj[jj][c];
        const float t2 = tau[c] * tau[c];
        s[c] = 0.f;
#pragma unroll
        for (int q = 0; q < QM; ++q) {
          if (q < Q) {
            const float e = ex2_approx(h.beta[q * D + c] * t2);
            float sn, cs;
            __sincosf(SM_TWO_PI * (pi[q * D + c] - zj[jj][D + q * D + c]), &sn, &cs);
            s[c] = fmaf(h.w[q], e * cs, s[c]);
            if (q / GQ == grp) {   // q % GQ is a compile-time index: the group's values stay in registers
              ge[q % GQ][c] = e;
              gc[q % GQ][c] = cs;
              gs[q % GQ][c] = sn;
            }
          }
        }
      }
      float pre[D + 1], suf[D + 1];
      pre[0] = suf[D] = 1.f;
#pragma unroll
      for (int c = 0; c < D; ++c) pre[c + 1] = pre[c] * s[c];
#pragma unroll
      for (int c = D - 1; c >= 0; --c) suf[c] = suf[c + 1] * s[c];
      acc[0] += (double)(g * pre[D]);
#pragma unroll
      for (int k = 0; k < GQ; ++k) {
        float dw = 0.f;
#pragma unroll
        for (int c = 0; c < D; ++c) {
          const float gpe = g * (pre[c] * suf[c + 1]) * ge[k][c];
          const float gpc = gpe * gc[k][c];
          dw += gpc;
          acc[1 + GQ + k * D + c] += (double)(gpe * gs[k][c] * tau[c]);
          acc[1 + GQ + GQ * D + k * D + c] += (double)(gpc * (tau[c] * tau[c]));
        }
        acc[1 + k] += (double)dw;
      }
    }
  }
  __shared__ double red[SIMT_TI];
  const int64_t blk = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
#pragma unroll
  for (int o = 0; o < NO; ++o) {
    __syncthreads();
    block_sum_store<SIMT_TI>(red, acc[o], gout + blk * gstride + grp * NO + o);
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------------------
// Q bound of the compiled case that runs Q components of d dimensions
static int sm_qcase(int d, int Q) {
  const int top = std::min(16, 32 / d);
  return Q == 1 ? 1 : (Q <= 4 ? 4 : top);
}

int spectral_pack(gp_plan* p) {
  const int d = p->d, Q = p->sm_Q;
  GP_REQUIRE((int)p->sm_mu.size() == Q * d, GP_E_SHAPE, "spectral plan: parameters for d=%d, data of d=%d columns",
             (int)p->sm_mu.size() / Q, d);
  GP_REQUIRE(p->backend == GP_BACKEND_SIMT, GP_E_STATE, "spectral plan: the packing did not select the CUDA-core layout");
  cudaStream_t st = p->stream;
  const int W = sm_width(d, Q);
  p->DP = W;
  GP_CHECK(p->mean.ensure(sizeof(float) * (d + 4 + SM_QMAX * SM_DMAX)));
  p->xbad = reinterpret_cast<int*>(p->mean.as<float>() + d);
  float* mu_d = p->mean.as<float>() + d + 4;
  GP_CUDA(cudaMemsetAsync(p->xbad, 0, sizeof(int), st));
  GP_CUDA(cudaMemcpyAsync(mu_d, p->sm_mu.data(), sizeof(float) * Q * d, cudaMemcpyHostToDevice, st));
  const float* X2 = p->same ? p->X1 : p->X2;
  const int64_t ld2 = p->same ? p->ld1 : p->ld2;
  GP_CHECK(p->Z2.ensure(sizeof(float) * p->n2 * W));
  spectral_pack_kernel<<<(unsigned)cdiv(p->n2, 256), 256, 0, st>>>(X2, p->n2, ld2, d, Q, W, mu_d, p->Z2.as<float>(), p->xbad);
  p->launches++;
  if (!p->same) {
    GP_CHECK(p->Z1.ensure(sizeof(float) * p->n1 * W));
    spectral_pack_kernel<<<(unsigned)cdiv(p->n1, 256), 256, 0, st>>>(p->X1, p->n1, p->ld1, d, Q, W, mu_d, p->Z1.as<float>(), p->xbad);
    p->launches++;
  }
  double sw = 0.0;
  for (int q = 0; q < Q; ++q) sw += (double)p->sm_w[q];
  p->sm_diag = (double)p->outputscale * pow(sw, d);
  p->nparts = p->nsplit;
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  GP_CUDA(cudaStreamSynchronize(st));   // sm_mu is read from host memory the plan may change
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

static const float* sm_z1(const gp_plan* p) { return p->same ? p->Z2.as<float>() : p->Z1.as<float>(); }

// the compiled (d, QM) cases, keyed d * 100 + QM
template <class F>
static bool with_sm_case(int key, F&& f) {
  return with_width<101, 104, 116, 201, 204, 216, 301, 304, 310, 401, 404, 408, 501, 504, 506, 601, 604, 605, 701, 704, 801, 804>(key, f);
}

int spectral_kmv_launch(gp_plan* p, const float* V16, const int* done_flag) {
  GP_REQUIRE(V16 != nullptr, GP_E_STATE, "spectral plan: fp32 rows of V needed");
  const SmHyp h = spectral_hyp(p);
  dim3 grid((unsigned)cdiv(p->row_count, SIMT_TI), (unsigned)p->nsplit);
  const int64_t cps = p->tiles_per_split * SIMT_TJ;
  const bool ok = with_sm_case(p->d * 100 + sm_qcase(p->d, h.Q), [&](auto key) {
    constexpr int K = decltype(key)::value;
    spectral_kmv_kernel<K / 100, K % 100><<<grid, SIMT_TI, 0, p->stream>>>(sm_z1(p), p->Z2.as<float>(), p->DP, V16, partial_ptr(p),
                                                                          p->row_count, p->n2, p->rows_pad, cps, h, done_flag);
  });
  if (!ok) {
    set_error("spectral plan: no compiled case for d=%d, Q=%d", p->d, h.Q);
    return GP_E_SHAPE;
  }
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int spectral_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "rows of a spectral plan: at most 65535 rows per call (m=%lld)", (long long)m);
  return launch_krows(p, SmEntry{sm_z1(p), p->Z2.as<float>(), p->DP, spectral_hyp(p)}, idx, m, OUT, ldo);
}

// square: the constant S (sum_q w_q)^d; cross: per pair.  NaN for non-finite inputs
int spectral_kdiag(gp_plan* p, float* OUT) {
  const float diag = (float)p->sm_diag;
  return launch_kdiag(p, OUT, &diag, SmEntry{p->Z1.as<float>(), p->Z2.as<float>(), p->DP, spectral_hyp(p)});
}

// grad_ls = [dF/dw_q (Q) | dF/dmu_qc (Q d, row-major) | dF/dv_qc (Q d, row-major)], *grad_os = dF/dS
int spectral_bilinear_grad(gp_plan* p, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  const SmHyp h = spectral_hyp(p);
  const int d = p->d, Q = h.Q;
  const int GQ = sm_gq(d), NO = 1 + GQ * (1 + 2 * d);
  const int ngrp = (int)cdiv(Q, GQ), nout = ngrp * NO;
  dim3 grid;
  int64_t cps;
  bilinear_split(p, p->n2, &grid, &cps);
  const int64_t nblk = (int64_t)grid.x * grid.y;
  grid.z = (unsigned)ngrp;
  std::vector<double> total;
  GP_CHECK(bilinear_sweep(p, Lf, ldl, Rt, ldr, s, p->row_count, nblk, nout, [&](const float* L16, const float* R16, double* gout) -> int {
    const bool ok = with_sm_case(d * 100 + sm_qcase(d, Q), [&](auto key) {
      constexpr int K = decltype(key)::value;
      spectral_bilinear_kernel<K / 100, K % 100><<<grid, SIMT_TI, 0, p->stream>>>(sm_z1(p), p->Z2.as<float>(), p->DP, L16, R16,
                                                                                 p->row_count, p->n2, cps, h, gout, nout);
    });
    if (!ok) {
      set_error("spectral plan: no compiled case for d=%d, Q=%d", d, Q);
      return GP_E_SHAPE;
    }
    p->launches++;
    GP_CUDA(cudaGetLastError());
    return GP_OK;
  }, total));
  const double S = p->outputscale;
  *grad_os = total[0];
  for (int q = 0; q < Q; ++q) {
    const int base = (q / GQ) * NO, k = q % GQ;
    const double w = p->sm_w[q];
    grad_ls[q] = S * total[base + 1 + k];
    for (int c = 0; c < d; ++c) {
      grad_ls[Q + q * d + c] = -2.0 * M_PI * S * w * total[base + 1 + GQ + k * d + c];
      grad_ls[Q + Q * d + q * d + c] = -4.0 * M_PI * M_PI * S * w * (double)p->sm_v[q * d + c] * total[base + 1 + GQ + GQ * d + k * d + c];
    }
  }
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_spectral(gp_plan* p, int Q, const float* weights, const float* means, const float* scales, int d) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  if (weights == nullptr || Q == 0) {   // back to a plain plan
    if (p->sm_Q == 0) return GP_OK;
    p->sm_Q = 0;
    p->sm_w.clear();
    p->sm_mu.clear();
    p->sm_v.clear();
    return (p->data_set && p->hypers_set) ? pack_inputs(p) : GP_OK;
  }
  GP_REQUIRE(p->data_set, GP_E_STATE, "spectral plan: call gp_plan_set_data first");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "a SKI plan cannot become a spectral plan");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel-sum plan cannot become a spectral plan");
  GP_CHECK(refuse_settings(p, CALL_SET_SPECTRAL));
  GP_CHECK(refuse_compact(p, "gp_plan_set_spectral"));
  GP_REQUIRE(p->row_begin == 0 && p->row_count == p->n1 && !(p->comm && p->comm->world > 1), GP_E_SHAPE,
             "a spectral plan is not available on a row-sharded plan");
  GP_REQUIRE(Q >= 1 && Q <= SM_QMAX && d >= 1 && d <= SM_DMAX && Q * d <= SM_QDMAX, GP_E_SHAPE,
             "a spectral plan takes 1 <= Q <= %d components over 1 <= d <= %d dimensions with Q d <= 32 (got Q=%d, d=%d)", SM_QMAX,
             SM_DMAX, Q, d);
  GP_REQUIRE(d == p->d, GP_E_SHAPE, "spectral plan: parameters for d=%d, data of d=%d columns", d, p->d);
  GP_REQUIRE(means != nullptr && scales != nullptr, GP_E_SHAPE, "spectral plan: null means or scales");
  GP_CUDA(cudaSetDevice(p->device));
  p->sm_Q = Q;
  p->sm_w.assign(weights, weights + Q);
  p->sm_mu.assign(means, means + Q * d);
  p->sm_v.assign(scales, scales + Q * d);
  return p->hypers_set ? pack_inputs(p) : GP_OK;
}
