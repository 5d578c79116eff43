// cg.cu -- modified batched preconditioned conjugate gradients (mBCG) on the device.
//
// Restates linear_operator.utils.linear_cg (SURVEY.md Appendix A.2; signature attested at
// /root/reference/gpytorch/variational/ciq_variational_strategy.py:56-64) with the matmul closure
// fixed to  v -> K(X,X) v + D v  (D = sigma^2 I, or a per-row diagonal for FixedNoiseGaussianLikelihood,
// likelihoods/gaussian_likelihood.py:245-363) evaluated by the fused kernels.  All vectors are [n_local][16]
// fp32 in HBM (L2 resident at the BASELINE sizes); alpha/beta/gamma, the convergence flags and the
// Lanczos tridiagonals live in a CgState struct on the device; the stop rule is evaluated on the
// device and later launches become no-ops, so the host never synchronises inside the loop.
//
// One iteration = 6 launches and TWO global reductions (round 1: 10 launches, three reductions):
//   K.V            fused kernel-matmul on the packed direction tiles                          (kmv_tc.cu) 
//   finishv_wtv    V = os sum_s partial_s + D P ; per-CTA partials of p.V and of W^T V        (W streamed once)
//   sum            fixed-order fp64 sums of the partials  -> message 1: [ pV (16) | W^T V (16 k) ]     (all-reduce)
//   update_precond alpha = gamma / pV ; U += alpha P ; R -= alpha V ; w = W^T R_k - alpha o W^T V ;
//                  Z = P^-1 R = a_r R - s W w ; per-CTA partials of r.r, z.r and W^T R_{k+1}  (W streamed once)
//   sum            -> message 2: [ r.r | z.r | W^T R_{k+1} ]                                                  (all-reduce)
//   dir_pack       beta, P = Z + beta P written both as [n][16] and as the packed tf32-hi/lo + bf16 tiles the fused
//                  kernel's TMA reads; stop rule + tridiagonals
// The preconditioner  P^-1 v = a v - s W (W^T v)  needs W^T R_{k+1} BEFORE Z can be formed -- a third dependent reduction in
// the textbook form.  Here it comes from ONE step of the recurrence  W^T R_{k+1} = W^T R_k - alpha o (W^T V), whose right-hand
// side rides in message 1, re-based every iteration on the directly computed W^T R_k that rides in message 2 (in exact
// arithmetic identical to applying the closure to R_{k+1}; in floating point they differ by one step's rounding, ~1e-7).
// Column-wise dots are two-stage (per-CTA fp32 partials -> fixed-order fp64 sum): deterministic, and the sums are the
// messages of the NCCL all-reduces when rows are sharded across GPUs.
#include <algorithm>
#include <dlfcn.h>

#include "rowpass.cuh"

namespace gp {

constexpr int KMAX = 128;     // max preconditioner rank handled by the fused apply

// shared-memory row pitch of a staged W chunk: a multiple of 4 floats with pitch % 32 == 4, so that the 8 rows a warp touches
// with one LDS.128 fall into 8 different 4-bank groups (conflict free)
static inline int w_pitch(int k) {
  int p = (k + 3) & ~3;
  while (p % 32 != 4) p += 4;
  return p;
}

// sum G partial vectors of length L (fp32) into fp64, fixed order.  Block = 32 outputs x 8 partial groups.
constexpr int SUM_GROUPS = 32;  // cg_sum_kernel: 32 outputs x 32 row groups per CTA
__global__ void __launch_bounds__(32 * SUM_GROUPS) cg_sum_kernel(const float* __restrict__ in, int G, int L, double* __restrict__ out,
                                                                  const int* done) {
  if (done && *done) return;
  __shared__ double sh[SUM_GROUPS][33];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int o = blockIdx.x * 32 + lane;
  double s = 0.0;
  if (o < L) {
    // independent loads first (the partial matrix is [G][L]: one 128-byte line per row and warp), fixed summation order
    int b = grp;
    for (; b + 3 * SUM_GROUPS < G; b += 4 * SUM_GROUPS) {
      const float v0 = in[(size_t)b * L + o], v1 = in[(size_t)(b + SUM_GROUPS) * L + o];
      const float v2 = in[(size_t)(b + 2 * SUM_GROUPS) * L + o], v3 = in[(size_t)(b + 3 * SUM_GROUPS) * L + o];
      s += (double)v0; s += (double)v1; s += (double)v2; s += (double)v3;
    }
    for (; b < G; b += SUM_GROUPS) s += (double)in[(size_t)b * L + o];
  }
  sh[grp][lane] = s;
  __syncthreads();
  if (grp == 0 && o < L) {
    double t = 0.0;
#pragma unroll
    for (int g2 = 0; g2 < SUM_GROUPS; ++g2) t += sh[g2][lane];
    out[o] = t;
  }
}

__global__ void cg_rhs_sq_kernel(const float* __restrict__ RHS, int64_t ldr, int t, int64_t n, float* __restrict__ part) {
  __shared__ __align__(16) float red[RP_ROWS * TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  float4 acc = make_float4(0, 0, 0, 0);
  for (int64_t r = (int64_t)blockIdx.x * RP_ROWS + rl; r < n; r += (int64_t)gridDim.x * RP_ROWS) {
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      int c = cg * 4 + q;
      v[q] = (c < t) ? RHS[r * ldr + c] : 0.f;
    }
    acc.x = fmaf(v[0], v[0], acc.x); acc.y = fmaf(v[1], v[1], acc.y);
    acc.z = fmaf(v[2], v[2], acc.z); acc.w = fmaf(v[3], v[3], acc.w);
  }
  block_reduce_cols(acc, red, part + (size_t)blockIdx.x * TP);
}

// R = rhs / |rhs| ; U = 0 ; state init
__global__ void cg_init_kernel(const float* __restrict__ RHS, int64_t ldr, int t, int64_t n, const double* __restrict__ sums,
                               float eps, float* __restrict__ U, float* __restrict__ R, CgState* __restrict__ st) {
  __shared__ float inv_norm[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  if (tid < TP) {
    float nrm = (float)sqrt(sums[tid]);
    int zero = nrm < eps;
    if (zero) nrm = 1.f;
    inv_norm[tid] = 1.f / nrm;
    if (blockIdx.x == 0) {
      st->rhs_norm[tid] = nrm;
      st->rhs_zero[tid] = zero;
      st->conv[tid] = zero;  // |R_0| = 1 for non-zero columns, < stop_updating_after for zero ones
      st->rnorm[tid] = zero ? 0.f : 1.f;
      st->alpha[tid] = 0.f; st->beta[tid] = 0.f; st->prev_ar[tid] = 0.f; st->prev_beta[tid] = 0.f;
      st->gamma[0][tid] = 0.0; st->gamma[1][tid] = 0.0;
      if (tid == 0) { st->update_tridiag = 1; st->last_tridiag_iter = 0; st->done = 0; st->iters = 0; st->tol_reached = 0; st->nan_flag = 0; }
    }
  }
  __syncthreads();
  for (int64_t r = (int64_t)blockIdx.x * RP_ROWS + rl; r < n; r += (int64_t)gridDim.x * RP_ROWS) {
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      int c = cg * 4 + q;
      v[q] = (c < t) ? RHS[r * ldr + c] * inv_norm[c] : 0.f;
    }
    reinterpret_cast<float4*>(R)[r * 4 + cg] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(U)[r * 4 + cg] = make_float4(0, 0, 0, 0);
  }
}

// stage rows [r0, r0 + nr) of W [n][k] (one contiguous block of nr * k floats) into Ws [64][wp] with coalesced loads
__device__ __forceinline__ void stage_w(const float* __restrict__ W, int k, int wp, int64_t r0, int nr, float* __restrict__ Ws) {
  const float* wsrc = W + r0 * k;
  const int tot = nr * k;
  const int tid = threadIdx.x;
  if ((k & 3) == 0) {
    for (int e = tid * 4; e < tot; e += RP_THREADS * 4) {
      const float4 v4 = *reinterpret_cast<const float4*>(wsrc + e);
      const int rr = e / k, kk = e - rr * k;
      *reinterpret_cast<float4*>(&Ws[rr * wp + kk]) = v4;
    }
  } else {
    for (int e = tid; e < tot; e += RP_THREADS) {
      const int rr = e / k, kk = e - rr * k;
      Ws[rr * wp + kk] = wsrc[e];
    }
  }
}

// ---- kernel B: V = os * sum_s partial + D P ; partial pV ; partial W^T X (X = V in the loop, X = R at start-up) -------------------
// Rows are processed in chunks of 64: phase 1 (thread = row lane x column group) builds the X rows, writes V and stages X in
// shared memory; phase 2 (thread = row half x 4 k x 4 columns) accumulates the [k x 16] skinny product in 4 x 4 register
// tiles from the W chunk staged in shared memory.
// out: part[blockIdx][0..16) = sum p.V (FINISH only) ; part[blockIdx][16 + kk*16 + c] = sum_r W[r][kk] X[r][c]
template <bool FINISH>
__global__ void __launch_bounds__(RP_THREADS)
cg_finishv_wtv_kernel(const float* __restrict__ kpart, int nsplit, int64_t rows_pad, float os, const float* __restrict__ pscale, float noise,
                      const float* __restrict__ dvec, const float* __restrict__ P, float* __restrict__ V,
                      const float* __restrict__ Xin, const float* __restrict__ W, int k, int wp, int64_t n,
                      float* __restrict__ part, int L, const int* done, const int* __restrict__ xbad) {
  if (done && *done) return;
  extern __shared__ __align__(16) float sh[];
  float* Xs = sh;                       // [64][16]
  float* red = sh + RP_ROWS * TP;       // [64][16]
  float* Ws = red + RP_ROWS * TP;       // [64][wp]  (reused as the [128][16] exchange buffer at the end)
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  const int kg = (tid >> 2) & 31, half = tid >> 7;
  const bool act = kg * 4 < k;
  const float poison = (FINISH && *xbad) ? __int_as_float(0x7fc00000) : 0.f;  // non-finite inputs: K.V is NaN in the reference
  float4 acc = make_float4(0, 0, 0, 0);
  float wacc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) wacc[a][b] = 0.f;
  const int64_t nchunk = cdiv(n, RP_ROWS);
  for (int64_t ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
    const int64_t r0 = ch * RP_ROWS;
    const int nr = (int)min((int64_t)RP_ROWS, n - r0);
    __syncthreads();   // previous chunk's phase 2 has finished with Xs / Ws
    if (k > 0) stage_w(W, k, wp, r0, nr, Ws);
    // phase 1: X rows
    {
      const int64_t r = r0 + rl;
      float4 x = make_float4(0, 0, 0, 0);
      if (rl < nr) {
        if (FINISH) {
          x = khat_row(kpart, nsplit, rows_pad, os, pscale, poison, P, dvec, noise, r, cg);
          const float4 p = reinterpret_cast<const float4*>(P)[r * 4 + cg];
          reinterpret_cast<float4*>(V)[r * 4 + cg] = x;
          acc.x = fmaf(p.x, x.x, acc.x); acc.y = fmaf(p.y, x.y, acc.y); acc.z = fmaf(p.z, x.z, acc.z); acc.w = fmaf(p.w, x.w, acc.w);
        } else {
          x = reinterpret_cast<const float4*>(Xin)[r * 4 + cg];
        }
      }
      reinterpret_cast<float4*>(Xs)[rl * 4 + cg] = x;
    }
    __syncthreads();
    // phase 2: wacc[a][b] += W[r][4 kg + a] X[r][4 cg + b] over this thread's row half
    if (k > 0 && act) {
#pragma unroll 4
      for (int rr = half; rr < nr; rr += 2) {
        const float4 wv = *reinterpret_cast<const float4*>(&Ws[rr * wp + kg * 4]);
        const float4 xv = *reinterpret_cast<const float4*>(&Xs[rr * TP + cg * 4]);
        const float w4[4] = {wv.x, wv.y, wv.z, wv.w}, x4[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) wacc[a][b] = fmaf(w4[a], x4[b], wacc[a][b]);
      }
    }
  }
  __syncthreads();
  float* o = part + (size_t)blockIdx.x * L;
  if (k > 0) {
    // combine the two row halves through shared memory (fixed order), then write the CTA partial
    float* xr = Ws;  // [128 kk][16]  (the host sizes the dynamic shared memory for max(64 * wp, 128 * 16) floats here)
    if (half == 1 && act) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) xr[((kg * 4 + a) * 4 + cg) * 4 + b] = wacc[a][b];
    }
    __syncthreads();
    if (half == 0 && act) {
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int kk = kg * 4 + a;
        if (kk < k) {
#pragma unroll
          for (int b = 0; b < 4; ++b) o[TP + kk * TP + cg * 4 + b] = wacc[a][b] + xr[((kg * 4 + a) * 4 + cg) * 4 + b];
        }
      }
    }
  }
  if (FINISH) block_reduce_cols(acc, red, o);
  else if (tid < TP) o[tid] = 0.f;
}

// ---- kernel D: alpha, U, R, w, Z = P^-1 R, partials of r.r, z.r and W^T R_new -----------------------------------------------------
// sums1 = [ pV (16) | W^T V (16 k) ] (fp64, all-reduced).  wprev = W^T R_k [k][16] fp64: the DIRECTLY computed product that the
// previous launch of this kernel shipped in message 2, so the recurrence  w_{k+1} = w_k - alpha o W^T V  is re-based every
// iteration and its rounding never accumulates (carried on its own it stalled tight-tolerance solves at ~3e-4 residual).
// INIT: alpha = 0, w = sums1[16..] (= W^T R_0 computed by the start-up pass), U / R untouched.
// Z = a_r R - s W w with (a_r, s) = (1/sigma^2, 1/sigma^2) for the constant diagonal, (1/d_r, 1) for a per-row diagonal whose
// factor W is pre-scaled (pivchol.cu).  Without a preconditioner (k == 0) Z aliases R and z.r = r.r.
template <bool INIT>
__global__ void __launch_bounds__(RP_THREADS, 2)   // sm_90 ptxas otherwise caps the INIT variant at 64 registers and spills
cg_update_precond_kernel(const double* __restrict__ sums1, int iter, float eps, const float* __restrict__ P,
                         const float* __restrict__ V, float* __restrict__ U, float* __restrict__ R, float* __restrict__ Z,
                         const float* __restrict__ W, int k, int wp, const double* __restrict__ wprev,
                         float inv_noise, const float* __restrict__ dvec, int64_t n, CgState* __restrict__ st,
                         float* __restrict__ part /*[G][L2], L2 = 32 + 16 k*/, int L2) {
  if (!INIT && st->done) return;
  extern __shared__ __align__(16) float sh[];
  float* red = sh;                                  // [64][16]
  float* Xs = red + RP_ROWS * TP;                   // [64][16] the new residual rows of the chunk
  float* ws = Xs + RP_ROWS * TP;                    // [k][16] w (float)
  float* Ws = ws + (size_t)k * TP;                  // [64][wp]  (reused as the [128][16] exchange buffer at the end)
  __shared__ float alpha_s[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  const int kg = (tid >> 2) & 31, half = tid >> 7;
  const bool act = kg * 4 < k;
  float wacc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) wacc[a][b] = 0.f;
  if (tid < TP) {
    float a = 0.f;
    if (!INIT) {
      const float pv = (float)sums1[tid];
      const float gam = (float)st->gamma[iter & 1][tid];
      const bool zero = pv < eps;
      a = zero ? 0.f : gam / pv;
      if (st->conv[tid]) a = 0.f;
      if (blockIdx.x == 0) {
        st->alpha[tid] = a;
        if (iter == 0 && !(pv == pv)) st->nan_flag = 1;
      }
    }
    alpha_s[tid] = a;
  }
  __syncthreads();
  for (int e = tid; e < k * TP; e += RP_THREADS) {
    const double w = INIT ? sums1[TP + e] : wprev[e] - (double)alpha_s[e & (TP - 1)] * sums1[TP + e];
    ws[e] = (float)w;
  }
  const float4 al = reinterpret_cast<float4*>(alpha_s)[cg];
  float4 arr = make_float4(0, 0, 0, 0), azr = make_float4(0, 0, 0, 0);
  const int64_t nchunk = cdiv(n, RP_ROWS);
  for (int64_t ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
    const int64_t r0 = ch * RP_ROWS;
    const int nr = (int)min((int64_t)RP_ROWS, n - r0);
    __syncthreads();   // ws ready / previous chunk done with Ws
    if (k > 0) stage_w(W, k, wp, r0, nr, Ws);
    const int64_t r = r0 + rl;
    float4 rr4 = make_float4(0, 0, 0, 0);
    if (rl < nr) {
      rr4 = reinterpret_cast<float4*>(R)[r * 4 + cg];
      if (!INIT) {
        const float4 p = reinterpret_cast<const float4*>(P)[r * 4 + cg];
        const float4 v = reinterpret_cast<const float4*>(V)[r * 4 + cg];
        float4 u = reinterpret_cast<float4*>(U)[r * 4 + cg];
        u.x = fmaf(al.x, p.x, u.x); u.y = fmaf(al.y, p.y, u.y); u.z = fmaf(al.z, p.z, u.z); u.w = fmaf(al.w, p.w, u.w);
        rr4.x = fmaf(-al.x, v.x, rr4.x); rr4.y = fmaf(-al.y, v.y, rr4.y); rr4.z = fmaf(-al.z, v.z, rr4.z); rr4.w = fmaf(-al.w, v.w, rr4.w);
        reinterpret_cast<float4*>(U)[r * 4 + cg] = u;
        reinterpret_cast<float4*>(R)[r * 4 + cg] = rr4;
      }
      arr.x = fmaf(rr4.x, rr4.x, arr.x); arr.y = fmaf(rr4.y, rr4.y, arr.y); arr.z = fmaf(rr4.z, rr4.z, arr.z); arr.w = fmaf(rr4.w, rr4.w, arr.w);
    }
    reinterpret_cast<float4*>(Xs)[rl * 4 + cg] = rr4;
    __syncthreads();   // Ws and Xs staged
    if (k > 0 && rl < nr) {
      float4 s = make_float4(0, 0, 0, 0);
      const float* wrow = Ws + rl * wp;
      int kk = 0;
      for (; kk + 4 <= k; kk += 4) {
        const float4 wv = *reinterpret_cast<const float4*>(wrow + kk);
        const float w4[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const float4 c4 = *reinterpret_cast<const float4*>(&ws[(kk + a) * TP + cg * 4]);
          s.x = fmaf(w4[a], c4.x, s.x); s.y = fmaf(w4[a], c4.y, s.y); s.z = fmaf(w4[a], c4.z, s.z); s.w = fmaf(w4[a], c4.w, s.w);
        }
      }
      for (; kk < k; ++kk) {
        const float wv = wrow[kk];
        const float4 c4 = *reinterpret_cast<const float4*>(&ws[kk * TP + cg * 4]);
        s.x = fmaf(wv, c4.x, s.x); s.y = fmaf(wv, c4.y, s.y); s.z = fmaf(wv, c4.z, s.z); s.w = fmaf(wv, c4.w, s.w);
      }
      const float ar = dvec ? 1.f / dvec[r] : inv_noise;
      const float sc = dvec ? 1.f : inv_noise;
      const float4 z = make_float4(fmaf(ar, rr4.x, -sc * s.x), fmaf(ar, rr4.y, -sc * s.y), fmaf(ar, rr4.z, -sc * s.z), fmaf(ar, rr4.w, -sc * s.w));
      reinterpret_cast<float4*>(Z)[r * 4 + cg] = z;
      azr.x = fmaf(z.x, rr4.x, azr.x); azr.y = fmaf(z.y, rr4.y, azr.y); azr.z = fmaf(z.z, rr4.z, azr.z); azr.w = fmaf(z.w, rr4.w, azr.w);
    }
    // W^T R_new, accumulated directly from the rows just written: 4 x 4 register tiles over this thread's row half
    if (k > 0 && act) {
#pragma unroll 4
      for (int rr = half; rr < nr; rr += 2) {
        const float4 wv = *reinterpret_cast<const float4*>(&Ws[rr * wp + kg * 4]);
        const float4 xv = *reinterpret_cast<const float4*>(&Xs[rr * TP + cg * 4]);
        const float w4[4] = {wv.x, wv.y, wv.z, wv.w}, x4[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) wacc[a][b] = fmaf(w4[a], x4[b], wacc[a][b]);
      }
    }
  }
  __syncthreads();
  float* o = part + (size_t)blockIdx.x * L2;
  if (k > 0) {
    float* xr = Ws;  // [128 kk][16]
    if (half == 1 && act) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) xr[((kg * 4 + a) * 4 + cg) * 4 + b] = wacc[a][b];
    }
    __syncthreads();
    if (half == 0 && act) {
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int kk = kg * 4 + a;
        if (kk < k) {
#pragma unroll
          for (int b = 0; b < 4; ++b) o[2 * TP + kk * TP + cg * 4 + b] = wacc[a][b] + xr[((kg * 4 + a) * 4 + cg) * 4 + b];
        }
      }
    }
  }
  block_reduce_cols(arr, red, o);
  __syncthreads();
  block_reduce_cols(k > 0 ? azr : arr, red, o + TP);   // no preconditioner: Z = R, z.r = r.r
}

// ---- kernel E: beta, P = Z + beta P (fp32 rows AND packed K.V tiles), stop rule, tridiagonals ------------------------------------
// sums2 = message 2 [ r.r (16) | z.r (16) | W^T R (16 k) ] (fp64; all-reduced when sharded); only the first 32 values are read here.
// Thread = (4-row chunk, column group): it owns a 4 x 4 block of P, which is exactly one float4 (4 consecutive rows of one
// column) of the tf32-hi tile, of the tf32-lo tile and one uint2 of the bf16 tile for each of its 4 columns (pack.cu layout).
// INIT: beta = 0 (P = Z), gamma[0] = z.r, no bookkeeping.
constexpr int V_TILE_FLOATS_CG = (2 * TILE_J * TP * 4 + TILE_J * TP * 2) / 4;  // 2560 floats per 64-row tile
template <bool INIT>
__global__ void __launch_bounds__(RP_THREADS)
cg_dir_pack_kernel(const double* __restrict__ sums2, int iter, float eps,
                   float stop_after, float tol, int t, int n_tridiag, int n_tridiag_iter, int max_iter,
                   const float* __restrict__ Z, float* __restrict__ P, int64_t n, int64_t nchunk_pack,
                   float* __restrict__ Vt, CgState* __restrict__ st, float* __restrict__ TMAT, int ldt) {
  if (!INIT && st->done) return;
  __shared__ double ssum[2 * TP];
  __shared__ float beta_s[TP];
  __shared__ float rn_s[TP];
  const int tid = threadIdx.x;
  if (tid < 2 * TP) ssum[tid] = sums2[tid];
  __syncthreads();
  if (tid < TP) {
    float b = 0.f;
    if (!INIT) {
      const float gold = (float)st->gamma[iter & 1][tid];
      const float gnew = (float)ssum[TP + tid];
      const bool zero = gold < eps;
      b = zero ? 0.f : gnew / gold;
    }
    beta_s[tid] = b;
    float rn = sqrtf((float)ssum[tid]);
    if (st->rhs_zero[tid]) rn = 0.f;
    rn_s[tid] = rn;
  }
  __syncthreads();
  // NOTE: block 0 mutates st->done / gamma[(iter+1)&1] / conv below; other CTAs of THIS launch only read
  // gamma[iter&1] and the pre-launch value of done, and P rows written after a stop are never read again.
  const float4 be = reinterpret_cast<float4*>(beta_s)[tid & 3];
  const int64_t tot = max(nchunk_pack, cdiv(n, (int64_t)4)) * 4;   // (chunk, column group) work items
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + tid; e < tot; e += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(e & 3);          // == tid & 3: blockDim and gridDim * blockDim are multiples of 4
    const int64_t chunk = e >> 2;         // 4-row chunk
    const int64_t r0 = chunk * 4;
    float pn[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t r = r0 + q;
      if (r < n) {
        const float4 z = reinterpret_cast<const float4*>(Z)[r * 4 + cg];
        float4 p = INIT ? make_float4(0, 0, 0, 0) : reinterpret_cast<float4*>(P)[r * 4 + cg];
        p.x = fmaf(be.x, p.x, z.x); p.y = fmaf(be.y, p.y, z.y); p.z = fmaf(be.z, p.z, z.z); p.w = fmaf(be.w, p.w, z.w);
        reinterpret_cast<float4*>(P)[r * 4 + cg] = p;
        pn[q][0] = p.x; pn[q][1] = p.y; pn[q][2] = p.z; pn[q][3] = p.w;
      } else {
        pn[q][0] = pn[q][1] = pn[q][2] = pn[q][3] = 0.f;
      }
    }
    if (Vt != nullptr && chunk < nchunk_pack) {
      // (the tiles are only written here when this rank owns ALL rows: local row == global row)
      const int64_t tile = chunk / (TILE_J / 4);
      const int kc = (int)(chunk % (TILE_J / 4));
      float* tbase = Vt + tile * (int64_t)V_TILE_FLOATS_CG;
      float4* base = reinterpret_cast<float4*>(tbase);
      uint2* wb = reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(tbase) + 2 * TILE_J * TP * 4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = cg * 4 + j;
        float hi[4], lo[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          hi[q] = tf32_hi(pn[q][j]);
          lo[q] = tf32_hi(pn[q][j] - hi[q]);
        }
        base[kc * (2 * TP) + c] = make_float4(hi[0], hi[1], hi[2], hi[3]);        // B rows 0..15  = V_hi columns
        base[kc * (2 * TP) + TP + c] = make_float4(lo[0], lo[1], lo[2], lo[3]);   // B rows 16..31 = V_lo columns
        uint32_t w0, w1;
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w0) : "f"(pn[1][j]), "f"(pn[0][j]));
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w1) : "f"(pn[3][j]), "f"(pn[2][j]));
        wb[((kc >> 1) * TP + c) * 2 + (kc & 1)] = make_uint2(w0, w1);
      }
    }
  }
  if (blockIdx.x == 0 && tid < 32) {
    const int c = tid;
    if (INIT) {
      if (c < TP) st->gamma[0][c] = ssum[TP + c];
      return;
    }
    float rn = (c < TP) ? rn_s[c] : 0.f;
    if (c < TP) {
      st->gamma[(iter + 1) & 1][c] = ssum[TP + c];
      st->beta[c] = beta_s[c];
      st->rnorm[c] = rn;
    }
    float msum = (c < t) ? rn : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) msum += __shfl_xor_sync(0xffffffffu, msum, o);
    const float mean_rn = msum / (float)t;
    const int kmin = min(10, max_iter - 1);
    const bool stop = (iter >= kmin) && (mean_rn < tol) && !(n_tridiag && iter < min(n_tridiag_iter, max_iter - 1));
    // tridiagonal update happens only when the loop does not break (linear_cg order)
    float off = 0.f;
    const bool do_tri = !stop && n_tridiag && iter < n_tridiag_iter && st->update_tridiag;
    if (do_tri && c < n_tridiag) {
      float a = st->alpha[c];
      float ar = 1.f / (a == 0.f ? 1.f : a);
      float* T = TMAT + (size_t)c * ldt * ldt;
      if (iter == 0) {
        T[0] = ar;
      } else {
        float pb = st->prev_beta[c], par = st->prev_ar[c];
        T[(size_t)iter * ldt + iter] = fmaf(pb, par, ar);
        off = sqrtf(pb) * par;
        T[(size_t)iter * ldt + iter - 1] = off;
        T[(size_t)(iter - 1) * ldt + iter] = off;
      }
      st->prev_ar[c] = ar;
      st->prev_beta[c] = beta_s[c];
    }
    float mx = (do_tri && c < n_tridiag) ? off : -1e30f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    __syncwarp();
    if (c < TP) st->conv[c] = (rn < stop_after) ? 1 : 0;
    if (c == 0) {
      if (do_tri) {
        if (iter > 0 && mx < 1e-6f) st->update_tridiag = 0;
        st->last_tridiag_iter = iter;
      }
      if (stop) {
        st->tol_reached = 1;
        st->iters = iter + 1;
        __threadfence();
        st->done = 1;
      } else if (st->nan_flag) {  // NaN in the first MVM: freeze (the host reports GP_E_NAN_MVM)
        st->iters = iter + 1;
        __threadfence();
        st->done = 1;
      } else if (iter == max_iter - 1) {
        st->iters = max_iter;
      }
    }
  }
}

// SOLVES[r][c] = U[r][c] * rhs_norm[c]
__global__ void cg_finalize_kernel(const float* __restrict__ U, const CgState* __restrict__ st, int64_t n, int t,
                                   float* __restrict__ S, int64_t lds) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * TP) return;
  int64_t r = idx / TP;
  int c = (int)(idx % TP);
  if (c < t) S[r * lds + c] = U[idx] * st->rhs_norm[c];
}

void cg_sum_launch(const float* in, int G, int L, double* out, const int* done, cudaStream_t st) {
  cg_sum_kernel<<<(unsigned)cdiv(L, 32), 32 * SUM_GROUPS, 0, st>>>(in, G, L, out, done);
}
void cg_rhs_sq_launch(const float* RHS, int64_t ldr, int t, int64_t n, float* part, int G, cudaStream_t st) {
  cg_rhs_sq_kernel<<<G, RP_THREADS, 0, st>>>(RHS, ldr, t, n, part);
}

static int allreduce(gp_plan* p, double* buf, size_t count) {
  if (p->comm && p->comm->world > 1) return nccl_allreduce_double(p->comm, buf, count, p->stream);
  return GP_OK;
}

int mbcg_run(gp_plan* p, const float* RHS, int64_t ldr, int t, int n_tridiag, float tol, int max_iter,
             int max_tridiag_iter, const float* W, int k, float* SOLVES, int64_t lds, float* TMAT, int* iters_out,
             int* tridiag_size, float* resid_out) {
  GP_REQUIRE(p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  KronColsScope kcols(p, t);   // the direction block's columns >= t stay zero
  GP_REQUIRE(p->same, GP_E_SHAPE, "mBCG needs a square operator (X2 == X1)");
  GP_REQUIRE(t >= 1 && t <= TP, GP_E_SHAPE, "mBCG handles 1..%d right-hand sides per call (t=%d)", TP, t);
  GP_REQUIRE(n_tridiag >= 0 && n_tridiag <= t, GP_E_SHAPE, "n_tridiag=%d out of range", n_tridiag);
  GP_REQUIRE(max_tridiag_iter <= max_iter, GP_E_SHAPE,
             "Getting a tridiagonalization larger than the number of CG iterations run is not possible!");
  GP_REQUIRE(W == nullptr || (k >= 1 && k <= KMAX), GP_E_SHAPE, "preconditioner rank %d not in [1,%d]", k, KMAX);
  if (W != nullptr) GP_CHECK(refuse_settings(p, CALL_MBCG_PRECOND));
  cudaStream_t st = p->stream;
  const int64_t n = p->row_count;       // local rows
  const int64_t N = p->n2;              // global size
  const bool sharded = p->comm && p->comm->world > 1;
  if (sharded) {
    // the all-gather of the direction blocks needs equal, rank-ordered shards (ncclAllGather has one count for all ranks)
    GP_REQUIRE(n * p->comm->world == N && p->row_begin == (int64_t)p->comm->rank * n, GP_E_SHAPE,
               "row-sharded mBCG needs equal contiguous shards: rank %d/%d owns [%lld,+%lld) of %lld rows (pad N to a multiple of the world size)",
               p->comm->rank, p->comm->world, (long long)p->row_begin, (long long)n, (long long)N);
  } else {
    GP_REQUIRE(n == N && p->row_begin == 0, GP_E_SHAPE, "a row shard [%lld,+%lld) of %lld rows needs a communicator (gp_plan_set_comm)",
               (long long)p->row_begin, (long long)n, (long long)N);
  }
  const float eps = 1e-10f, stop_after = 1e-10f;
  const int n_tridiag_iter = (int)std::min<int64_t>(max_tridiag_iter, N);
  const bool precond = W != nullptr;
  if (!precond) k = 0;
  const int wp = precond ? w_pitch(k) : 0;
  // CTAs per SM of the row-pass kernels: 2 with a preconditioner (the W chunk staged in shared memory bounds residency; 3 or 4
  // measured no faster at C2), 8 without one (pure streaming over the vectors: N = 10^6 rows at BASELINE C5)
  const int grid_mult = precond ? 2 : 8;
  const int G = (int)std::min<int64_t>(cdiv(n, RP_ROWS), (int64_t)grid_mult * p->n_sm);
  const int L1 = TP + k * TP;           // message 1: pV | W^T V
  const float* dvec = p->noise_diag ? p->noise_diag + p->row_begin : nullptr;
  GP_REQUIRE(!precond || dvec != nullptr || p->noise > 0.f, GP_E_SHAPE, "the preconditioner needs noise > 0");

  GP_CHECK(p->cgU.ensure(sizeof(float) * n * TP));
  GP_CHECK(p->cgR.ensure(sizeof(float) * n * TP));
  GP_CHECK(p->cgV.ensure(sizeof(float) * n * TP));
  if (precond) GP_CHECK(p->cgZ.ensure(sizeof(float) * n * TP));
  GP_CHECK(p->cgPfull.ensure(sizeof(float) * N * TP));
  const int L2 = 2 * TP + k * TP;       // message 2: r.r | z.r | W^T R
  GP_CHECK(p->red.ensure(sizeof(float) * (size_t)G * (L1 + L2)));
  GP_CHECK(p->sums.ensure(sizeof(double) * (size_t)(L1 + L2 + TP)));
  GP_CHECK(p->state.ensure(sizeof(CgState)));
  float* U = p->cgU.as<float>();
  float* R = p->cgR.as<float>();
  float* V = p->cgV.as<float>();
  float* Z = precond ? p->cgZ.as<float>() : R;
  float* Pfull = p->cgPfull.as<float>();
  float* P = Pfull + p->row_begin * TP;
  float* red1 = p->red.as<float>();              // [G][L1]
  float* red2 = red1 + (size_t)G * L1;           // [G][L2]
  double* sums1 = p->sums.as<double>();          // [L1]
  double* sums2 = sums1 + L1;                    // [L2]
  double* sums0 = sums2 + L2;                    // [16]  rhs^2
  CgState* S = p->state.as<CgState>();
  const int* done = &S->done;
  const float inv_noise = p->noise > 0.f ? 1.f / p->noise : 0.f;
  const size_t sh_b = sizeof(float) * ((size_t)2 * RP_ROWS * TP + std::max<size_t>((size_t)RP_ROWS * wp, 128 * TP));
  const size_t sh_d = sizeof(float) * ((size_t)2 * RP_ROWS * TP + (size_t)k * TP + std::max<size_t>((size_t)RP_ROWS * wp, 128 * TP));
  GP_CHECK(opt_in_smem<cg_finishv_wtv_kernel<true>>(p->device, 100 * 1024));
  GP_CHECK(opt_in_smem<cg_finishv_wtv_kernel<false>>(p->device, 100 * 1024));
  GP_CHECK(opt_in_smem<cg_update_precond_kernel<true>>(p->device, 100 * 1024));
  GP_CHECK(opt_in_smem<cg_update_precond_kernel<false>>(p->device, 100 * 1024));
  if (n_tridiag > 0) GP_CUDA(cudaMemsetAsync(TMAT, 0, sizeof(float) * (size_t)n_tridiag * max_tridiag_iter * max_tridiag_iter, st));

  // the direction block is written straight into the packed K.V tiles when this rank owns all rows and the tensor-core
  // kernel runs; sharded runs all-gather the fp32 rows first and pack the gathered block (pack.cu)
  const bool tc = plan_is_tc(p);
  // a multitask product packs its own task-ordered tiles (tasks.cu); a Kronecker product packs its B-mixed chunks (kron.cu)
  const bool fuse_pack = tc && !sharded && !p->tasks && !p->kron;
  float* Vt = fuse_pack ? p->Vtiles.as<float>() : nullptr;
  const int64_t nchunk_pack = fuse_pack ? p->ntile_j * (TILE_J / 4) : 0;
  const int Gd = (int)std::min<int64_t>(cdiv(std::max<int64_t>(nchunk_pack, cdiv(n, (int64_t)4)) * 4, (int64_t)RP_THREADS), 4 * p->n_sm);
  auto kmv = [&]() -> int {
    if (fuse_pack) {   // the direction block's fp32 rows (Pfull) feed the low-rank slot
      GP_CHECK(kmv_tc_launch(p, done));
      return lowrank_partials(p, Pfull, done);
    }
    if (sharded) GP_CHECK(nccl_allgather_float(p->comm, Pfull, (size_t)n * TP, st));
    return kmv_partials(p, Pfull, done);
  };

  // ---- init: normalise rhs, R, U ; w = W^T R ; Z = P^-1 R ; P = Z ; gamma = z.r ----
  cg_rhs_sq_launch(RHS, ldr, t, n, red1, G, st);
  cg_sum_launch(red1, G, TP, sums0, nullptr, st);
  GP_CHECK(allreduce(p, sums0, TP));
  cg_init_kernel<<<G, RP_THREADS, 0, st>>>(RHS, ldr, t, n, sums0, eps, U, R, S);
  p->launches += 3;
  if (precond) {
    cg_finishv_wtv_kernel<false><<<G, RP_THREADS, sh_b, st>>>(nullptr, 0, 0, 0.f, nullptr, 0.f, nullptr, nullptr, nullptr, R, W, k, wp, n, red1, L1,
                                                           nullptr, p->xbad);
    cg_sum_launch(red1, G, L1, sums1, nullptr, st);
    GP_CHECK(allreduce(p, sums1, L1));
    p->launches += 2;
  }
  cg_update_precond_kernel<true><<<G, RP_THREADS, sh_d, st>>>(sums1, 0, eps, nullptr, nullptr, U, R, Z, W, k, wp, nullptr, inv_noise, dvec, n, S,
                                                             red2, L2);
  cg_sum_launch(red2, G, L2, sums2, nullptr, st);
  GP_CHECK(allreduce(p, sums2, L2));
  cg_dir_pack_kernel<true><<<Gd, RP_THREADS, 0, st>>>(sums2, 0, eps, stop_after, tol, t, n_tridiag, n_tridiag_iter, max_iter, Z, P, n,
                                                     nchunk_pack, Vt, S, TMAT, max_tridiag_iter);
  p->launches += 3;
  GP_CUDA(cudaGetLastError());

  // ---- iterations ----
  const int first_stop = std::max(std::min(10, max_iter - 1), n_tridiag ? std::min(n_tridiag_iter, max_iter - 1) : 0);
  SolverLoop loop(p, "mBCG", done, first_stop);
  GP_CHECK(loop.create_events());
  int status = GP_OK;
  bool finished = false;
  for (int kk = 0; kk < max_iter && !finished; ++kk) {
    if ((status = kmv()) != GP_OK) break;
    cg_finishv_wtv_kernel<true><<<G, RP_THREADS, sh_b, st>>>(p->partial.as<float>(), nslots(p), p->rows_pad, kernel_scale(p), part_scale_ptr(p), p->noise, dvec, P, V,
                                                          nullptr, W, k, wp, n, red1, L1, done, p->xbad);
    cg_sum_launch(red1, G, L1, sums1, done, st);
    if ((status = allreduce(p, sums1, L1)) != GP_OK) break;
    // w_kk = W^T R_kk: the direct product shipped in message 2 of the previous launch of this kernel (start-up pass for kk = 0)
    cg_update_precond_kernel<false><<<G, RP_THREADS, sh_d, st>>>(sums1, kk, eps, P, V, U, R, Z, W, k, wp, sums2 + 2 * TP, inv_noise, dvec, n, S,
                                                                red2, L2);
    cg_sum_launch(red2, G, L2, sums2, done, st);
    if ((status = allreduce(p, sums2, L2)) != GP_OK) break;
    cg_dir_pack_kernel<false><<<Gd, RP_THREADS, 0, st>>>(sums2, kk, eps, stop_after, tol, t, n_tridiag, n_tridiag_iter, max_iter, Z, P, n,
                                                        nchunk_pack, Vt, S, TMAT, max_tridiag_iter);
    p->launches += 5;
    finished = loop.finished(kk);
  }
  status = loop.launch_status(status);
  if (status == GP_OK) {
    cg_finalize_kernel<<<(unsigned)cdiv(n * TP, 256), 256, 0, st>>>(U, S, n, t, SOLVES, lds);
    p->launches += 1;
    CgState* hs = reinterpret_cast<CgState*>(static_cast<char*>(p->pinned) + PIN_CG_STATE);
    cudaMemcpyAsync(hs, S, sizeof(CgState), cudaMemcpyDeviceToHost, st);
    status = loop.sync();
    if (status == GP_OK) {
      if (iters_out) *iters_out = hs->done ? hs->iters : max_iter;
      if (tridiag_size) *tridiag_size = n_tridiag ? hs->last_tridiag_iter + 1 : 0;
      if (resid_out)
        for (int c = 0; c < t; ++c) resid_out[c] = hs->rnorm[c];
      if (hs->nan_flag) {
        set_error("NaNs encountered when trying to perform matrix-vector multiplication");
        status = GP_E_NAN_MVM;
      } else if (!hs->tol_reached) {
        float m = 0.f;
        for (int c = 0; c < t; ++c) m += hs->rnorm[c];
        set_error("CG terminated in %d iterations with average residual norm %g which is larger than the tolerance of %g",
                  max_iter, m / t, tol);
        status = GP_W_NOT_CONVERGED;
      }
    }
  }
  return status;
}

}  // namespace gp

extern "C" int gp_mbcg(gp_plan* plan, const float* RHS, int64_t ldr, int t, int n_tridiag, float tolerance, int max_iter,
                       int max_tridiag_iter, const float* W, int k, float* SOLVES, int64_t lds, float* TMAT,
                       int* iters_out, int* tridiag_size, float* resid_out) {
  GP_REQUIRE(plan != nullptr, GP_E_STATE, "null plan");
  return gp::mbcg_run(plan, RHS, ldr, t, n_tridiag, tolerance, max_iter, max_tridiag_iter, W, k, SOLVES, lds, TMAT,
                      iters_out, tridiag_size, resid_out);
}
