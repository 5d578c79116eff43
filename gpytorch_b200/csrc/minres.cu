// minres.cu -- multi-shift MINRES on the device and the contour-integral-quadrature (CIQ) square-root product.
//
//   OUT = K_hat * sum_q w_q (K_hat + tau_q I)^{-1} B  ~=  K_hat^{1/2} B        (Pleiss et al. 2020, arXiv 2006.11267)
//
// K_hat is the plan's operator with its noise, exactly the closure gp_mbcg solves with (scalar sigma^2, a per-row diagonal, a
// kernel sum or SKI).  One Lanczos process per column is shared by all Q shifts (the Krylov space is shift-invariant); each
// (shift, column) pair runs its own Givens QR of T_k + tau_q I (Paige & Saunders 1975) with its scalar state in fp64 on the
// device, and each shift keeps two direction blocks.  The per-shift solutions are never stored: the update kernel accumulates
// Z = sum_q w_q x_q directly, and one more product after the loop gives OUT = K_hat Z.  (The identity form
// sum_q w_q (b - tau_q x_q) saves that product but cancels sum_q w_q ~ 200 down to 1, about 8 bits of fp32.)
//
// One iteration = the fused K.V launch(es) + 5 launches, two fixed-order reductions, no host synchronisation:
//   K.V        on the current Lanczos block q_k                                                      (kmv_partials)
//   finish     v = K q_k + D q_k - beta_k q_{k-1} ; per-CTA partials of q_k . v
//   sum        alpha_k  (cg_sum_kernel: fixed-order fp64)
//   orth       v -= alpha_k q_k ; per-CTA partials of v . v
//   sum        beta_{k+1}^2
//   update     q_{k+1} = v / beta_{k+1} ; rotations of every (shift, column) pair ; d_new = (q_k - delta d_{k-1} - eps d_{k-2}) / gamma ;
//              Z += w_q phi_q d_new ; stop rule
// Stop rule: column c has converged when max_q |phibar_q| <= tol (b_c is normalised, so |phibar| is the relative residual of
// MINRES on the shifted system), or on a Lanczos breakdown (beta_{k+1} below 1e-6 of the column's |T| entries: the Krylov space
// is exhausted and every shifted residual is exactly zero), or when b_c = 0 (Z = 0, OUT = 0).  The loop ends when every column
// has converged or at max_iter; the host reads the done flag one iteration behind (look-ahead, as cg.cu).
//
// Split preconditioning (gp_ciq_sqrt_matmul_precond).  P = L L^T + D is the pivoted-Cholesky preconditioner of K_hat = K + D
// (D = sigma^2 I or the per-row diagonal, > 0).  For any F with F F^T = P, A = F^-1 K_hat F^-T satisfies F A F^T = K_hat, so
// F A^{1/2} xi ~ N(0, K_hat), and by CIQ on A
//     F A sum_q w_q (A + tau_q I)^-1 xi = K_hat F^-T Z ,   Z = sum_q w_q (A + tau_q I)^-1 xi :
// only F^-1 and F^-T are ever applied.  F = D^{1/2} (I + M M^T)^{1/2} with M = D^{-1/2} L; with (V, s) = eigh(M^T M),
//     (I + M M^T)^{-1/2} = I - U U^T ,  U = D^{-1/2} L V diag(h) ,  h_j = (sqrt(1 + s_j) (1 + sqrt(1 + s_j)))^{-1/2}
// (gp_ciq_precond_build, pivchol.cu), so F^-1 = (I - U U^T) D^{-1/2} and F^-T = D^{-1/2} (I - U U^T).  E = K - L L^T >= 0 (the
// Schur complement pivoted Cholesky leaves) gives A = I + F^-1 E F^-T, hence 1 <= lambda(A) <= 1 + tr(E) / min d: the quadrature
// interval needs no Lanczos run.  One preconditioned iteration (c_k = U^T q_k, carried from the previous reduction):
//   pre        x_k = D^-1/2 (q_k - U c_k) = F^-T q_k                                       (ms_scale_kernel, preconditioned overload)
//   K.V        on x_k
//   finish     y = D^-1/2 K_hat x_k ; v = y - beta_k q_{k-1} ; partials of [ q_k . v | U^T y ]
//   sum        alpha_k = q_k . v - c_k . (U^T y)          (A q_k = y - U U^T y)
//   orth       v -= U (U^T y) + alpha_k q_k ; partials of [ v . v | U^T v ]
//   sum        beta_{k+1}^2 ; c_{k+1} = U^T v / beta_{k+1}  (re-based on the actual vector every iteration)
//   update     as above, with x_k in place of q_k in the direction recurrence: the directions and Z are then the F^-T images
//              of A's, and the tail OUT = K_hat (|b| Z) is the unpreconditioned one unchanged.
// finish, orth and update are one kernel each with a template flag PRE, whose preconditioned instance adds the U / D^-1/2 terms;
// pre is an overload of ms_scale_kernel.  The kernel names stay those of the unpreconditioned loop, so per-kernel resource
// checks cover both.  The preconditioned row passes stage each 64-row chunk's rows of U [n][k] in shared memory for U c and U^T v.
#include <math.h>

#include <algorithm>
#include <climits>
#include <cstddef>

#include "rowpass.cuh"

namespace gp {

constexpr int MS_QMAX = 32;     // shifts per call
constexpr int MS_KMAX = 128;    // preconditioner rank (the range of gp_precond_build)

// scalar state of one run; the per-iteration parts are double-buffered by iteration parity (every CTA of the update kernel
// reads parity k & 1 while block 0 writes parity (k + 1) & 1)
struct MsState {
  double c1[2][MS_QMAX * TP], s1[2][MS_QMAX * TP];   // rotation G_{k-1} per (shift, column)
  double c2[2][MS_QMAX * TP], s2[2][MS_QMAX * TP];   // rotation G_{k-2}
  double phibar[2][MS_QMAX * TP];
  double beta[2][TP];                                // beta_k: coupling of q_k to q_{k-1}
  int conv[2][TP];
  double tau[MS_QMAX], w[MS_QMAX];
  float rhs_norm[TP];
  int done;        // set with done_iter; K.V / finish / orth launches become no-ops
  int done_iter;   // iteration whose update kernel fired the stop (INT_MAX while running): later update launches return
  // read back by the host
  float resid[MS_QMAX * TP];   // |phibar| per (shift, column) after the last executed iteration
  int iters, nan_flag, all_conv, pad_;
};
constexpr size_t MS_READBACK = sizeof(MsState) - offsetof(MsState, resid);   // resid .. pad_
static_assert(MS_READBACK == sizeof(float) * MS_QMAX * TP + 4 * sizeof(int), "the read-back is resid, iters, nan_flag, all_conv, pad_");
static_assert(2 * MS_QMAX * sizeof(double) <= PIN_CIQ_OUT - PIN_CIQ_TW, "tau | w overflows its pinned slot");
static_assert(PIN_CIQ_OUT + MS_READBACK <= PINNED_BYTES, "the msMINRES read-back overflows the pinned scratch");

// q_1 = b / |b| (zero columns and columns >= t stay 0) ; q_0 = 0 ; Z = 0 ; scalar state of iteration 0
__global__ void __launch_bounds__(RP_THREADS)
ms_init_kernel(const float* __restrict__ B, int64_t ldb, int t, int64_t n, const double* __restrict__ sums, int Q,
               const double* __restrict__ tw /*[2][Q] tau | w*/, float* __restrict__ Qcur, float* __restrict__ Qprev,
               float* __restrict__ Z, MsState* __restrict__ st) {
  __shared__ float inv_norm[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  if (tid < TP) {
    const float nrm = (float)sqrt(sums[tid]);
    const bool zero = !(nrm >= 1e-10f) && nrm == nrm;   // a NaN norm is not "zero": it must reach the NaN check
    inv_norm[tid] = (tid < t && !zero) ? 1.f / nrm : 0.f;
    if (blockIdx.x == 0) {
      st->rhs_norm[tid] = (tid < t && !zero) ? nrm : 0.f;
      st->beta[0][tid] = 0.0;
      st->conv[0][tid] = (tid >= t || zero) ? 1 : 0;
    }
  }
  __syncthreads();
  if (blockIdx.x == 0) {
    for (int e = tid; e < MS_QMAX * TP; e += RP_THREADS) {
      const int c = e % TP;
      st->c1[0][e] = 1.0; st->s1[0][e] = 0.0; st->c2[0][e] = 1.0; st->s2[0][e] = 0.0;
      const bool live = c < t && (e / TP) < Q && inv_norm[c] != 0.f;   // a zero column starts (and stays) at residual 0
      st->phibar[0][e] = live ? 1.0 : 0.0;
      st->resid[e] = 0.f;
    }
    if (tid < MS_QMAX) {
      st->tau[tid] = tid < Q ? tw[tid] : 0.0;
      st->w[tid] = tid < Q ? tw[Q + tid] : 0.0;
    }
    if (tid == 0) { st->done = 0; st->done_iter = INT_MAX; st->iters = 0; st->nan_flag = 0; st->all_conv = 0; }
  }
  __syncthreads();
  for (int64_t r = (int64_t)blockIdx.x * RP_ROWS + rl; r < n; r += (int64_t)gridDim.x * RP_ROWS) {
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = cg * 4 + q;
      v[q] = (c < t) ? B[r * ldb + c] * inv_norm[c] : 0.f;
    }
    reinterpret_cast<float4*>(Qcur)[r * 4 + cg] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(Qprev)[r * 4 + cg] = make_float4(0, 0, 0, 0);
    reinterpret_cast<float4*>(Z)[r * 4 + cg] = make_float4(0, 0, 0, 0);
  }
}

// ---- row passes: finish and orth take PRE = true with a preconditioner ----------------------------------------------------------
// dynamic shared memory of the preconditioned passes: U rows of one chunk [64][kp] (kp = k | 1: an odd pitch puts the 8 rows a
// warp reads in 8 banks; the region is at least [64][16] and doubles as the reduction scratch after the last chunk) |
// X block [64][16] | coefficients [k][16]
__host__ __device__ inline int ms_upitch(int k) { return k | 1; }
__host__ __device__ inline int ms_urows(int k) { return RP_ROWS * (ms_upitch(k) > TP ? ms_upitch(k) : TP); }
inline size_t ms_pre_smem(int k) { return sizeof(float) * ((size_t)ms_urows(k) + RP_ROWS * TP + (size_t)k * TP); }

// rows [r0, r0 + nr) of U [n][k] (one contiguous block) -> us [nr][kp]
__device__ __forceinline__ int ms_stage_u(const float* __restrict__ U, int k, int64_t r0, int64_t n, float* __restrict__ us) {
  const int nr = (int)min((int64_t)RP_ROWS, n - r0);
  const int kp = ms_upitch(k);
  const float* src = U + r0 * k;
  for (int e = threadIdx.x; e < nr * k; e += RP_THREADS) {
    const int r = e / k;
    us[r * kp + (e - r * k)] = src[e];
  }
  return nr;
}

// acc[j] += sum_{r < nr} U[r][a0 + 16 j] xs[r][c]  (thread: c = tid & 15, a0 = tid >> 4)
__device__ __forceinline__ void ms_ut_acc(const float* __restrict__ us, int k, const float* __restrict__ xs, int nr,
                                          float (&acc)[MS_KMAX / 16]) {
  const int c = threadIdx.x & 15, a0 = threadIdx.x >> 4, kp = ms_upitch(k);
  for (int r = 0; r < nr; ++r) {
    const float xv = xs[r * TP + c];
#pragma unroll
    for (int j = 0; j < MS_KMAX / 16; ++j)
      if (a0 + 16 * j < k) acc[j] = fmaf(us[r * kp + a0 + 16 * j], xv, acc[j]);
  }
}

__device__ __forceinline__ void ms_ut_store(const float (&acc)[MS_KMAX / 16], int k, float* __restrict__ out /*[k][16]*/) {
  const int c = threadIdx.x & 15, a0 = threadIdx.x >> 4;
#pragma unroll
  for (int j = 0; j < MS_KMAX / 16; ++j)
    if (a0 + 16 * j < k) out[(a0 + 16 * j) * TP + c] = acc[j];
}

// sum_a U[rl][a] cs[a][4 cg .. 4 cg + 4)
__device__ __forceinline__ float4 ms_uc(const float* __restrict__ us, int k, const float* __restrict__ cs, int rl, int cg) {
  const float* u = us + rl * ms_upitch(k);
  float4 s = make_float4(0, 0, 0, 0);
  for (int a = 0; a < k; ++a) {
    const float ua = u[a];
    const float4 c4 = reinterpret_cast<const float4*>(cs)[a * 4 + cg];
    s.x = fmaf(ua, c4.x, s.x); s.y = fmaf(ua, c4.y, s.y); s.z = fmaf(ua, c4.z, s.z); s.w = fmaf(ua, c4.w, s.w);
  }
  return s;
}

// alpha_k of column c from [ q_k . v (16) | U^T y (16 k) ] and c_k = U^T q_k [k][16] (fp64, fixed order: every CTA of orth and
// update computes the same value)
__device__ __forceinline__ double ms_pre_alpha(const double* __restrict__ sums, const double* __restrict__ cvec, int k, int c) {
  double a = sums[c];
  for (int j = 0; j < k; ++j) a -= cvec[j * TP + c] * sums[TP + j * TP + c];
  return a;
}

// pre: X = D^-1/2 (Q - U c) = F^-T Q   (c = U^T Q, fp64 [k][16])
__global__ void __launch_bounds__(RP_THREADS)
ms_scale_kernel(const float* __restrict__ Qin, const double* __restrict__ cvec, const float* __restrict__ U, int k, float noise,
                const float* __restrict__ dvec, float* __restrict__ X, int64_t n, const int* __restrict__ done) {
  if (done && *done) return;
  extern __shared__ __align__(16) float msh[];
  float* us = msh;
  float* cs = msh + ms_urows(k) + RP_ROWS * TP;
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  for (int e = tid; e < k * TP; e += RP_THREADS) cs[e] = (float)cvec[e];
  for (int64_t r0 = (int64_t)blockIdx.x * RP_ROWS; r0 < n; r0 += (int64_t)gridDim.x * RP_ROWS) {
    ms_stage_u(U, k, r0, n, us);
    __syncthreads();
    const int64_t r = r0 + rl;
    if (r < n) {
      const float4 uc = ms_uc(us, k, cs, rl, cg);
      const float4 q = reinterpret_cast<const float4*>(Qin)[r * 4 + cg];
      const float rs = 1.f / sqrtf(dvec ? dvec[r] : noise);
      reinterpret_cast<float4*>(X)[r * 4 + cg] = make_float4((q.x - uc.x) * rs, (q.y - uc.y) * rs, (q.z - uc.z) * rs, (q.w - uc.w) * rs);
    }
    __syncthreads();
  }
}

// finish: v = K_hat q_k - beta_k q_{k-1} ; partials of q_k . v   (X unused, k = 0)
// PRE: y = D^-1/2 K_hat x_k ; v = y - beta_k q_{k-1} ; partials [ q_k . v | U^T y ]  (row pitch 16 (k + 1))
template <bool PRE>
__global__ void __launch_bounds__(RP_THREADS)
ms_finish_kernel(const float* __restrict__ kpart, int nsplit, int64_t rows_pad, float os, const float* __restrict__ pscale,
                 float noise, const float* __restrict__ dvec, const float* __restrict__ X, const float* __restrict__ Qcur,
                 const float* __restrict__ Qprev, float* __restrict__ V, int64_t n, const MsState* __restrict__ st, int kk,
                 const float* __restrict__ U, int k, float* __restrict__ part, const int* __restrict__ done,
                 const int* __restrict__ xbad) {
  if (*done) return;
  extern __shared__ __align__(16) float msh[];   // PRE: layout above; else the [64][16] reduction scratch
  float* us = msh;
  float* ys = msh + ms_urows(k);
  __shared__ __align__(16) float bk[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  if (tid < TP) bk[tid] = (float)st->beta[kk & 1][tid];
  __syncthreads();
  const float poison = *xbad ? __int_as_float(0x7fc00000) : 0.f;   // non-finite inputs: K.V is NaN in the reference
  const float4 b4 = reinterpret_cast<const float4*>(bk)[cg];
  float4 acc = make_float4(0, 0, 0, 0);
  float uacc[MS_KMAX / 16] = {};
  // PRE: the whole CTA walks every 64-row chunk r0 = r - rl (U staging, U^T reduction); else a thread stops after its last row
  for (int64_t r = (int64_t)blockIdx.x * RP_ROWS + rl; (PRE ? r - rl : r) < n; r += (int64_t)gridDim.x * RP_ROWS) {
    int nr = 0;
    if constexpr (PRE) nr = ms_stage_u(U, k, r - rl, n, us);
    float4 y = make_float4(0, 0, 0, 0);
    if (r < n) {
      y = khat_row(kpart, nsplit, rows_pad, os, pscale, poison, PRE ? X : Qcur, dvec, noise, r, cg);
      if constexpr (PRE) {
        const float rs = 1.f / sqrtf(dvec ? dvec[r] : noise);
        y = make_float4(y.x * rs, y.y * rs, y.z * rs, y.w * rs);
      }
      const float4 q = reinterpret_cast<const float4*>(Qcur)[r * 4 + cg];
      const float4 qp = reinterpret_cast<const float4*>(Qprev)[r * 4 + cg];
      float4 v;
      v.x = fmaf(-b4.x, qp.x, y.x); v.y = fmaf(-b4.y, qp.y, y.y); v.z = fmaf(-b4.z, qp.z, y.z); v.w = fmaf(-b4.w, qp.w, y.w);
      reinterpret_cast<float4*>(V)[r * 4 + cg] = v;
      acc.x = fmaf(q.x, v.x, acc.x); acc.y = fmaf(q.y, v.y, acc.y); acc.z = fmaf(q.z, v.z, acc.z); acc.w = fmaf(q.w, v.w, acc.w);
    }
    if constexpr (PRE) {
      reinterpret_cast<float4*>(ys)[rl * 4 + cg] = y;
      __syncthreads();
      ms_ut_acc(us, k, ys, nr, uacc);
      __syncthreads();
    }
  }
  float* out = part + (size_t)blockIdx.x * TP * (k + 1);
  block_reduce_cols(acc, msh, out);
  if constexpr (PRE) ms_ut_store(uacc, k, out + TP);
}

// orth: v -= alpha_k q_k ; partials of v . v   (sums[0..16) = alpha_k ; cvec, U unused, k = 0)
// PRE: v -= U (U^T y) + alpha_k q_k ; partials [ v . v | U^T v ]  (sums = [ q_k . v | U^T y ], cvec = c_k).  Without sums
// (start-up pass) V is only read: partials [ v . v | U^T v ] of the block as it is.
template <bool PRE>
__global__ void __launch_bounds__(RP_THREADS)
ms_orth_kernel(const double* __restrict__ sums, const double* __restrict__ cvec, const float* __restrict__ Qcur,
               float* __restrict__ V, int64_t n, const float* __restrict__ U, int k, float* __restrict__ part,
               const int* __restrict__ done) {
  if (done && *done) return;
  extern __shared__ __align__(16) float msh[];   // PRE: layout above; else the [64][16] reduction scratch
  float* us = msh;
  float* vs = msh + ms_urows(k);
  float* cs = vs + RP_ROWS * TP;
  __shared__ __align__(16) float al[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  const bool update = !PRE || sums != nullptr;   // false: the read-only start-up pass
  if (update) {
    if constexpr (PRE)
      for (int e = tid; e < k * TP; e += RP_THREADS) cs[e] = (float)sums[TP + e];
    if (tid < TP) al[tid] = (float)(PRE ? ms_pre_alpha(sums, cvec, k, tid) : sums[tid]);
  }
  __syncthreads();
  const float4 a4 = reinterpret_cast<const float4*>(al)[cg];
  float4 acc = make_float4(0, 0, 0, 0);
  float uacc[MS_KMAX / 16] = {};
  // PRE: the whole CTA walks every 64-row chunk r0 = r - rl (U staging, U^T reduction); else a thread stops after its last row
  for (int64_t r = (int64_t)blockIdx.x * RP_ROWS + rl; (PRE ? r - rl : r) < n; r += (int64_t)gridDim.x * RP_ROWS) {
    int nr = 0;
    if constexpr (PRE) {
      nr = ms_stage_u(U, k, r - rl, n, us);
      __syncthreads();
    }
    float4 v = make_float4(0, 0, 0, 0);
    if (r < n) {
      v = reinterpret_cast<const float4*>(V)[r * 4 + cg];
      if (update) {
        if constexpr (PRE) {
          const float4 uc = ms_uc(us, k, cs, rl, cg);
          v.x -= uc.x; v.y -= uc.y; v.z -= uc.z; v.w -= uc.w;
        }
        const float4 q = reinterpret_cast<const float4*>(Qcur)[r * 4 + cg];
        v.x = fmaf(-a4.x, q.x, v.x); v.y = fmaf(-a4.y, q.y, v.y); v.z = fmaf(-a4.z, q.z, v.z); v.w = fmaf(-a4.w, q.w, v.w);
        reinterpret_cast<float4*>(V)[r * 4 + cg] = v;
      }
      acc.x = fmaf(v.x, v.x, acc.x); acc.y = fmaf(v.y, v.y, acc.y); acc.z = fmaf(v.z, v.z, acc.z); acc.w = fmaf(v.w, v.w, acc.w);
    }
    if constexpr (PRE) {
      reinterpret_cast<float4*>(vs)[rl * 4 + cg] = v;
      __syncthreads();
      ms_ut_acc(us, k, vs, nr, uacc);
      __syncthreads();
    }
  }
  float* out = part + (size_t)blockIdx.x * TP * (k + 1);
  block_reduce_cols(acc, msh, out);
  if constexpr (PRE) ms_ut_store(uacc, k, out + TP);
}

// rotations + q_{k+1} + direction blocks + Z + stop rule.  sums = [ alpha_k (16) | beta_{k+1}^2 (16) ].
// Preconditioned (PRE): sums = [ q_k . v | U^T y ] (alpha_k through ms_pre_alpha with cprev = c_k), sums2 = [ v . v | U^T v ],
// Qcur = x_k = F^-T q_k (the direction recurrence runs on the F^-T images), and block 0 writes c_{k+1} = U^T v / beta_{k+1} to
// cnext (0 for a converged or broken-down column, whose q_{k+1} is 0).
// D holds 2 blocks per shift: at iteration kk, d_{k-1} is block 2q + ((kk + 1) & 1) and d_{k-2} is block 2q + (kk & 1); the new
// direction overwrites d_{k-2}.
template <bool PRE>
__global__ void __launch_bounds__(RP_THREADS)
ms_update_kernel(const double* __restrict__ sums, const double* __restrict__ sums2, const double* __restrict__ cprev,
                 double* __restrict__ cnext, int k, int kk, int Q, int t, float tol, const float* __restrict__ V,
                 const float* __restrict__ Qcur, float* __restrict__ Qnext, float* __restrict__ D, float* __restrict__ Z, int64_t n,
                 MsState* __restrict__ st) {
  if (st->done_iter < kk) return;
  __shared__ __align__(16) float cD[MS_QMAX * TP], cE[MS_QMAX * TP], cG[MS_QMAX * TP], cW[MS_QMAX * TP];
  __shared__ float aphi[MS_QMAX * TP];
  __shared__ __align__(16) float invb[TP];
  __shared__ int brk_s[TP], nan_s[TP];
  __shared__ double bnext_s[TP], alpha_s[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  const int P = kk & 1, Pn = P ^ 1;
  const bool writer = blockIdx.x == 0;
  if (tid < TP) {
    const double alpha = PRE ? ms_pre_alpha(sums, cprev, k, tid) : sums[tid];
    const double bn2 = PRE ? sums2[tid] : sums[TP + tid];
    double bn = sqrt(fmax(bn2, 0.0));
    const double bk = st->beta[P][tid];
    // breakdown: the Krylov space of this column is exhausted (also taken for a NaN column, which the nan flag reports)
    const bool brk = !(bn > 1e-6 * sqrt(alpha * alpha + bk * bk + bn * bn));
    if (brk) bn = 0.0;
    bnext_s[tid] = bn;
    alpha_s[tid] = alpha;
    brk_s[tid] = brk;
    nan_s[tid] = !(alpha == alpha && bn2 == bn2);
    invb[tid] = (brk || st->conv[P][tid]) ? 0.f : (float)(1.0 / bn);
  }
  __syncthreads();
  if (PRE && writer)
    for (int e = tid; e < k * TP; e += RP_THREADS) {
      const int c = e % TP;
      cnext[e] = (brk_s[c] || st->conv[P][c]) ? 0.0 : sums2[TP + e] / bnext_s[c];
    }
  for (int e = tid; e < Q * TP; e += RP_THREADS) {
    const int q = e / TP, c = e % TP;
    const double a = alpha_s[c] + st->tau[q];
    const double bk = st->beta[P][c], bn = bnext_s[c];
    const double c1 = st->c1[P][e], s1 = st->s1[P][e], c2 = st->c2[P][e], s2 = st->s2[P][e], pb = st->phibar[P][e];
    const double eps = s2 * bk, dbar = c2 * bk;           // G_{k-2} applied to (0, beta_k)
    const double delta = c1 * dbar + s1 * a;              // G_{k-1} applied to (dbar, alpha_k + tau_q)
    const double gbar = -s1 * dbar + c1 * a;
    const double gamma = hypot(gbar, bn);                 // G_k annihilates beta_{k+1}
    float kD = 0.f, kE = 0.f, kG = 0.f, kW = 0.f;
    double nc1 = c1, ns1 = s1, nc2 = c2, ns2 = s2, npb = pb;
    if (!st->conv[P][c] && gamma > 0.0) {
      const double cn = gbar / gamma, sn = bn / gamma;
      const double phi = cn * pb;
      npb = -sn * pb;
      kD = (float)(delta / gamma); kE = (float)(eps / gamma); kG = (float)(1.0 / gamma); kW = (float)(st->w[q] * phi);
      nc2 = c1; ns2 = s1; nc1 = cn; ns1 = sn;
    }
    cD[e] = kD; cE[e] = kE; cG[e] = kG; cW[e] = kW;
    aphi[e] = (float)fabs(npb);
    if (writer) {
      st->c1[Pn][e] = nc1; st->s1[Pn][e] = ns1; st->c2[Pn][e] = nc2; st->s2[Pn][e] = ns2; st->phibar[Pn][e] = npb;
    }
  }
  __syncthreads();
  // rows: q_{k+1}, new directions, Z
  const float4 ib = reinterpret_cast<const float4*>(invb)[cg];
  const int64_t blk = n * TP;
  for (int64_t r = (int64_t)blockIdx.x * RP_ROWS + rl; r < n; r += (int64_t)gridDim.x * RP_ROWS) {
    const int64_t o = r * 4 + cg;
    const float4 v = reinterpret_cast<const float4*>(V)[o];
    const float4 q = reinterpret_cast<const float4*>(Qcur)[o];
    // a converged or broken-down column gets q_{k+1} = 0 (select, so that a NaN v cannot leak through 0 * v)
    reinterpret_cast<float4*>(Qnext)[o] = make_float4(ib.x != 0.f ? v.x * ib.x : 0.f, ib.y != 0.f ? v.y * ib.y : 0.f,
                                                      ib.z != 0.f ? v.z * ib.z : 0.f, ib.w != 0.f ? v.w * ib.w : 0.f);
    float4 z = reinterpret_cast<float4*>(Z)[o];
    for (int s = 0; s < Q; ++s) {
      float4* d1p = reinterpret_cast<float4*>(D + (int64_t)(2 * s + (Pn)) * blk) + o;   // d_{k-1}
      float4* d2p = reinterpret_cast<float4*>(D + (int64_t)(2 * s + P) * blk) + o;      // d_{k-2} -> d_k
      const float4 d1 = *d1p, d2 = *d2p;
      const float4 kd = reinterpret_cast<const float4*>(cD)[s * 4 + cg], ke = reinterpret_cast<const float4*>(cE)[s * 4 + cg];
      const float4 kg = reinterpret_cast<const float4*>(cG)[s * 4 + cg], kw = reinterpret_cast<const float4*>(cW)[s * 4 + cg];
      float4 dn;
      dn.x = fmaf(kg.x, q.x, fmaf(-ke.x, d2.x, -kd.x * d1.x));
      dn.y = fmaf(kg.y, q.y, fmaf(-ke.y, d2.y, -kd.y * d1.y));
      dn.z = fmaf(kg.z, q.z, fmaf(-ke.z, d2.z, -kd.z * d1.z));
      dn.w = fmaf(kg.w, q.w, fmaf(-ke.w, d2.w, -kd.w * d1.w));
      *d2p = dn;
      z.x = fmaf(kw.x, dn.x, z.x); z.y = fmaf(kw.y, dn.y, z.y); z.z = fmaf(kw.z, dn.z, z.z); z.w = fmaf(kw.w, dn.w, z.w);
    }
    reinterpret_cast<float4*>(Z)[o] = z;
  }
  // bookkeeping (block 0): beta_{k+1}, convergence, stop rule
  if (writer && tid < 32) {
    const int c = tid;
    int conv = 1;
    if (c < TP) {
      float mx = 0.f;
      for (int s = 0; s < Q; ++s) {
        mx = fmaxf(mx, aphi[s * TP + c]);
        st->resid[s * TP + c] = aphi[s * TP + c];
      }
      conv = st->conv[P][c] || brk_s[c] || mx <= tol;
      st->conv[Pn][c] = conv;
      st->beta[Pn][c] = bnext_s[c];
    }
    const bool bad = kk == 0 && c < t && nan_s[c];
    const bool all = __all_sync(0xffffffffu, conv);
    const bool anybad = __any_sync(0xffffffffu, bad);
    if (c == 0) {
      st->iters = kk + 1;
      st->all_conv = all;
      if (anybad) st->nan_flag = 1;
      if (all || anybad) {
        st->done_iter = kk;
        __threadfence();
        st->done = 1;
      }
    }
  }
}

// Z[r][c] *= |b_c|: the product after the loop then gives OUT for the un-normalised right-hand side
__global__ void ms_scale_kernel(float* __restrict__ Z, const MsState* __restrict__ st, int64_t n) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n * TP) Z[idx] *= st->rhs_norm[idx % TP];
}

// U == nullptr: OUT = K_hat sum_q w_q (K_hat + tau_q I)^-1 B.  U [n][k]: OUT = K_hat F^-T sum_q w_q (A + tau_q I)^-1 B (header).
int ciq_run(gp_plan* p, const float* B, int64_t ldb, int t, const float* U, int k, const double* tau, const double* w, int Q,
            float tol, int max_iter, float* OUT, int64_t ldo, int* iters_out, float* resid_out) {
  GP_REQUIRE(p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  KronColsScope kcols(p, t);   // the Lanczos blocks' columns >= t stay zero
  const bool pre = U != nullptr || k != 0;
  if (pre) {
    GP_REQUIRE(U != nullptr && k >= 1 && k <= MS_KMAX, GP_E_SHAPE, "preconditioner factor U [n, k] with k in [1,%d] (k=%d, U %s)",
               MS_KMAX, k, U ? "set" : "null");
    GP_REQUIRE(p->noise_diag != nullptr || p->noise > 0.f, GP_E_SHAPE, "the preconditioned CIQ needs noise > 0");
  }
  GP_REQUIRE(p->same, GP_E_SHAPE, "CIQ needs a square operator (X2 == X1)");
  GP_REQUIRE(!(p->comm && p->comm->world > 1) && p->row_begin == 0 && p->row_count == p->n2, GP_E_SHAPE,
             "gp_ciq_sqrt_matmul is not supported on row-sharded plans");
  GP_REQUIRE(t >= 1 && t <= TP, GP_E_SHAPE, "CIQ handles 1..%d right-hand sides per call (t=%d)", TP, t);
  GP_REQUIRE(Q >= 1 && Q <= MS_QMAX, GP_E_SHAPE, "CIQ takes 1..%d quadrature shifts (Q=%d)", MS_QMAX, Q);
  GP_REQUIRE(tau != nullptr && w != nullptr, GP_E_SHAPE, "tau / w missing");
  for (int q = 0; q < Q; ++q)
    GP_REQUIRE(isfinite(tau[q]) && tau[q] >= 0.0 && isfinite(w[q]), GP_E_SHAPE,
               "quadrature shift %d: tau=%g must be finite and >= 0, w=%g finite", q, tau[q], w[q]);
  GP_REQUIRE(max_iter >= 1, GP_E_SHAPE, "max_iter must be >= 1");
  GP_REQUIRE(B != nullptr && OUT != nullptr && ldb >= t && ldo >= t, GP_E_SHAPE, "bad B / OUT (ldb=%lld, ldo=%lld, t=%d)",
             (long long)ldb, (long long)ldo, t);
  GP_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = p->stream;
  const int64_t n = p->n2;
  // the preconditioned row passes hold ~45 KB of shared memory (k = 128): 4 CTAs per SM
  const int G = (int)std::min<int64_t>(cdiv(n, RP_ROWS), (int64_t)(pre ? 4 : 8) * p->n_sm);
  const size_t blk = (size_t)n * TP;
  const int L = pre ? TP * (k + 1) : TP;   // partial row: [ dot (16) | U^T block (16 k) ]
  // workspace: q (2 blocks) | v | Z | directions (2 Q blocks) | x (preconditioned) | partials [2][G][L] | sums | tau, w | state
  // sums: [16] |b|^2 | [32] alpha | beta^2 ; preconditioned: [16] |b|^2 | A, B, start-up sums [3][L] | c_k buffer [16 k]
  const size_t vec_floats = blk * (4 + 2 * (size_t)Q + (pre ? 1 : 0));
  const size_t nsums = pre ? TP + 3 * (size_t)L + (size_t)TP * k : 48;
  const size_t off_part = vec_floats * sizeof(float);
  const size_t off_sums = off_part + sizeof(float) * 2 * (size_t)G * L;
  const size_t off_tw = off_sums + sizeof(double) * nsums;
  const size_t off_state = off_tw + sizeof(double) * 2 * MS_QMAX;
  GP_CHECK(p->msw.ensure(off_state + sizeof(MsState)));
  char* base = p->msw.as<char>();
  float* Qb[2] = {reinterpret_cast<float*>(base), reinterpret_cast<float*>(base) + blk};
  float* V = Qb[1] + blk;
  float* Z = V + blk;
  float* D = Z + blk;
  float* X = D + 2 * (size_t)Q * blk;   // x_k = F^-T q_k (preconditioned only)
  float* part1 = reinterpret_cast<float*>(base + off_part);
  float* part2 = part1 + (size_t)G * L;
  double* sums0 = reinterpret_cast<double*>(base + off_sums);   // [16] |b|^2
  double* sums = sums0 + TP;                                    // [32] alpha | beta^2
  double* sumsA = sums0 + TP;                                   // preconditioned: [ q.v | U^T y ]
  double* sumsB = sumsA + L;                                    //                 [ v.v | U^T v ]
  double* sumsI = sumsB + L;                                    //                 [ q_1.q_1 | U^T q_1 ]
  double* cbuf[2] = {sumsI + TP, sumsI + L};                    // c_k = U^T q_k by iteration parity (c_1 from the start-up pass)
  double* d_tw = reinterpret_cast<double*>(base + off_tw);
  MsState* S = reinterpret_cast<MsState*>(base + off_state);
  const int* done = &S->done;
  const float* dvec = p->noise_diag;

  double* h_tw = reinterpret_cast<double*>(static_cast<char*>(p->pinned) + PIN_CIQ_TW);
  for (int q = 0; q < Q; ++q) { h_tw[q] = tau[q]; h_tw[Q + q] = w[q]; }
  GP_CUDA(cudaMemcpyAsync(d_tw, h_tw, sizeof(double) * 2 * Q, cudaMemcpyHostToDevice, st));
  GP_CUDA(cudaMemsetAsync(D, 0, sizeof(float) * blk * 2 * Q, st));

  // ---- init ----
  cg_rhs_sq_launch(B, ldb, t, n, part1, G, st);
  cg_sum_launch(part1, G, TP, sums0, nullptr, st);
  ms_init_kernel<<<G, RP_THREADS, 0, st>>>(B, ldb, t, n, sums0, Q, d_tw, Qb[0], Qb[1], Z, S);
  p->launches += 3;
  const size_t shp = pre ? ms_pre_smem(k) : sizeof(float) * RP_ROWS * TP;
  if (pre) {   // c_1 = U^T q_1
    ms_orth_kernel<true><<<G, RP_THREADS, shp, st>>>(nullptr, nullptr, nullptr, Qb[0], n, U, k, part2, nullptr);
    cg_sum_launch(part2, G, L, sumsI, nullptr, st);
    p->launches += 2;
  }
  GP_CUDA(cudaGetLastError());

  // ---- iterations ----
  SolverLoop loop(p, "msMINRES", done, 0);
  GP_CHECK(loop.create_events());
  int status = GP_OK;
  bool finished = false;
  for (int kk = 0; kk < max_iter && !finished; ++kk) {
    float* Qcur = Qb[kk & 1];
    float* Qoth = Qb[(kk + 1) & 1];   // q_{k-1} on entry, q_{k+1} on exit
    if (pre) {
      const double* ck = cbuf[kk & 1];
      ms_scale_kernel<<<G, RP_THREADS, shp, st>>>(Qcur, ck, U, k, p->noise, dvec, X, n, done);
      if ((status = kmv_partials(p, X, done)) != GP_OK) break;
      ms_finish_kernel<true><<<G, RP_THREADS, shp, st>>>(p->partial.as<float>(), nslots(p), p->rows_pad, kernel_scale(p), part_scale_ptr(p),
                                                         p->noise, dvec, X, Qcur, Qoth, V, n, S, kk, U, k, part1, done, p->xbad);
      cg_sum_launch(part1, G, L, sumsA, done, st);
      ms_orth_kernel<true><<<G, RP_THREADS, shp, st>>>(sumsA, ck, Qcur, V, n, U, k, part2, done);
      cg_sum_launch(part2, G, L, sumsB, done, st);
      ms_update_kernel<true><<<G, RP_THREADS, 0, st>>>(sumsA, sumsB, ck, cbuf[(kk + 1) & 1], k, kk, Q, t, tol, V, X, Qoth, D, Z, n, S);
      p->launches += 6;
    } else {
      if ((status = kmv_partials(p, Qcur, done)) != GP_OK) break;
      ms_finish_kernel<false><<<G, RP_THREADS, shp, st>>>(p->partial.as<float>(), nslots(p), p->rows_pad, kernel_scale(p), part_scale_ptr(p),
                                                          p->noise, dvec, nullptr, Qcur, Qoth, V, n, S, kk, nullptr, 0, part1, done, p->xbad);
      cg_sum_launch(part1, G, TP, sums, done, st);
      ms_orth_kernel<false><<<G, RP_THREADS, shp, st>>>(sums, nullptr, Qcur, V, n, nullptr, 0, part2, done);
      cg_sum_launch(part2, G, TP, sums + TP, done, st);
      ms_update_kernel<false><<<G, RP_THREADS, 0, st>>>(sums, nullptr, nullptr, nullptr, 0, kk, Q, t, tol, V, Qcur, Qoth, D, Z, n, S);
      p->launches += 5;
    }
    finished = loop.finished(kk);
  }
  status = loop.launch_status(status);
  if (status == GP_OK) {
    // OUT = K_hat (|b| Z)   (preconditioned: Z already holds F^-T sum_q w_q (A + tau_q I)^-1 q_1)
    ms_scale_kernel<<<(unsigned)cdiv((int64_t)blk, 256), 256, 0, st>>>(Z, S, n);
    p->launches++;
    status = kmv_partials(p, Z, nullptr);
    if (status == GP_OK) status = kmv_finish_user(p, Z, OUT, ldo, t, 1);
  }
  if (status == GP_OK) {
    float* hs = reinterpret_cast<float*>(static_cast<char*>(p->pinned) + PIN_CIQ_OUT);
    cudaMemcpyAsync(hs, S->resid, MS_READBACK, cudaMemcpyDeviceToHost, st);
    status = loop.sync();
    if (status == GP_OK) {
      const int* hi = reinterpret_cast<const int*>(hs + MS_QMAX * TP);   // iters, nan_flag, all_conv
      if (iters_out) *iters_out = hi[0];
      if (resid_out)
        for (int q = 0; q < Q; ++q)
          for (int c = 0; c < t; ++c) resid_out[q * t + c] = hs[q * TP + c];
      if (hi[1]) {
        set_error("NaNs encountered when trying to perform matrix-vector multiplication");
        status = GP_E_NAN_MVM;
      } else if (!hi[2]) {
        float m = 0.f;
        for (int q = 0; q < Q; ++q)
          for (int c = 0; c < t; ++c) m = std::max(m, hs[q * TP + c]);
        set_error("msMINRES terminated in %d iterations with max relative residual %g which is larger than the tolerance of %g",
                  hi[0], m, tol);
        status = GP_W_NOT_CONVERGED;
      }
    }
  }
  return status;
}

}  // namespace gp

extern "C" int gp_ciq_sqrt_matmul(gp_plan* plan, const float* B, int64_t ldb, int t, const double* tau, const double* w, int Q,
                                  float tol, int max_iter, float* OUT, int64_t ldo, int* iters_out, float* resid_out) {
  GP_REQUIRE(plan != nullptr, GP_E_STATE, "null plan");
  return gp::ciq_run(plan, B, ldb, t, nullptr, 0, tau, w, Q, tol, max_iter, OUT, ldo, iters_out, resid_out);
}

extern "C" int gp_ciq_sqrt_matmul_precond(gp_plan* plan, const float* B, int64_t ldb, int t, const float* U, int k, const double* tau,
                                          const double* w, int Q, float tol, int max_iter, float* OUT, int64_t ldo, int* iters_out,
                                          float* resid_out) {
  GP_REQUIRE(plan != nullptr, GP_E_STATE, "null plan");
  GP_CHECK(gp::refuse_settings(plan, gp::CALL_CIQ_SQRT_MATMUL_PRECOND));
  GP_REQUIRE(U != nullptr, GP_E_SHAPE, "preconditioned CIQ without a factor U (k=%d)", k);
  return gp::ciq_run(plan, B, ldb, t, U, k, tau, w, Q, tol, max_iter, OUT, ldo, iters_out, resid_out);
}
