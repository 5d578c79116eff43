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
#include <math.h>

#include <algorithm>
#include <climits>

#include "gp_common.cuh"

namespace gp {

constexpr int MS_THREADS = 256;
constexpr int MS_ROWS = 64;     // rows per pass of a CTA (4 float4 column groups x 64 row lanes)
constexpr int MS_QMAX = 32;     // shifts per call

void cg_sum_launch(const float* in, int G, int L, double* out, const int* done, cudaStream_t st);   // cg.cu
void cg_rhs_sq_launch(const float* RHS, int64_t ldr, int t, int64_t n, float* part, int G, cudaStream_t st);

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

__device__ __forceinline__ void ms_block_reduce(float4 acc, float* red /*[MS_ROWS][TP]*/, float* out /*[TP] global*/) {
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  reinterpret_cast<float4*>(red)[rl * 4 + cg] = acc;
  __syncthreads();
  for (int s = MS_ROWS / 2; s > 0; s >>= 1) {
    if (rl < s) {
      float4 a = reinterpret_cast<float4*>(red)[rl * 4 + cg];
      float4 b = reinterpret_cast<float4*>(red)[(rl + s) * 4 + cg];
      reinterpret_cast<float4*>(red)[rl * 4 + cg] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    __syncthreads();
  }
  if (tid < TP) out[tid] = red[tid];
}

// q_1 = b / |b| (zero columns and columns >= t stay 0) ; q_0 = 0 ; Z = 0 ; scalar state of iteration 0
__global__ void __launch_bounds__(MS_THREADS)
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
    for (int e = tid; e < MS_QMAX * TP; e += MS_THREADS) {
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
  for (int64_t r = (int64_t)blockIdx.x * MS_ROWS + rl; r < n; r += (int64_t)gridDim.x * MS_ROWS) {
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

// v = os sum_s partial_s + D q_k - beta_k q_{k-1} ; partials of q_k . v
__global__ void __launch_bounds__(MS_THREADS)
ms_finish_kernel(const float* __restrict__ kpart, int nsplit, int64_t rows_pad, float os, const float* __restrict__ pscale,
                 float noise, const float* __restrict__ dvec, const float* __restrict__ Qcur, const float* __restrict__ Qprev,
                 float* __restrict__ V, int64_t n, const MsState* __restrict__ st, int kk, float* __restrict__ part,
                 const int* __restrict__ done, const int* __restrict__ xbad) {
  if (*done) return;
  __shared__ __align__(16) float red[MS_ROWS * TP];
  __shared__ __align__(16) float bk[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  if (tid < TP) bk[tid] = (float)st->beta[kk & 1][tid];
  __syncthreads();
  const float poison = *xbad ? __int_as_float(0x7fc00000) : 0.f;   // non-finite inputs: K.V is NaN in the reference
  const float4 b4 = reinterpret_cast<const float4*>(bk)[cg];
  float4 acc = make_float4(0, 0, 0, 0);
  for (int64_t r = (int64_t)blockIdx.x * MS_ROWS + rl; r < n; r += (int64_t)gridDim.x * MS_ROWS) {
    float4 s = make_float4(poison, poison, poison, poison);
    float osr = os;
    if (pscale) {   // kernel sum: slot sp belongs to the term with outputscale pscale[sp]
      for (int sp = 0; sp < nsplit; ++sp) {
        const float4 a = reinterpret_cast<const float4*>(kpart)[((int64_t)sp * rows_pad + r) * 4 + cg];
        const float w = pscale[sp];
        s.x = fmaf(w, a.x, s.x); s.y = fmaf(w, a.y, s.y); s.z = fmaf(w, a.z, s.z); s.w = fmaf(w, a.w, s.w);
      }
      osr = 1.f;
    } else {
      for (int sp = 0; sp < nsplit; ++sp) {
        const float4 a = reinterpret_cast<const float4*>(kpart)[((int64_t)sp * rows_pad + r) * 4 + cg];
        s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
      }
    }
    const float4 q = reinterpret_cast<const float4*>(Qcur)[r * 4 + cg];
    const float4 qp = reinterpret_cast<const float4*>(Qprev)[r * 4 + cg];
    const float d = dvec ? dvec[r] : noise;
    float4 x = make_float4(fmaf(d, q.x, osr * s.x), fmaf(d, q.y, osr * s.y), fmaf(d, q.z, osr * s.z), fmaf(d, q.w, osr * s.w));
    x.x = fmaf(-b4.x, qp.x, x.x); x.y = fmaf(-b4.y, qp.y, x.y); x.z = fmaf(-b4.z, qp.z, x.z); x.w = fmaf(-b4.w, qp.w, x.w);
    reinterpret_cast<float4*>(V)[r * 4 + cg] = x;
    acc.x = fmaf(q.x, x.x, acc.x); acc.y = fmaf(q.y, x.y, acc.y); acc.z = fmaf(q.z, x.z, acc.z); acc.w = fmaf(q.w, x.w, acc.w);
  }
  ms_block_reduce(acc, red, part + (size_t)blockIdx.x * TP);
}

// v -= alpha_k q_k ; partials of v . v     (sums[0..16) = alpha_k)
__global__ void __launch_bounds__(MS_THREADS)
ms_orth_kernel(const double* __restrict__ sums, const float* __restrict__ Qcur, float* __restrict__ V, int64_t n,
               float* __restrict__ part, const int* __restrict__ done) {
  if (*done) return;
  __shared__ __align__(16) float red[MS_ROWS * TP];
  __shared__ __align__(16) float al[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  if (tid < TP) al[tid] = (float)sums[tid];
  __syncthreads();
  const float4 a4 = reinterpret_cast<const float4*>(al)[cg];
  float4 acc = make_float4(0, 0, 0, 0);
  for (int64_t r = (int64_t)blockIdx.x * MS_ROWS + rl; r < n; r += (int64_t)gridDim.x * MS_ROWS) {
    const float4 q = reinterpret_cast<const float4*>(Qcur)[r * 4 + cg];
    float4 v = reinterpret_cast<float4*>(V)[r * 4 + cg];
    v.x = fmaf(-a4.x, q.x, v.x); v.y = fmaf(-a4.y, q.y, v.y); v.z = fmaf(-a4.z, q.z, v.z); v.w = fmaf(-a4.w, q.w, v.w);
    reinterpret_cast<float4*>(V)[r * 4 + cg] = v;
    acc.x = fmaf(v.x, v.x, acc.x); acc.y = fmaf(v.y, v.y, acc.y); acc.z = fmaf(v.z, v.z, acc.z); acc.w = fmaf(v.w, v.w, acc.w);
  }
  ms_block_reduce(acc, red, part + (size_t)blockIdx.x * TP);
}

// rotations + q_{k+1} + direction blocks + Z + stop rule.  sums = [ alpha_k (16) | beta_{k+1}^2 (16) ].
// D holds 2 blocks per shift: at iteration kk, d_{k-1} is block 2q + ((kk + 1) & 1) and d_{k-2} is block 2q + (kk & 1); the new
// direction overwrites d_{k-2}.
__global__ void __launch_bounds__(MS_THREADS)
ms_update_kernel(const double* __restrict__ sums, int kk, int Q, int t, float tol, const float* __restrict__ V,
                 const float* __restrict__ Qcur, float* __restrict__ Qnext, float* __restrict__ D, float* __restrict__ Z, int64_t n,
                 MsState* __restrict__ st) {
  if (st->done_iter < kk) return;
  __shared__ __align__(16) float cD[MS_QMAX * TP], cE[MS_QMAX * TP], cG[MS_QMAX * TP], cW[MS_QMAX * TP];
  __shared__ float aphi[MS_QMAX * TP];
  __shared__ __align__(16) float invb[TP];
  __shared__ int brk_s[TP];
  __shared__ double bnext_s[TP];
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  const int P = kk & 1, Pn = P ^ 1;
  const bool writer = blockIdx.x == 0;
  if (tid < TP) {
    const double alpha = sums[tid];
    double bn = sqrt(fmax(sums[TP + tid], 0.0));
    const double bk = st->beta[P][tid];
    // breakdown: the Krylov space of this column is exhausted (also taken for a NaN column, which the nan flag reports)
    const bool brk = !(bn > 1e-6 * sqrt(alpha * alpha + bk * bk + bn * bn));
    if (brk) bn = 0.0;
    bnext_s[tid] = bn;
    brk_s[tid] = brk;
    invb[tid] = (brk || st->conv[P][tid]) ? 0.f : (float)(1.0 / bn);
  }
  __syncthreads();
  for (int e = tid; e < Q * TP; e += MS_THREADS) {
    const int q = e / TP, c = e % TP;
    const double a = sums[c] + st->tau[q];
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
  for (int64_t r = (int64_t)blockIdx.x * MS_ROWS + rl; r < n; r += (int64_t)gridDim.x * MS_ROWS) {
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
    const bool bad = kk == 0 && c < t && !(sums[c] == sums[c] && sums[TP + c] == sums[TP + c]);
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

int ciq_run(gp_plan* p, const float* B, int64_t ldb, int t, const double* tau, const double* w, int Q, float tol, int max_iter,
            float* OUT, int64_t ldo, int* iters_out, float* resid_out) {
  GP_REQUIRE(p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
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
  const int G = (int)std::min<int64_t>(cdiv(n, MS_ROWS), (int64_t)8 * p->n_sm);
  const size_t blk = (size_t)n * TP;
  // workspace: q (2 blocks) | v | Z | directions (2 Q blocks) | partials [2][G][16] | sums [48] | tau, w | state
  const size_t vec_floats = blk * (4 + 2 * (size_t)Q);
  const size_t off_part = vec_floats * sizeof(float);
  const size_t off_sums = off_part + sizeof(float) * 2 * (size_t)G * TP;
  const size_t off_tw = off_sums + sizeof(double) * 48;
  const size_t off_state = off_tw + sizeof(double) * 2 * MS_QMAX;
  GP_CHECK(p->msw.ensure(off_state + sizeof(MsState)));
  char* base = p->msw.as<char>();
  float* Qb[2] = {reinterpret_cast<float*>(base), reinterpret_cast<float*>(base) + blk};
  float* V = Qb[1] + blk;
  float* Z = V + blk;
  float* D = Z + blk;
  float* part1 = reinterpret_cast<float*>(base + off_part);
  float* part2 = part1 + (size_t)G * TP;
  double* sums0 = reinterpret_cast<double*>(base + off_sums);   // [16] |b|^2
  double* sums = sums0 + TP;                                    // [32] alpha | beta^2
  double* d_tw = reinterpret_cast<double*>(base + off_tw);
  MsState* S = reinterpret_cast<MsState*>(base + off_state);
  const int* done = &S->done;
  const float* dvec = p->noise_diag;

  double* h_tw = reinterpret_cast<double*>(reinterpret_cast<char*>(p->pinned) + 8192);
  for (int q = 0; q < Q; ++q) { h_tw[q] = tau[q]; h_tw[Q + q] = w[q]; }
  GP_CUDA(cudaMemcpyAsync(d_tw, h_tw, sizeof(double) * 2 * Q, cudaMemcpyHostToDevice, st));
  GP_CUDA(cudaMemsetAsync(D, 0, sizeof(float) * blk * 2 * Q, st));

  // ---- init ----
  cg_rhs_sq_launch(B, ldb, t, n, part1, G, st);
  cg_sum_launch(part1, G, TP, sums0, nullptr, st);
  ms_init_kernel<<<G, MS_THREADS, 0, st>>>(B, ldb, t, n, sums0, Q, d_tw, Qb[0], Qb[1], Z, S);
  p->launches += 3;
  GP_CUDA(cudaGetLastError());

  // ---- iterations ----
  int* h_done = reinterpret_cast<int*>(p->pinned);   // [0..1] ring of done flags
  cudaEvent_t ev[2];
  GP_CUDA(cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming));
  GP_CUDA(cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming));
  int status = GP_OK;
  bool finished = false;
  for (int kk = 0; kk < max_iter && !finished; ++kk) {
    float* Qcur = Qb[kk & 1];
    float* Qoth = Qb[(kk + 1) & 1];   // q_{k-1} on entry, q_{k+1} on exit
    if ((status = kmv_partials(p, Qcur, done)) != GP_OK) break;
    ms_finish_kernel<<<G, MS_THREADS, 0, st>>>(p->partial.as<float>(), p->nparts, p->rows_pad, p->outputscale, part_scale_ptr(p),
                                               p->noise, dvec, Qcur, Qoth, V, n, S, kk, part1, done, p->xbad);
    cg_sum_launch(part1, G, TP, sums, done, st);
    ms_orth_kernel<<<G, MS_THREADS, 0, st>>>(sums, Qcur, V, n, part2, done);
    cg_sum_launch(part2, G, TP, sums + TP, done, st);
    ms_update_kernel<<<G, MS_THREADS, 0, st>>>(sums, kk, Q, t, tol, V, Qcur, Qoth, D, Z, n, S);
    p->launches += 5;
    // look-ahead stop check: read the flag of iteration kk after iteration kk + 1 has been enqueued
    cudaMemcpyAsync(&h_done[kk & 1], &S->done, sizeof(int), cudaMemcpyDeviceToHost, st);
    cudaEventRecord(ev[kk & 1], st);
    if (kk > 0) {
      cudaEventSynchronize(ev[(kk - 1) & 1]);
      if (h_done[(kk - 1) & 1]) finished = true;
    }
  }
  cudaError_t le = cudaGetLastError();
  if (status == GP_OK && le != cudaSuccess) {
    set_error("msMINRES launch failed: %s", cudaGetErrorString(le));
    status = GP_E_CUDA;
  }
  if (status == GP_OK) {
    // OUT = K_hat (|b| Z)
    ms_scale_kernel<<<(unsigned)cdiv((int64_t)blk, 256), 256, 0, st>>>(Z, S, n);
    p->launches++;
    status = kmv_partials(p, Z, nullptr);
    if (status == GP_OK) status = kmv_finish_user(p, Z, OUT, ldo, t, 1);
  }
  if (status == GP_OK) {
    float* hs = reinterpret_cast<float*>(reinterpret_cast<char*>(p->pinned) + 12288);
    const size_t nout = sizeof(float) * MS_QMAX * TP + 4 * sizeof(int);
    cudaMemcpyAsync(hs, S->resid, nout, cudaMemcpyDeviceToHost, st);
    cudaError_t se = cudaStreamSynchronize(st);
    if (se != cudaSuccess) {
      set_error("msMINRES execution failed: %s", cudaGetErrorString(se));
      status = GP_E_CUDA;
    } else {
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
  cudaEventDestroy(ev[0]);
  cudaEventDestroy(ev[1]);
  return status;
}

}  // namespace gp

extern "C" int gp_ciq_sqrt_matmul(gp_plan* plan, const float* B, int64_t ldb, int t, const double* tau, const double* w, int Q,
                                  float tol, int max_iter, float* OUT, int64_t ldo, int* iters_out, float* resid_out) {
  GP_REQUIRE(plan != nullptr, GP_E_STATE, "null plan");
  return gp::ciq_run(plan, B, ldb, t, tau, w, Q, tol, max_iter, OUT, ldo, iters_out, resid_out);
}
