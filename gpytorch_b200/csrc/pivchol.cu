// pivchol.cu -- pivoted-Cholesky preconditioner: greedy partial Cholesky, Woodbury factor, N(0,P) probes.
//
// gp_pivoted_cholesky restates linear_operator.functions._pivoted_cholesky (SURVEY.md Appendix A.3;
// surfaced at /root/reference/gpytorch/__init__.py:146-173): k sequential steps, each picks the largest
// remaining diagonal entry (ties -> earliest position in the running permutation, as torch.max over
// permuted_diags does), evaluates ONE kernel row on the fly, and applies the rank-m update.
// gp_precond_build restates AddedDiagLinearOperator._init_cache_for_constant_diag (Appendix A.4)
// through the k x k Cholesky of (L^T L + sigma^2 I) in fp64 instead of a QR of [L; sigma I]:
// W = L C^{-T} spans the same column space as Q[:n] with W W^T == Q Q^T, and
// log det P = log det(L^T L + sigma^2 I) + (n - k) log sigma^2.
// gp_ciq_precond_build turns the same L into the split factor U of the preconditioned CIQ sampler (minres.cu header).
#include <algorithm>
#include <cmath>

#include "deriv_table.cuh"
#include "gp_common.cuh"
#include "ski_rows.cuh"

namespace gp {

struct PcState {
  int done;        // stop rule fired (error <= tol, or NaN) -> later launches are no-ops
  int rank;        // steps completed
  int pivot;       // pivot (global row) selected for the NEXT step to run
  int nan_flag;
  float dpiv;      // sqrt(max diag) = L[m][pivot]
  float orig_err;  // max of the initial diagonal
  float err;
  unsigned int counter;  // last-block-done ticket (step-wise path)
  unsigned int bar;      // monotonic grid-barrier counter (persistent path)
};
static_assert(PIN_PC_STATE + sizeof(PcState) <= PIN_PRECOND, "PcState overflows its pinned slot");

constexpr int PC_THREADS = 128;

// One launch per step m (SURVEY.md Appendix A.3), fused: row update with the pivot chosen by the previous launch,
// then -- in the same pass -- the per-CTA (max, earliest permutation position, sum |diag|) over the remaining
// entries; the last CTA to finish reduces the partials, applies the stop rule and selects / swaps the next pivot.
//   L[m][j] = (K[pi, j] - sum_{q<m} L[q][pi] L[q][j]) / L[m][pi] ; diag[j] -= L[m][j]^2
template <int KIND>
__global__ void __launch_bounds__(PC_THREADS)
pc_step_kernel(const float* __restrict__ Z, int DP, float os, float* __restrict__ Lt, int64_t n, int m, int max_rank,
               float tol, float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos, PcState* __restrict__ st,
               int64_t* __restrict__ piv_out, float* __restrict__ pval, int* __restrict__ ppos, double* __restrict__ psum, CovParam cp) {
  if (st->done) return;
  extern __shared__ float sh[];
  float* zp = sh;           // [DP]
  float* lp = sh + DP;      // [m]   L[q][pivot]
  __shared__ float s_val[PC_THREADS];
  __shared__ int s_pos[PC_THREADS];
  __shared__ double s_sum[PC_THREADS];
  __shared__ bool s_last;
  const int tid = threadIdx.x;
  const int pi = st->pivot;
  const float dpiv = st->dpiv;
  for (int c = tid; c < DP; c += PC_THREADS) zp[c] = Z[(int64_t)pi * DP + c];
  for (int q = tid; q < m; q += PC_THREADS) lp[q] = Lt[(int64_t)q * n + pi];
  __syncthreads();
  const int64_t j = (int64_t)blockIdx.x * PC_THREADS + tid;
  float best = -INFINITY;
  int best_pos = 0x7fffffff;
  double asum = 0.0;
  if (j < n) {
    float* Lm = Lt + (int64_t)m * n;
    const int pj = pos[j];
    if (pj < m) {
      Lm[j] = 0.f;               // earlier pivots stay zero in this row
    } else if (pj == m) {
      Lm[j] = dpiv;              // the pivot itself
    } else {
      float s = 0.f;
      for (int c = 0; c < DP; ++c) {
        float df = zp[c] - Z[j * DP + c];
        s = fmaf(df, df, s);
      }
      float v = os * cov_from_arg<KIND>(-0.5f * s, cp);
      {
        // independent partial sums keep 8 L2 loads in flight per thread (the step is latency bound, not bandwidth bound)
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        int q = 0;
        for (; q + 4 <= m; q += 4) {
          s0 = fmaf(lp[q], Lt[(int64_t)q * n + j], s0);
          s1 = fmaf(lp[q + 1], Lt[(int64_t)(q + 1) * n + j], s1);
          s2 = fmaf(lp[q + 2], Lt[(int64_t)(q + 2) * n + j], s2);
          s3 = fmaf(lp[q + 3], Lt[(int64_t)(q + 3) * n + j], s3);
        }
        for (; q < m; ++q) s0 = fmaf(lp[q], Lt[(int64_t)q * n + j], s0);
        v -= (s0 + s1) + (s2 + s3);
      }
      v /= dpiv;
      Lm[j] = v;
      float dn = diag[j] - v * v;
      diag[j] = dn;
      if (dn != dn) { best = INFINITY; best_pos = -1; }  // NaN poisons the selection
      else { best = dn; best_pos = pj; }
      asum = fabs((double)dn);
    }
  }
  s_val[tid] = best; s_pos[tid] = best_pos; s_sum[tid] = asum;
  __syncthreads();
  for (int s = PC_THREADS / 2; s > 0; s >>= 1) {
    if (tid < s) {
      float v2 = s_val[tid + s]; int p2 = s_pos[tid + s];
      if (v2 > s_val[tid] || (v2 == s_val[tid] && p2 < s_pos[tid])) { s_val[tid] = v2; s_pos[tid] = p2; }
      s_sum[tid] += s_sum[tid + s];
    }
    __syncthreads();
  }
  if (tid == 0) {
    pval[blockIdx.x] = s_val[0]; ppos[blockIdx.x] = s_pos[0]; psum[blockIdx.x] = s_sum[0];
    __threadfence();
    unsigned int ticket = atomicAdd(&st->counter, 1u);
    s_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- last CTA: fixed-order reduction of the partials, stop rule, next pivot ----
  best = -INFINITY; best_pos = 0x7fffffff; asum = 0.0;
  for (int b = tid; b < (int)gridDim.x; b += PC_THREADS) {   // fixed assignment + fixed tree => deterministic
    float v2 = ((volatile float*)pval)[b]; int p2 = ((volatile int*)ppos)[b];
    if (v2 > best || (v2 == best && p2 < best_pos)) { best = v2; best_pos = p2; }
    asum += ((volatile double*)psum)[b];
  }
  s_val[tid] = best; s_pos[tid] = best_pos; s_sum[tid] = asum;
  __syncthreads();
  for (int s = PC_THREADS / 2; s > 0; s >>= 1) {
    if (tid < s) {
      float v2 = s_val[tid + s]; int p2 = s_pos[tid + s];
      if (v2 > s_val[tid] || (v2 == s_val[tid] && p2 < s_pos[tid])) { s_val[tid] = v2; s_pos[tid] = p2; }
      s_sum[tid] += s_sum[tid + s];
    }
    __syncthreads();
  }
  if (tid == 0) {
    const double tot = s_sum[0];
    st->counter = 0;
    st->rank = m + 1;
    const float err = (float)(tot / (double)st->orig_err);
    st->err = err;
    const float mx = s_val[0];
    const int pp = s_pos[0];
    // while (m == 0) or (m < max_iter and max(errors) > error_tol): will step m+1 run?
    if (m + 1 >= max_rank || (int64_t)(m + 1) >= n || !(err > tol)) {
      st->done = 1;
    } else if (pp < 0 || !(mx > 0.f)) {  // NaN / non-positive pivot: the reference ends up with NaNs in L
      st->nan_flag = 1;
      st->done = 1;
    } else {
      const int pi_new = perm[pp];
      const int pi_old = perm[m + 1];
      perm[m + 1] = pi_new; perm[pp] = pi_old;
      pos[pi_new] = m + 1; pos[pi_old] = pp;
      st->pivot = pi_new;
      st->dpiv = sqrtf(mx);
      piv_out[m + 1] = (int64_t)pi_new;
    }
  }
}

// ---- persistent variant: ALL steps in one cooperative launch -----------------------------------------------------------
// The step-wise path above pays a kernel launch + a last-CTA hand-off (~20 us) per step for ~2 us of work.  Here the
// grid stays resident (cudaLaunchCooperativeKernel guarantees co-residency), every thread owns the same rows in every
// step, and the steps are separated by one grid barrier (pc_persistent1_kernel below).  Arithmetic per entry is identical to
// pc_step_kernel.
__device__ __forceinline__ void pc_grid_barrier(unsigned int* bar, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    while (*((volatile unsigned int*)bar) < target) { }
    __threadfence();
  }
  __syncthreads();
}

constexpr int PCP_THREADS = 384;  // persistent kernel: one CTA per SM keeps the grid barrier small (one arrival per SM)
constexpr int PCP_RED = 512;

// Persistent kernel with ONE grid barrier per step.  Every CTA reduces the per-CTA partials itself (same loads, same tree => the
// same pivot, error and stop decision everywhere), so no second barrier ("state published"; the round-1 form had one) is
// needed: nothing global is read back except the partials, which are double-buffered by step parity (a CTA can only
// overwrite buffer m & 1 at step m + 2, i.e. after barrier m + 1, which every CTA reaches after it has read the step-m
// partials).  The permutation is not materialised: a row's position is private to the thread that owns the row (pos[j],
// patched by the owner when the row is swapped), the winning partial carries its row index, and the row that sits at
// position m + 1 (the one the swap moves to the winner's old position) announces itself through one more partial.
// Arithmetic and tie-breaking (earliest position) per entry are those of pc_step_kernel: bit-identical pivots.
// kernel sums (GP_BACKEND_SUM): K[pivot, j] = sum_t os_t k_t(|z_t,pivot - z_t,j|^2), every term with its own packed inputs
constexpr int PC_KIND_SUM = 64;
// SKI (GP_BACKEND_SKI): K[pivot, j] = s prod_k w_jk^T u_k[f_jk : f_jk + 4] with u of the pivot staged where the pivot row of Z sits
// (ski_rows.cuh); DP = sum_k G_k (0 on grids too large to stage u: the entries form it from the pivot's interpolation data)
constexpr int PC_KIND_SKI = 65;
// multitask (tasks.cu, kron.cu): K[r, r'] = s B[task(r), task(r')] k(|z_point(r) - z_point(r')|^2), covariance kind kind[0]; row r is
// point r / rep, task task[r] (Hadamard: rep = 1, task ids) or point r / T, task r mod T (Kronecker: rep = T, task = nullptr)
constexpr int PC_KIND_TASK = 66;
// derivative observations (deriv.cu): row r is point r / rep, component r mod rep (rep = d + 1); the entry of rows (a, b) is the
// RBF table's block entry (deriv_table.cuh) with u_c = dz_c w[c] and 1 / l_c^2 = il2[c] from dh (a DerivHyp on the device)
constexpr int PC_KIND_DERIV = 67;
// kernel products (GP_BACKEND_PRODUCT): K[pivot, j] = S prod_f k_f(|z_f,pivot - z_f,j|^2), the sum's staging and loop with a multiply
constexpr int PC_KIND_PRODUCT = 68;
// Matern-5/2 derivative observations: rows as PC_KIND_DERIV, entries from the Matern-5/2 table
constexpr int PC_KIND_M52GRAD = 69;
// additive GPs (additive.cu): K[pivot, j] = sum_{m=1}^{M} e_m(s_i k_i(z_pivot,i - z_j,i)) from the plan's packed rows
constexpr int PC_KIND_ADDITIVE = 70;
// spectral mixture kernels (spectral.cu): K[pivot, j] = S prod_d sum_q w_q e_qd cos_qd from the plan's packed rows
constexpr int PC_KIND_SPECTRAL = 71;
// Kronecker with observed rows (kron.cu, gp_plan_set_kron_observed): row r is interleaved row g = task[r] (the row map), point
// g / T, task g mod T; entries as PC_KIND_TASK
constexpr int PC_KIND_KRON_OBS = 72;
// Kronecker with several terms (kron.cu, gp_plan_set_kron_terms): row r is point r / rep, task r mod rep (rep = T); K[r, r'] =
// sum_t os_t B_t[a, b] k_t(|z_t,point(r) - z_t,point(r')|^2) with B the terms' T x T blocks back to back; the pivot rows of all
// terms are staged back to back, as PC_KIND_SUM does
constexpr int PC_KIND_KRON_TERMS = 73;
struct PcTerms {
  int n;
  int kind[4], DP[4];
  float os[4];
  const float* Z[4];
  const int* task;   // PC_KIND_TASK: task ids (user order; nullptr: r mod rep) and B [T][T]
  const float* B;
  int T;
  int rep;           // PC_KIND_TASK / PC_KIND_DERIV / PC_KIND_M52GRAD: rows per point
  const DerivHyp* dh;   // PC_KIND_DERIV / PC_KIND_M52GRAD
  AddHyp ah;            // PC_KIND_ADDITIVE
  SmHyp sh;             // PC_KIND_SPECTRAL
  CovParam cp[4];       // each term's (PC_KIND_SUM) or the plain plan's (cp[0]) covariance parameters: an RQ term's alpha
  int rank_stop;        // a polynomial plan or a sum with a polynomial term: a non-positive largest residual ends the factor
};
__device__ __forceinline__ int pc_task_of(const PcTerms& tt, int r) { return tt.task ? tt.task[r] : r % tt.rep; }
__device__ __forceinline__ float pc_cov_rt(int kind, float a, CovParam cp) {
  switch (kind) {
    case GP_RBF: return cov_from_arg<GP_RBF>(a, cp);
    case GP_MATERN12: return cov_from_arg<GP_MATERN12>(a, cp);
    case GP_MATERN32: return cov_from_arg<GP_MATERN32>(a, cp);
    case GP_RQ: return cov_from_arg<RQ_K>(a, cp);
    default: return cov_from_arg<GP_MATERN52>(a, cp);
  }
}
// the initial diagonal of a plain polynomial plan (tt.n = 1) or of a sum with a polynomial term, term by term in term order:
// os_t for a stationary term, os_t (|x_j|^2 + c_t)^p_t for a polynomial one; identity permutation; then pc_first_pivot_kernel
__global__ void pc_init_dot_kernel(const PcTerms tt, float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos, int64_t n) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  float v = 0.f;
  for (int t = 0; t < tt.n; ++t) {
    const float* z = tt.Z[t] + j * tt.DP[t];
    v = fmaf(tt.os[t], tt.kind[t] == GP_POLY ? cov_from_arg<POLY_K>(poly_arg(z, z, tt.DP[t], tt.cp[t].offset), tt.cp[t]) : 1.f, v);
  }
  diag[j] = v;
  perm[j] = (int)j;
  pos[j] = (int)j;
}

struct PcPart {
  double sum;
  float val;
  int pos, idx, old;
};

template <int KIND>
__global__ void __launch_bounds__(PCP_THREADS)
pc_persistent1_kernel(const float* __restrict__ Z, int DP, float os, float* Lt, int64_t n, int max_rank, float tol,
                      float* diag, int* pos, PcState* st, int64_t* piv_out, PcPart* part, const PcTerms tt, const SkiRows sk) {
  extern __shared__ float sh[];
  float* zp = sh;
  float* lp = sh + DP;
  float* col = lp + max_rank;
  __shared__ float s_val[PCP_RED];
  __shared__ int s_pos[PCP_RED];
  __shared__ int s_idx[PCP_RED];
  __shared__ double s_sum[PCP_RED];
  __shared__ int s_old;
  const int tid = threadIdx.x;
  const int G = (int)gridDim.x;
  if (tid < PCP_RED - PCP_THREADS) {
    s_val[PCP_THREADS + tid] = -INFINITY; s_pos[PCP_THREADS + tid] = 0x7fffffff; s_idx[PCP_THREADS + tid] = -1; s_sum[PCP_THREADS + tid] = 0.0;
  }
  const int64_t stride = (int64_t)G * PCP_THREADS;
  const int64_t jfirst = (int64_t)blockIdx.x * PCP_THREADS + tid;
  // CTA-uniform running state (identical in every CTA)
  int pi = st->pivot;                 // pivot row of the step about to run (position m)
  float dpiv = st->dpiv;
  const float orig_err = st->orig_err;
  int fx_new = -1, fx_old = -1, fx_pp = 0;   // pending position patches from the previous selection
  auto better = [](float v2, int p2, float v1, int p1) { return v2 > v1 || (v2 == v1 && p2 < p1); };
  for (int m = 0; m < max_rank; ++m) {
    if (tid == 0) s_old = -1;
    if (KIND == PC_KIND_SUM || KIND == PC_KIND_PRODUCT) {   // DP = sum of the terms' widths: the pivot rows of all terms back to back
      int off = 0;
      for (int t = 0; t < tt.n; ++t) {
        for (int c = tid; c < tt.DP[t]; c += PCP_THREADS) zp[off + c] = tt.Z[t][(int64_t)pi * tt.DP[t] + c];
        off += tt.DP[t];
      }
    } else if (KIND == PC_KIND_SKI) {
      ski_stage_u(sk, pi, zp, tid, PCP_THREADS);
    } else if constexpr (KIND == PC_KIND_KRON_OBS) {
      const int64_t zr = tt.task[pi] / tt.T;
      for (int c = tid; c < DP; c += PCP_THREADS) zp[c] = Z[zr * DP + c];
    } else if constexpr (KIND == PC_KIND_KRON_TERMS) {
      const int64_t zr = pi / tt.rep;
      int off = 0;
      for (int t = 0; t < tt.n; ++t) {
        for (int c = tid; c < tt.DP[t]; c += PCP_THREADS) zp[off + c] = tt.Z[t][zr * tt.DP[t] + c];
        off += tt.DP[t];
      }
    } else {
      const int64_t zr = (KIND == PC_KIND_TASK || KIND == PC_KIND_DERIV || KIND == PC_KIND_M52GRAD) ? pi / tt.rep : pi;
      for (int c = tid; c < DP; c += PCP_THREADS) zp[c] = Z[zr * DP + c];
    }
    for (int q = tid; q < m; q += PCP_THREADS) lp[q] = __ldcg(Lt + (int64_t)q * n + pi);   // written by another SM, before the last barrier
    __syncthreads();
    float best = -INFINITY;
    int best_pos = 0x7fffffff, best_idx = -1;
    double asum = 0.0;
    float* Lm = Lt + (int64_t)m * n;
    for (int64_t j = jfirst; j < n; j += stride) {
      int pj = pos[j];                                   // owner-private
      if ((int)j == fx_new) { pj = m; pos[j] = m; }      // pos[pi_new] = m (this step's pivot)
      else if ((int)j == fx_old) { pj = fx_pp; pos[j] = fx_pp; }
      if (pj == m + 1) s_old = (int)j;                   // exactly one thread of the grid
      const bool cached = (j == jfirst);
      if (pj < m) {
        Lm[j] = 0.f;
        if (cached) col[m * PCP_THREADS + tid] = 0.f;
      } else if (pj == m) {
        Lm[j] = dpiv;
        if (cached) col[m * PCP_THREADS + tid] = dpiv;
      } else {
        float v;
        if (KIND == PC_KIND_SUM) {
          v = 0.f;
          int off = 0;
          for (int t = 0; t < tt.n; ++t) {
            const float* zj = tt.Z[t] + j * tt.DP[t];
            if (tt.kind[t] == GP_POLY) {   // a polynomial term: a = x_pivot . x_j + c
              v = fmaf(tt.os[t], cov_from_arg<POLY_K>(poly_arg(zp + off, zj, tt.DP[t], tt.cp[t].offset), tt.cp[t]), v);
              off += tt.DP[t];
              continue;
            }
            float s = 0.f;
            for (int c = 0; c < tt.DP[t]; ++c) {
              float df = zp[off + c] - zj[c];
              s = fmaf(df, df, s);
            }
            v = fmaf(tt.os[t], pc_cov_rt(tt.kind[t], -0.5f * s, tt.cp[t]), v);
            off += tt.DP[t];
          }
        } else if (KIND == PC_KIND_PRODUCT) {
          v = os;
          int off = 0;
          for (int t = 0; t < tt.n; ++t) {
            const float* zj = tt.Z[t] + j * tt.DP[t];
            float s = 0.f;
            for (int c = 0; c < tt.DP[t]; ++c) {
              float df = zp[off + c] - zj[c];
              s = fmaf(df, df, s);
            }
            v *= pc_cov_rt(tt.kind[t], -0.5f * s, CovParam{});
            off += tt.DP[t];
          }
        } else if (KIND == PC_KIND_SKI) {
          v = ski_entry(sk, zp, pi, j);
        } else if (KIND == PC_KIND_ADDITIVE) {
          v = add_pair_rt(tt.ah, zp, Z + j * DP);
        } else if (KIND == PC_KIND_SPECTRAL) {
          v = sm_pair(tt.sh, zp, Z + j * DP);
        } else if (KIND == PC_KIND_TASK) {
          const float* zj = Z + (int64_t)((int)j / tt.rep) * DP;
          float s = 0.f;
          for (int c = 0; c < DP; ++c) {
            float df = zp[c] - zj[c];
            s = fmaf(df, df, s);
          }
          v = os * tt.B[pc_task_of(tt, pi) * tt.T + pc_task_of(tt, (int)j)] * pc_cov_rt(tt.kind[0], -0.5f * s, CovParam{});
        } else if constexpr (KIND == PC_KIND_KRON_OBS) {
          const int gp_ = tt.task[pi], gj = tt.task[j];
          const float* zj = Z + (int64_t)(gj / tt.T) * DP;
          float s = 0.f;
          for (int c = 0; c < DP; ++c) {
            float df = zp[c] - zj[c];
            s = fmaf(df, df, s);
          }
          v = os * tt.B[(gp_ % tt.T) * tt.T + gj % tt.T] * pc_cov_rt(tt.kind[0], -0.5f * s, CovParam{});
        } else if constexpr (KIND == PC_KIND_KRON_TERMS) {
          const int64_t zr = (int)j / tt.rep;
          const int a = pi % tt.rep, b = (int)j % tt.rep;
          v = 0.f;
          int off = 0;
          for (int t = 0; t < tt.n; ++t) {
            const float* zj = tt.Z[t] + zr * tt.DP[t];
            float s = 0.f;
            for (int c = 0; c < tt.DP[t]; ++c) {
              float df = zp[off + c] - zj[c];
              s = fmaf(df, df, s);
            }
            v = fmaf(tt.os[t] * tt.B[(t * tt.T + a) * tt.T + b], pc_cov_rt(tt.kind[t], -0.5f * s, CovParam{}), v);
            off += tt.DP[t];
          }
        } else if (KIND == PC_KIND_DERIV || KIND == PC_KIND_M52GRAD) {
          using K = DerivTable<KIND == PC_KIND_M52GRAD ? GP_MATERN52 : GP_RBF>;
          const float* zj = Z + (int64_t)((int)j / tt.rep) * DP;
          float s = 0.f;
          for (int c = 0; c < DP; ++c) {
            float df = zp[c] - zj[c];
            s = fmaf(df, df, s);
          }
          const int a = pi % tt.rep, b = (int)j % tt.rep;
          const float ua = a ? (zp[a - 1] - zj[a - 1]) * tt.dh->w[a - 1] : 0.f;
          const float ub = b ? (zp[b - 1] - zj[b - 1]) * tt.dh->w[b - 1] : 0.f;
          v = K::entry(K::pair(s).scaled(os), a, b, ua, ub, *tt.dh);
        } else if constexpr (KIND == POLY_K) {
          v = os * cov_from_arg<POLY_K>(poly_arg(zp, Z + j * DP, DP, tt.cp[0].offset), tt.cp[0]);
        } else {
          float s = 0.f;
          for (int c = 0; c < DP; ++c) {
            float df = zp[c] - Z[j * DP + c];
            s = fmaf(df, df, s);
          }
          v = os * cov_from_arg<(KIND >= PC_KIND_SUM ? GP_RBF : KIND)>(-0.5f * s, tt.cp[0]);
        }
        {
          float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
          int q = 0;
          if (cached) {
            const float* cj = col + tid;
            for (; q + 4 <= m; q += 4) {
              s0 = fmaf(lp[q], cj[q * PCP_THREADS], s0);
              s1 = fmaf(lp[q + 1], cj[(q + 1) * PCP_THREADS], s1);
              s2 = fmaf(lp[q + 2], cj[(q + 2) * PCP_THREADS], s2);
              s3 = fmaf(lp[q + 3], cj[(q + 3) * PCP_THREADS], s3);
            }
            for (; q < m; ++q) s0 = fmaf(lp[q], cj[q * PCP_THREADS], s0);
          } else {
            for (; q + 4 <= m; q += 4) {
              s0 = fmaf(lp[q], Lt[(int64_t)q * n + j], s0);
              s1 = fmaf(lp[q + 1], Lt[(int64_t)(q + 1) * n + j], s1);
              s2 = fmaf(lp[q + 2], Lt[(int64_t)(q + 2) * n + j], s2);
              s3 = fmaf(lp[q + 3], Lt[(int64_t)(q + 3) * n + j], s3);
            }
            for (; q < m; ++q) s0 = fmaf(lp[q], Lt[(int64_t)q * n + j], s0);
          }
          v -= (s0 + s1) + (s2 + s3);
        }
        v /= dpiv;
        Lm[j] = v;
        if (cached) col[m * PCP_THREADS + tid] = v;
        const float dn = diag[j] - v * v;
        diag[j] = dn;
        float cv; int cp;
        if (dn != dn) { cv = INFINITY; cp = -1; }
        else { cv = dn; cp = pj; }
        if (better(cv, cp, best, best_pos)) { best = cv; best_pos = cp; best_idx = (int)j; }
        asum += fabs((double)dn);
      }
    }
    s_val[tid] = best; s_pos[tid] = best_pos; s_idx[tid] = best_idx; s_sum[tid] = asum;
    __syncthreads();
    for (int s = PCP_RED / 2; s > 0; s >>= 1) {
      if (tid < s && tid + s < PCP_RED) {
        if (better(s_val[tid + s], s_pos[tid + s], s_val[tid], s_pos[tid])) { s_val[tid] = s_val[tid + s]; s_pos[tid] = s_pos[tid + s]; s_idx[tid] = s_idx[tid + s]; }
        s_sum[tid] += s_sum[tid + s];
      }
      __syncthreads();
    }
    PcPart* mine = part + (size_t)(m & 1) * G;
    if (tid == 0) {
      PcPart pp; pp.sum = s_sum[0]; pp.val = s_val[0]; pp.pos = s_pos[0]; pp.idx = s_idx[0]; pp.old = s_old;
      mine[blockIdx.x] = pp;
    }
    pc_grid_barrier(&st->bar, (unsigned)(m + 1) * gridDim.x);   // all partials of step m are visible
    best = -INFINITY; best_pos = 0x7fffffff; best_idx = -1; asum = 0.0;
    int old = -1;
    for (int b = tid; b < G; b += PCP_THREADS) {   // fixed assignment + fixed tree => deterministic, identical in every CTA
      const PcPart* q = mine + b;
      const float v2 = __ldcg(&q->val); const int p2 = __ldcg(&q->pos);
      if (better(v2, p2, best, best_pos)) { best = v2; best_pos = p2; best_idx = __ldcg(&q->idx); }
      asum += __ldcg(&q->sum);
      old = max(old, __ldcg(&q->old));
    }
    s_val[tid] = best; s_pos[tid] = best_pos; s_idx[tid] = best_idx; s_sum[tid] = asum;
    if (old >= 0) s_old = old;     // at most one thread of the CTA (after the loop barrier below: s_old is re-read only then)
    __syncthreads();
    for (int s = PCP_RED / 2; s > 0; s >>= 1) {
      if (tid < s) {
        if (better(s_val[tid + s], s_pos[tid + s], s_val[tid], s_pos[tid])) { s_val[tid] = s_val[tid + s]; s_pos[tid] = s_pos[tid + s]; s_idx[tid] = s_idx[tid + s]; }
        s_sum[tid] += s_sum[tid + s];
      }
      __syncthreads();
    }
    const double tot = s_sum[0];
    const float err = (float)(tot / (double)orig_err);
    const float mx = s_val[0];
    const int ppw = s_pos[0], inew = s_idx[0], iold = s_old;
    bool stop = false, nan = false;
    if (m + 1 >= max_rank || (int64_t)(m + 1) >= n || !(err > tol)) stop = true;
    else if (ppw < 0 || !(mx > 0.f)) {   // NaN, or nothing positive left: on a polynomial operator (rank_stop) its rank is spent
      stop = true;
      nan = (KIND == POLY_K || KIND == PC_KIND_SUM) ? (ppw < 0 || !tt.rank_stop) : true;
    }
    if (blockIdx.x == 0 && tid == 0) {
      st->rank = m + 1;
      st->err = err;
      if (stop) st->done = 1;
      if (nan) st->nan_flag = 1;
      if (!stop) { st->pivot = inew; st->dpiv = sqrtf(mx); piv_out[m + 1] = (int64_t)inew; }
    }
    if (stop) break;
    pi = inew; dpiv = sqrtf(mx);
    fx_new = inew; fx_old = (iold == inew) ? -1 : iold; fx_pp = ppw;
    __syncthreads();   // s_val / s_old are rewritten at the top of the next step
  }
}

__global__ void pc_init_kernel(float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos, int64_t n, float os,
                               PcState* __restrict__ st, int64_t* __restrict__ piv_out) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j == 0) {
    // the initial diagonal of a stationary kernel is constant: torch.max returns the first entry -> pivot 0
    st->done = 0; st->rank = 0; st->pivot = 0; st->nan_flag = (os > 0.f) ? 0 : 1; st->dpiv = sqrtf(os);
    st->orig_err = os; st->err = 0.f; st->counter = 0u; st->bar = 0u;
    piv_out[0] = 0;
  }
  if (j >= n) return;
  diag[j] = os;  // _approx_diagonal of a stationary kernel
  perm[j] = (int)j;
  pos[j] = (int)j;
}

// SKI: the initial diagonal is not constant.  diag[j] = K_ski(j, j), identity permutation; then pc_first_pivot_kernel
__global__ void pc_init_ski_kernel(const SkiRows sk, float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos, int64_t n) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  diag[j] = ski_diag_entry(sk, j);
  perm[j] = (int)j;
  pos[j] = (int)j;
}

// multitask: diag[j] = s B[t_j, t_j] (not constant across tasks), identity permutation; then pc_first_pivot_kernel
__global__ void pc_init_task_kernel(const PcTerms tt, float os, float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos,
                                    int64_t n) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int a = pc_task_of(tt, (int)j);
  diag[j] = os * tt.B[a * tt.T + a];
  perm[j] = (int)j;
  pos[j] = (int)j;
}

// Kronecker with observed rows: diag[j] = s B[a, a], a = rowmap[j] mod T (tt.task = the row map); then pc_first_pivot_kernel
__global__ void pc_init_kron_obs_kernel(const PcTerms tt, float os, float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos,
                                        int64_t n) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int a = tt.task[j] % tt.T;
  diag[j] = os * tt.B[a * tt.T + a];
  perm[j] = (int)j;
  pos[j] = (int)j;
}

// Kronecker with several terms: diag[j] = sum_t os_t B_t[a, a], a = j mod T (not constant across tasks); then pc_first_pivot_kernel
__global__ void pc_init_kron_terms_kernel(const PcTerms tt, float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos,
                                          int64_t n) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int a = (int)(j % tt.rep);
  float v = 0.f;
  for (int t = 0; t < tt.n; ++t) v = fmaf(tt.os[t], tt.B[(t * tt.T + a) * tt.T + a], v);
  diag[j] = v;
  perm[j] = (int)j;
  pos[j] = (int)j;
}

// derivative observations: diag[j] = s (value rows), c s / l_b^2 (derivative rows b; c = the table's DIAG); then
// pc_first_pivot_kernel
__global__ void pc_init_deriv_kernel(const PcTerms tt, float os, float c, float* __restrict__ diag, int* __restrict__ perm,
                                     int* __restrict__ pos, int64_t n) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int b = (int)(j % tt.rep);
  diag[j] = b ? os * (c * tt.dh->il2[b - 1]) : os;
  perm[j] = (int)j;
  pos[j] = (int)j;
}

// one CTA: first pivot = argmax of the diagonal, earliest index among equal maxima (torch.max over the whole diagonal), moved
// to position 0; orig_err = that maximum (oracle/linalg.pivoted_cholesky).  A NaN or a non-positive maximum stops at once.
constexpr int PC_FIRST_THREADS = 1024;
__global__ void __launch_bounds__(PC_FIRST_THREADS)
pc_first_pivot_kernel(const float* __restrict__ diag, int* __restrict__ perm, int* __restrict__ pos, int64_t n, PcState* __restrict__ st,
                      int64_t* __restrict__ piv_out) {
  __shared__ float s_val[PC_FIRST_THREADS];
  __shared__ int s_idx[PC_FIRST_THREADS];
  const int tid = threadIdx.x;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int64_t j = tid; j < n; j += PC_FIRST_THREADS) {   // ascending j per thread: strict > keeps the earliest
    const float v = diag[j];
    const float cv = (v != v) ? INFINITY : v;           // NaN wins and is reported below
    if (cv > best) { best = cv; bi = (int)j; }
  }
  s_val[tid] = best; s_idx[tid] = bi;
  __syncthreads();
  for (int s = PC_FIRST_THREADS / 2; s > 0; s >>= 1) {
    if (tid < s) {
      const float v2 = s_val[tid + s]; const int i2 = s_idx[tid + s];
      if (v2 > s_val[tid] || (v2 == s_val[tid] && i2 < s_idx[tid])) { s_val[tid] = v2; s_idx[tid] = i2; }
    }
    __syncthreads();
  }
  if (tid == 0) {
    const int im = s_idx[0];
    const float mx = diag[im];
    st->done = 0; st->rank = 0; st->pivot = im; st->nan_flag = (mx > 0.f && mx < INFINITY) ? 0 : 1; st->dpiv = sqrtf(mx);
    st->orig_err = mx; st->err = 0.f; st->counter = 0u; st->bar = 0u;
    piv_out[0] = im;
    perm[0] = im; perm[im] = 0;   // the swap of step 0 (im == 0: no-op)
    pos[0] = im; pos[im] = 0;
  }
}

// ---- preconditioner factor ---------------------------------------------------------------------
// Gpart[z][a][b] = sum_{j in slice z} L[a][j] L[b][j] s_j     (s_j = 1, or 1 / d_j for a per-row noise diagonal)
// 64 x 64 output tiles, 4 x 4 register tiles per thread.  Products and sums run in fp32 over chunks of 64 columns (<= 64 terms of
// magnitude <= outputscale: absolute error ~1e-6 per chunk), every chunk is then added to fp64 accumulators: the error of G
// stays orders of magnitude below the noise floor it is compared with in  log det P = log det(L^T L + sigma^2 I) + ...  (an
// error E in G shifts log det P by ~tr(E) / sigma^2), at a fraction of the cost of the all-fp64 product of round 1 (0.38 ms at C2).
constexpr int GT = 64;
__global__ void __launch_bounds__(256)
gram_kernel(const float* __restrict__ Lt, int k, int64_t n, int64_t jslice, const float* __restrict__ dvec, double* __restrict__ Gpart) {
  if (blockIdx.x > blockIdx.y) return;   // lower triangle of tiles only; the mirror image is written below
  __shared__ __align__(16) float As[32][GT + 4];   // [column][row of L^T = index a]
  __shared__ __align__(16) float Bs[32][GT + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int a0 = blockIdx.y * GT, b0 = blockIdx.x * GT;
  const int64_t j_begin = (int64_t)blockIdx.z * jslice, j_end = min(n, j_begin + jslice);
  double acc64[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc64[i][j] = 0.0;
  for (int64_t j0 = j_begin; j0 < j_end; j0 += 64) {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int hf = 0; hf < 2; ++hf) {
      const int64_t jb = j0 + hf * 32;
      __syncthreads();
      for (int e = tid; e < GT * 32; e += 256) {
        const int r = e >> 5, cc = e & 31;
        const int64_t j = jb + cc;
        const bool ok = j < j_end;
        const float sc = (ok && dvec) ? 1.f / dvec[j] : 1.f;
        As[cc][r] = (ok && a0 + r < k) ? Lt[(int64_t)(a0 + r) * n + j] * sc : 0.f;
        Bs[cc][r] = (ok && b0 + r < k) ? Lt[(int64_t)(b0 + r) * n + j] : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int cc = 0; cc < 32; ++cc) {
        const float4 av = *reinterpret_cast<const float4*>(&As[cc][ty * 4]);
        const float4 bv = *reinterpret_cast<const float4*>(&Bs[cc][tx * 4]);
        const float a4[4] = {av.x, av.y, av.z, av.w}, b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a4[i], b4[j], acc[i][j]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc64[i][j] += (double)acc[i][j];
  }
  double* G = Gpart + (int64_t)blockIdx.z * k * k;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int a = a0 + ty * 4 + i, b = b0 + tx * 4 + j;
      if (a < k && b < k) {
        G[(int64_t)a * k + b] = acc64[i][j];
        if (blockIdx.x != blockIdx.y) G[(int64_t)b * k + a] = acc64[i][j];
      }
    }
}

// single CTA: G = sum_z Gpart + noise I ; in-place lower Cholesky C ; logdet
// diag_add = sigma^2 and logdet_tail = (n - k) log sigma^2 for the constant diagonal; 1 and sum_j log d_j for a per-row diagonal
// (then G = L^T D^-1 L and log det P = log det(I + L^T D^-1 L) + sum log d)
__global__ void chol_small_kernel(const double* __restrict__ Gpart, int nz, int k, double diag_add, const double* __restrict__ logdet_tail,
                                  double* __restrict__ C, double* __restrict__ logdet_out, int* __restrict__ fail) {
  extern __shared__ double G[];  // [k][k]
  const int tid = threadIdx.x;
  for (int e = tid; e < k * k; e += blockDim.x) {
    double s = 0.0;
    for (int z = 0; z < nz; ++z) s += Gpart[(int64_t)z * k * k + e];
    if (e / k == e % k) s += diag_add;
    G[e] = s;
  }
  __syncthreads();
  // Right-looking factorisation with ONE barrier per step: the scaled column j goes straight to the output (nobody reads it
  // back), the trailing update uses the unscaled column and 1 / d_jj:  G[i][l] -= G[i][j] G[l][j] / d_jj.
  double ld = 0.0;
  for (int j = 0; j < k; ++j) {
    double d = G[j * k + j];
    if (!(d > 0.0)) { if (tid == 0) *fail = 1; d = 1e-300; }
    const double rinv = 1.0 / d;
    if (tid == 0) ld += log(d);
    if (tid >= 256) {   // upper half of the CTA also writes column j of C (rows j..k-1) and the zeros above the diagonal
      const double rs = 1.0 / sqrt(d);
      for (int i = tid - 256; i < k; i += (int)blockDim.x - 256) C[i * k + j] = (i < j) ? 0.0 : G[i * k + j] * rs;
    }
    // (2-D thread mapping, no integer division: every (i, l), j < l <= i, is updated exactly once)
    for (int i = j + 1 + (tid >> 5); i < k; i += (int)(blockDim.x >> 5)) {
      const double gij = G[i * k + j] * rinv;
      for (int l = j + 1 + (tid & 31); l <= i; l += 32) G[i * k + l] -= gij * G[l * k + j];
    }
    __syncthreads();
  }
  if (tid == 0) *logdet_out = ld + *logdet_tail;
}

// Cinv = C^{-1} (lower triangular, fp64): one WARP (= one CTA) per column j, forward substitution with the column held in
// registers (entry b on lane b & 31) and the inner product of step i split over the lanes + a shuffle tree: ~100 dependent
// steps of ~150 cycles instead of 5000 dependent FMAs of one thread per column.  k <= 128.
__global__ void __launch_bounds__(32) cinv_kernel(const double* __restrict__ C, int k, double* __restrict__ Cinv) {
  const int j = blockIdx.x, lane = threadIdx.x;
  double x[4] = {0.0, 0.0, 0.0, 0.0};   // x[t] = Cinv[lane + 32 t][j]
  for (int i = 0; i < k; ++i) {
    double xi = 0.0;
    if (i >= j) {
      const double* ci = C + (size_t)i * k;
      double s = 0.0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int b = lane + 32 * t;
        if (b >= j && b < i) s = fma(ci[b], x[t], s);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      xi = (((i == j) ? 1.0 : 0.0) - s) / ci[i];
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (lane + 32 * t == i) x[t] = xi;
    }
    if (lane == 0) Cinv[(size_t)i * k + j] = xi;
  }
}

constexpr int WS_BLOCKS = 4;
// W[r][a] = sum_{b<=a} Cinv[a][b] L[b][r]   (W = L C^{-T}); 32 rows x 4 interleaved a-groups per pass, fp64 accumulate
__global__ void __launch_bounds__(128)
wsolve_kernel(const float* __restrict__ Lt, int k, int64_t n_total, int64_t row_begin, int64_t n_local,
              const double* __restrict__ Cinv, const float* __restrict__ dvec, float* __restrict__ W) {
  extern __shared__ double shw[];
  double* Ci = shw;                        // [k][k]
  double* Ls = shw + (size_t)k * k;        // [k][32], fp64 copy of the L rows (exact conversion, once per element)
  for (int e = threadIdx.x; e < k * k; e += 128) Ci[e] = Cinv[e];
  const int rl = threadIdx.x & 31, ag = threadIdx.x >> 5;
  for (int blk = 0; blk < WS_BLOCKS; ++blk) {          // C^{-1} (80 KB at k = 100) is loaded once per WS_BLOCKS * 32 rows
    const int64_t r0 = ((int64_t)blockIdx.x * WS_BLOCKS + blk) * 32;
    if (r0 >= n_local) break;
    __syncthreads();
    for (int e = threadIdx.x; e < k * 32; e += 128) {
      int b = e >> 5, rr = e & 31;
      Ls[e] = (r0 + rr < n_local) ? (double)Lt[(int64_t)b * n_total + row_begin + r0 + rr] : 0.0;
    }
    __syncthreads();
    const int64_t r = r0 + rl;
    for (int a = ag; a < k; a += 4) {
      double s = 0.0;
      for (int b = 0; b <= a; ++b) s = fma(Ci[a * k + b], Ls[b * 32 + rl], s);
      if (r < n_local) W[r * k + a] = (float)(dvec ? s / (double)dvec[row_begin + r] : s);   // per-row noise: W = D^-1 L C^-T
    }
  }
}

// sum_j log d_j (fp64, one CTA; the per-row-noise tail of log det P)
__global__ void logsum_kernel(const float* __restrict__ d, int64_t n, double* __restrict__ out) {
  __shared__ double sh[256];
  double s = 0.0;
  for (int64_t j = threadIdx.x; j < n; j += 256) s += log((double)d[j]);
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st) sh[threadIdx.x] += sh[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}

// ---- split-preconditioner factor of the CIQ sampler (gp_ciq_precond_build, minres.cu header) ----
// U[r][j] = s_r sum_b T[j][b] L[b][r]  (T = diag(h) V^T, s_r = d_r^{-1/2}); the row / j-group mapping of wsolve_kernel, all b
__global__ void __launch_bounds__(128)
usolve_kernel(const float* __restrict__ Lt, int k, int64_t n, const double* __restrict__ T, const float* __restrict__ dvec,
              double sigma_inv, float* __restrict__ U) {
  extern __shared__ double shw[];
  double* Ts = shw;                        // [k][k]
  double* Ls = shw + (size_t)k * k;        // [k][32]
  for (int e = threadIdx.x; e < k * k; e += 128) Ts[e] = T[e];
  const int rl = threadIdx.x & 31, ag = threadIdx.x >> 5;
  for (int blk = 0; blk < WS_BLOCKS; ++blk) {
    const int64_t r0 = ((int64_t)blockIdx.x * WS_BLOCKS + blk) * 32;
    if (r0 >= n) break;
    __syncthreads();
    for (int e = threadIdx.x; e < k * 32; e += 128) {
      int b = e >> 5, rr = e & 31;
      Ls[e] = (r0 + rr < n) ? (double)Lt[(int64_t)b * n + r0 + rr] : 0.0;
    }
    __syncthreads();
    const int64_t r = r0 + rl;
    if (r >= n) continue;
    const double sr = dvec ? 1.0 / sqrt((double)dvec[r]) : sigma_inv;
    for (int a = ag; a < k; a += 4) {
      double s = 0.0;
      for (int b = 0; b < k; ++b) s = fma(Ts[a * k + b], Ls[b * 32 + rl], s);
      U[r * k + a] = (float)(s * sr);
    }
  }
}

// per-CTA fp64 partials [sum Lt^2 | min d] (min d = -1 once a d is <= 0 or NaN), reduced on the host in CTA order
__global__ void __launch_bounds__(256)
ciq_stats_kernel(const float* __restrict__ Lt, int64_t total, const float* __restrict__ dvec, int64_t n, double* __restrict__ part) {
  __shared__ double s_sum[256], s_min[256];
  const int tid = threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * 256;
  double s = 0.0, m = INFINITY;
  for (int64_t e = (int64_t)blockIdx.x * 256 + tid; e < total; e += stride) {
    const double v = Lt[e];
    s = fma(v, v, s);
  }
  if (dvec)
    for (int64_t j = (int64_t)blockIdx.x * 256 + tid; j < n; j += stride) {
      const float v = dvec[j];
      m = (v > 0.f) ? fmin(m, (double)v) : -1.0;
    }
  s_sum[tid] = s; s_min[tid] = m;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (tid < h) { s_sum[tid] += s_sum[tid + h]; s_min[tid] = fmin(s_min[tid], s_min[tid + h]); }
    __syncthreads();
  }
  if (tid == 0) { part[2 * blockIdx.x] = s_sum[0]; part[2 * blockIdx.x + 1] = s_min[0]; }
}

// Cyclic Jacobi eigen-decomposition of the symmetric k x k matrix A (fp64, fixed rotation order: deterministic).  On return the
// diagonal of A holds the eigenvalues and the columns of V the eigenvectors.
static void jacobi_eigh(int k, double* A, double* V) {
  double fro = 0.0;
  for (int e = 0; e < k * k; ++e) { V[e] = (e / k == e % k) ? 1.0 : 0.0; fro += A[e] * A[e]; }
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < k; ++p)
      for (int q = p + 1; q < k; ++q) off += A[p * k + q] * A[p * k + q];
    if (off <= 1e-32 * fro) break;
    for (int p = 0; p < k - 1; ++p)
      for (int q = p + 1; q < k; ++q) {
        const double apq = A[p * k + q];
        if (apq == 0.0) continue;
        const double theta = (A[q * k + q] - A[p * k + p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int r = 0; r < k; ++r) {   // A J
          const double arp = A[r * k + p], arq = A[r * k + q];
          A[r * k + p] = c * arp - s * arq; A[r * k + q] = s * arp + c * arq;
        }
        for (int r = 0; r < k; ++r) {   // J^T (A J)
          const double apr = A[p * k + r], aqr = A[q * k + r];
          A[p * k + r] = c * apr - s * aqr; A[q * k + r] = s * apr + c * aqr;
        }
        for (int r = 0; r < k; ++r) {   // V J
          const double vrp = V[r * k + p], vrq = V[r * k + q];
          V[r * k + p] = c * vrp - s * vrq; V[r * k + q] = s * vrp + c * vrq;
        }
      }
  }
}

// Z[r][c] = sum_a L[a][r] eps1[a][c] + sigma eps2[r][c]
__global__ void probes_kernel(const float* __restrict__ Lt, int k, int64_t n_total, int64_t row_begin, int64_t n_local,
                              const float* __restrict__ eps1, const float* __restrict__ eps2, int tp, float sigma,
                              const float* __restrict__ dvec, float* __restrict__ Z) {
  extern __shared__ float e1[];  // [k][tp]
  for (int e = threadIdx.x; e < k * tp; e += blockDim.x) e1[e] = eps1[e];
  __syncthreads();
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_local * tp) return;
  int64_t r = idx / tp;
  int c = (int)(idx % tp);
  float s = (dvec ? sqrtf(dvec[row_begin + r]) : sigma) * eps2[r * tp + c];   // z = L eps1 + D^1/2 eps2
  for (int a = 0; a < k; ++a) s = fmaf(Lt[(int64_t)a * n_total + row_begin + r], e1[a * tp + c], s);
  Z[r * tp + c] = s;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_pivoted_cholesky(gp_plan* p, int rank, float error_tol, float* Lt, int64_t* piv, int* rank_out) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_CHECK(refuse_settings(p, CALL_PIVOTED_CHOLESKY));
  GP_REQUIRE(p->same, GP_E_SHAPE, "pivoted Cholesky needs a square operator");
  GP_CHECK(slot_scales_prepare(p));
  const bool prod = p->backend == GP_BACKEND_PRODUCT;
  if (prod) GP_CHECK(product_refresh(p));   // S = prod_f s_f into p->outputscale
  const int64_t n = p->n2;
  GP_REQUIRE(n < (int64_t)1 << 31, GP_E_SHAPE, "n too large");
  rank = (int)std::min<int64_t>(rank, n);
  GP_REQUIRE(rank >= 1, GP_E_SHAPE, "rank must be >= 1");
  cudaStream_t st = p->stream;
  const unsigned gb = (unsigned)cdiv(n, PC_THREADS);
  GP_CHECK(p->pcdiag.ensure(sizeof(float) * n));
  GP_CHECK(p->pcperm.ensure(sizeof(int) * n));
  GP_CHECK(p->pcpos.ensure(sizeof(int) * n));
  GP_CHECK(p->pcstate.ensure(sizeof(PcState) + 256 + (sizeof(float) + sizeof(int) + sizeof(double)) * gb + 64));
  float* diag = p->pcdiag.as<float>();
  int* perm = p->pcperm.as<int>();
  int* pos = p->pcpos.as<int>();
  PcState* S = p->pcstate.as<PcState>();
  double* psum = reinterpret_cast<double*>(reinterpret_cast<char*>(S) + 256);
  float* pval = reinterpret_cast<float*>(psum + gb);
  int* ppos = reinterpret_cast<int*>(pval + gb);
  GP_CUDA(cudaMemsetAsync(Lt, 0, sizeof(float) * (size_t)rank * n, st));
  GP_CUDA(cudaMemsetAsync(piv, 0, sizeof(int64_t) * rank, st));
  const bool sum = p->backend == GP_BACKEND_SUM;
  const bool ski = p->backend == GP_BACKEND_SKI;
  const bool add = p->add_M > 0;
  const bool spec = p->sm_Q > 0;
  PcTerms tt;
  memset(&tt, 0, sizeof(tt));
  SkiRows sk;
  memset(&sk, 0, sizeof(sk));
  float os_total = p->outputscale;
  int dp_total = p->DP;
  if (sum) {
    os_total = 0.f;
    dp_total = 0;
    tt.n = (int)p->terms.size();
    for (int t = 0; t < tt.n; ++t) {
      const gp_plan* q = p->terms[t];
      tt.kind[t] = q->kind; tt.DP[t] = q->DP; tt.os[t] = q->outputscale; tt.Z[t] = q->Z2.as<float>(); tt.cp[t] = cov_param(q);
      os_total += q->outputscale;
      dp_total += q->DP;
    }
  } else {
    tt.cp[0] = cov_param(p);
  }
  // a dot-product kernel's diagonal is not constant: a plain polynomial plan is staged as a one-term sum for the initial diagonal
  const bool dot = p->kind == GP_POLY || (sum && sum_has_poly(p));
  if (dot && !sum) {
    tt.n = 1; tt.kind[0] = GP_POLY; tt.DP[0] = p->DP; tt.os[0] = p->outputscale; tt.Z[0] = p->Z2.as<float>();
  }
  tt.rank_stop = dot ? 1 : 0;
  if (prod) {   // os_total = S, dp_total = the factors' widths back to back (product_pack)
    tt.n = (int)p->factors.size();
    for (int t = 0; t < tt.n; ++t) {
      const gp_plan* q = p->factors[t];
      tt.kind[t] = q->kind; tt.DP[t] = q->DP; tt.Z[t] = q->Z2.as<float>();
    }
  }
  const bool kron = p->kron != nullptr;
  const bool tasks = p->tasks != nullptr || kron;
  const bool kron_obs = kron && p->kron->masked;
  const bool kron_terms = kron && p->kron->nterm > 1;
  const bool deriv = p->deriv != nullptr;
  const float* Zsrc = p->Z2.as<float>();
  if (deriv) {   // entries of the value / gradient operator from the data plan's packed rows
    GP_CHECK(deriv_refresh(p));
    const gp_plan* q = p->deriv->data;
    tt.rep = q->d + 1; tt.dh = p->deriv->hypd.as<DerivHyp>();
    Zsrc = q->Z2.as<float>();
    dp_total = q->DP;
    os_total = q->outputscale;
  } else if (kron) {   // entries of (s K_data) (x) B from the data plan's packed rows
    GP_REQUIRE(p->kron->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
    GP_CHECK(kron_refresh(p));
    const gp_plan* q = p->kron->data;
    tt.kind[0] = q->kind; tt.task = nullptr; tt.B = p->kron->Bd.as<float>(); tt.T = p->kron->T; tt.rep = p->kron->T;
    if (p->kron->masked) tt.task = p->kron->rowmap.as<int>();   // PC_KIND_KRON_OBS
    Zsrc = q->Z2.as<float>();
    dp_total = q->DP;
    os_total = q->outputscale;
    if (kron_terms) {   // PC_KIND_KRON_TERMS: every term's packed rows, widths back to back
      tt.n = p->kron->nterm;
      dp_total = 0;
      for (int t = 0; t < tt.n; ++t) {
        const gp_plan* qt = p->kron->term[t];
        tt.kind[t] = qt->kind; tt.DP[t] = qt->DP; tt.os[t] = qt->outputscale; tt.Z[t] = qt->Z2.as<float>();
        dp_total += qt->DP;
      }
    }
  } else if (tasks) {
    GP_REQUIRE(p->tasks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
    tt.kind[0] = p->kind; tt.task = p->tasks->d_t1; tt.B = p->tasks->Bd.as<float>(); tt.T = p->tasks->T; tt.rep = 1;
  } else if (add) {   // the constant initial diagonal sum_m e_m(s), entries from the packed rows
    tt.ah = additive_hyp(p);
    os_total = (float)p->add_diag;
  } else if (spec) {   // the constant initial diagonal S (sum_q w_q)^d, entries from the packed rows
    tt.sh = spectral_hyp(p);
    os_total = (float)p->sm_diag;
  }
  if (deriv) {
    const float c = (float)deriv_with_kind(p->deriv->kind, [](auto K) { return decltype(K)::DIAG; });
    pc_init_deriv_kernel<<<gb, PC_THREADS, 0, st>>>(tt, os_total, c, diag, perm, pos, n);
    pc_first_pivot_kernel<<<1, PC_FIRST_THREADS, 0, st>>>(diag, perm, pos, n, S, piv);
    p->launches += 2;
  } else if (kron_terms) {
    pc_init_kron_terms_kernel<<<gb, PC_THREADS, 0, st>>>(tt, diag, perm, pos, n);
    pc_first_pivot_kernel<<<1, PC_FIRST_THREADS, 0, st>>>(diag, perm, pos, n, S, piv);
    p->launches += 2;
  } else if (kron_obs) {
    pc_init_kron_obs_kernel<<<gb, PC_THREADS, 0, st>>>(tt, os_total, diag, perm, pos, n);
    pc_first_pivot_kernel<<<1, PC_FIRST_THREADS, 0, st>>>(diag, perm, pos, n, S, piv);
    p->launches += 2;
  } else if (tasks) {
    pc_init_task_kernel<<<gb, PC_THREADS, 0, st>>>(tt, os_total, diag, perm, pos, n);
    pc_first_pivot_kernel<<<1, PC_FIRST_THREADS, 0, st>>>(diag, perm, pos, n, S, piv);
    p->launches += 2;
  } else if (ski) {
    GP_CHECK(ski_rows_args(p, &sk));
    dp_total = sk.staged ? sk.usum : 0;   // the pivot's u_k take the place of its packed inputs in shared memory (staged grids)
    pc_init_ski_kernel<<<gb, PC_THREADS, 0, st>>>(sk, diag, perm, pos, n);
    pc_first_pivot_kernel<<<1, PC_FIRST_THREADS, 0, st>>>(diag, perm, pos, n, S, piv);
    p->launches += 2;
  } else if (dot) {
    pc_init_dot_kernel<<<gb, PC_THREADS, 0, st>>>(tt, diag, perm, pos, n);
    pc_first_pivot_kernel<<<1, PC_FIRST_THREADS, 0, st>>>(diag, perm, pos, n, S, piv);
    p->launches += 2;
  } else {
    pc_init_kernel<<<gb, PC_THREADS, 0, st>>>(diag, perm, pos, n, os_total, S, piv);   // stationary terms: constant initial diagonal
    p->launches += 1;
  }
  const float* Z = (sum || ski || prod) ? nullptr : Zsrc;
  const bool stepwise = getenv("GP_PC_STEPWISE") != nullptr;   // debugging / A-B switch: one launch per step
  int coop = 0;
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, p->device);
  GP_REQUIRE(!sum || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of a kernel sum needs the cooperative kernel");
  GP_REQUIRE(!prod || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of a kernel product needs the cooperative kernel");
  GP_REQUIRE(!ski || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of a SKI operator needs the cooperative kernel");
  GP_REQUIRE(!tasks || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of a multitask operator needs the cooperative kernel");
  GP_REQUIRE(!deriv || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of a derivative operator needs the cooperative kernel");
  GP_REQUIRE(!add || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of an additive operator needs the cooperative kernel");
  GP_REQUIRE(!spec || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of a spectral mixture operator needs the cooperative kernel");
  GP_REQUIRE(!dot || (coop && !stepwise), GP_E_STATE, "pivoted Cholesky of a polynomial operator needs the cooperative kernel");
  if (coop && !stepwise) {
    const size_t sh = sizeof(float) * (dp_total + rank + (size_t)rank * PCP_THREADS);
    const void* fn1;
    switch (sum ? PC_KIND_SUM : prod ? PC_KIND_PRODUCT : ski ? PC_KIND_SKI : deriv ? (p->deriv->kind == GP_MATERN52 ? PC_KIND_M52GRAD : PC_KIND_DERIV) : kron_terms ? PC_KIND_KRON_TERMS : kron_obs ? PC_KIND_KRON_OBS : tasks ? PC_KIND_TASK : add ? PC_KIND_ADDITIVE : spec ? PC_KIND_SPECTRAL : p->kind) {
      case PC_KIND_ADDITIVE: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_ADDITIVE>; break;
      case PC_KIND_SPECTRAL: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_SPECTRAL>; break;
      case PC_KIND_TASK: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_TASK>; break;
      case PC_KIND_KRON_OBS: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_KRON_OBS>; break;
      case PC_KIND_KRON_TERMS: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_KRON_TERMS>; break;
      case PC_KIND_DERIV: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_DERIV>; break;
      case PC_KIND_M52GRAD: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_M52GRAD>; break;
      case GP_RBF: fn1 = (const void*)pc_persistent1_kernel<GP_RBF>; break;
      case GP_MATERN12: fn1 = (const void*)pc_persistent1_kernel<GP_MATERN12>; break;
      case GP_MATERN32: fn1 = (const void*)pc_persistent1_kernel<GP_MATERN32>; break;
      case GP_RQ: fn1 = (const void*)pc_persistent1_kernel<RQ_K>; break;
      case GP_POLY: fn1 = (const void*)pc_persistent1_kernel<POLY_K>; break;
      case GP_PPOLY: fn1 = (const void*)pc_persistent1_kernel<PP_K>; break;
      case PC_KIND_SUM: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_SUM>; break;
      case PC_KIND_PRODUCT: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_PRODUCT>; break;
      case PC_KIND_SKI: fn1 = (const void*)pc_persistent1_kernel<PC_KIND_SKI>; break;
      default: fn1 = (const void*)pc_persistent1_kernel<GP_MATERN52>; break;
    }
    GP_CUDA(cudaFuncSetAttribute(fn1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
    int per_sm1 = 0;
    GP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm1, fn1, PCP_THREADS, sh));
    GP_REQUIRE(per_sm1 >= 1, GP_E_CUDA, "pivoted Cholesky kernel does not fit on an SM");
    const unsigned grid1 = (unsigned)std::min<int64_t>(cdiv(n, PCP_THREADS), (int64_t)per_sm1 * p->n_sm);
    GP_CHECK(p->pcpart.ensure(sizeof(PcPart) * 2 * (size_t)grid1));
    PcPart* part = p->pcpart.as<PcPart>();
    int DPv = dp_total, rk = rank;
    float osv = os_total, tolv = error_tol;
    int64_t nn = n;
    void* args[] = {(void*)&Z, &DPv, &osv, &Lt, &nn, &rk, &tolv, &diag, &pos, &S, &piv, &part, &tt, &sk};
    GP_CUDA(cudaLaunchCooperativeKernel(fn1, dim3(grid1), dim3(PCP_THREADS), args, sh, st));
    p->launches += 1;
  } else {
  for (int m = 0; m < rank; ++m) {
    size_t sh = sizeof(float) * (p->DP + m);
#define GP_PC_LAUNCH(KK) pc_step_kernel<KK><<<gb, PC_THREADS, sh, st>>>(Z, p->DP, p->outputscale, Lt, n, m, rank, error_tol, diag, perm, pos, S, piv, pval, ppos, psum, cov_param(p))
    switch (p->kind) {
      case GP_RQ: GP_PC_LAUNCH(RQ_K); break;
      case GP_PPOLY: GP_PC_LAUNCH(PP_K); break;
      case GP_RBF: GP_PC_LAUNCH(GP_RBF); break;
      case GP_MATERN12: GP_PC_LAUNCH(GP_MATERN12); break;
      case GP_MATERN32: GP_PC_LAUNCH(GP_MATERN32); break;
      default: GP_PC_LAUNCH(GP_MATERN52); break;
    }
#undef GP_PC_LAUNCH
    p->launches += 1;
  }
  }
  GP_CUDA(cudaGetLastError());
  PcState* hs = reinterpret_cast<PcState*>(static_cast<char*>(p->pinned) + PIN_PC_STATE);
  GP_CUDA(cudaMemcpyAsync(hs, S, sizeof(PcState), cudaMemcpyDeviceToHost, st));
  GP_CUDA(cudaStreamSynchronize(st));
  if (rank_out) *rank_out = hs->rank;
  if (hs->nan_flag) {
    set_error("NaNs encountered in preconditioner computation. Attempting to continue without preconditioning.");
    return GP_W_PIVCHOL_NAN;
  }
  return GP_OK;
}

// launch split of gram_kernel: ntile x ntile output tiles times nz slices of jslice rows, about 2 CTAs per SM
struct GramSplit {
  int ntile, nz;
  int64_t jslice;
};
static GramSplit gram_split(const gp_plan* p, int k, int64_t n) {
  GramSplit g;
  g.ntile = (int)cdiv(k, GT);
  g.nz = (int)std::min<int64_t>(64, std::max<int64_t>(1, std::min<int64_t>(n / 1024, (2 * p->n_sm) / (g.ntile * (g.ntile + 1) / 2))));
  g.jslice = cdiv(cdiv(n, g.nz), 64) * 64;
  return g;
}

extern "C" int gp_precond_build(gp_plan* p, const float* Lt, int k, float* W, double* logdet_out) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_CHECK(refuse_settings(p, CALL_PRECOND_BUILD));
  GP_REQUIRE(k >= 1 && k <= 128, GP_E_SHAPE, "preconditioner rank %d not in [1,128]", k);
  const float* dvec = p->noise_diag;
  GP_REQUIRE(dvec != nullptr || p->noise > 0.f, GP_E_SHAPE, "preconditioner needs noise > 0");
  cudaStream_t st = p->stream;
  const int64_t n = p->n2;
  const GramSplit g = gram_split(p, k, n);
  GP_CHECK(p->gram.ensure(sizeof(double) * (size_t)g.nz * k * k));
  GP_CHECK(p->cholC.ensure(sizeof(double) * ((size_t)2 * k * k + 4) + 64));
  double* C = p->cholC.as<double>();
  double* Cinv = C + (size_t)k * k;
  double* d_logdet = Cinv + (size_t)k * k;
  double* d_tail = d_logdet + 1;
  int* d_fail = reinterpret_cast<int*>(d_tail + 1);
  GP_CUDA(cudaMemsetAsync(d_fail, 0, sizeof(int), st));
  gram_kernel<<<dim3((unsigned)g.ntile, (unsigned)g.ntile, (unsigned)g.nz), 256, 0, st>>>(Lt, k, n, g.jslice, dvec, p->gram.as<double>());
  if (dvec) {
    logsum_kernel<<<1, 256, 0, st>>>(dvec, n, d_tail);
    p->launches++;
  } else {
    const double tail = (double)(n - k) * log((double)p->noise);
    GP_CUDA(cudaMemcpyAsync(d_tail, &tail, sizeof(double), cudaMemcpyHostToDevice, st));   // pageable source: copied before return
  }
  const size_t shc = sizeof(double) * (size_t)k * k;
  GP_CHECK(opt_in_smem<chol_small_kernel>(p->device, 160 * 1024));   // k <= 128: 128 KB
  GP_CHECK(opt_in_smem<wsolve_kernel>(p->device, 168 * 1024));       // 128 KB + 32 KB
  chol_small_kernel<<<1, 512, shc, st>>>(p->gram.as<double>(), g.nz, k, dvec ? 1.0 : (double)p->noise, d_tail, C, d_logdet, d_fail);
  // W = L C^-T through the explicit inverse (a per-row forward substitution against C in shared memory was tried: 0.52 ms at C2
  // against 0.16 + 0.19 ms for these two kernels -- one 128-thread CTA per SM is latency bound on 5000 dependent steps per row)
  cinv_kernel<<<k, 32, 0, st>>>(C, k, Cinv);
  wsolve_kernel<<<(unsigned)cdiv(p->row_count, 32 * WS_BLOCKS), 128, shc + sizeof(double) * (size_t)k * 32, st>>>(Lt, k, n, p->row_begin,
                                                                                                      p->row_count, Cinv, dvec, W);
  p->launches += 4;
  GP_CUDA(cudaGetLastError());
  double* h = reinterpret_cast<double*>(static_cast<char*>(p->pinned) + PIN_PRECOND);
  GP_CUDA(cudaMemcpyAsync(h, d_logdet, sizeof(double) * 2 + sizeof(int), cudaMemcpyDeviceToHost, st));
  GP_CUDA(cudaStreamSynchronize(st));
  if (logdet_out) *logdet_out = h[0];
  int fail = *reinterpret_cast<int*>(h + 2);
  GP_REQUIRE(!fail, GP_W_PIVCHOL_NAN, "preconditioner Gram matrix is not positive definite");
  return GP_OK;
}

// sum of the per-row diagonal (gp_kdiag's) of a polynomial plan or of a sum with a polynomial term, in fp64 in row order
static int dot_diag_sum(gp_plan* p, double* out) {
  const int64_t n = p->n2;
  GP_CHECK(p->misc.ensure(sizeof(float) * n));
  if (p->backend == GP_BACKEND_SUM) GP_CHECK(sum_kdiag_terms(p, p->misc.as<float>()));
  else GP_CHECK(gp_kdiag(p, p->misc.as<float>()));
  std::vector<float> h(n);
  GP_CUDA(cudaMemcpyAsync(h.data(), p->misc.p, sizeof(float) * n, cudaMemcpyDeviceToHost, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));
  double s = 0.0;
  for (int64_t i = 0; i < n; ++i) s += (double)h[i];
  *out = s;
  return GP_OK;
}

extern "C" int gp_ciq_precond_build(gp_plan* p, const float* Lt, int k, float* U, double* trace_resid_out) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_CHECK(refuse_settings(p, CALL_CIQ_PRECOND_BUILD));
  GP_REQUIRE(k >= 1 && k <= 128, GP_E_SHAPE, "preconditioner rank %d not in [1,128]", k);
  GP_REQUIRE(Lt != nullptr && U != nullptr, GP_E_SHAPE, "Lt / U missing");
  GP_REQUIRE(p->same, GP_E_SHAPE, "the CIQ preconditioner needs a square operator");
  GP_REQUIRE(!(p->comm && p->comm->world > 1) && p->row_begin == 0 && p->row_count == p->n2, GP_E_SHAPE,
             "gp_ciq_precond_build is not supported on row-sharded plans");
  const float* dvec = p->noise_diag;
  GP_REQUIRE(dvec != nullptr || p->noise > 0.f, GP_E_SHAPE, "the CIQ preconditioner needs noise > 0");
  cudaStream_t st = p->stream;
  const int64_t n = p->n2;
  // Gram G = L^T D^-1 L (per-row noise) or L^T L (scalar noise, divided by sigma^2 below)
  const GramSplit g = gram_split(p, k, n);
  const int nz = g.nz;
  const int gs = (int)std::max<int64_t>(1, std::min<int64_t>(cdiv((int64_t)k * n, 4096), (int64_t)2 * p->n_sm));
  GP_CHECK(p->gram.ensure(sizeof(double) * ((size_t)nz * k * k + 2 * (size_t)gs)));
  GP_CHECK(p->cholC.ensure(sizeof(double) * ((size_t)2 * k * k + 4) + 64));
  double* gpart = p->gram.as<double>();
  double* spart = gpart + (size_t)nz * k * k;
  double* d_T = p->cholC.as<double>();
  gram_kernel<<<dim3((unsigned)g.ntile, (unsigned)g.ntile, (unsigned)nz), 256, 0, st>>>(Lt, k, n, g.jslice, dvec, gpart);
  ciq_stats_kernel<<<gs, 256, 0, st>>>(Lt, (int64_t)k * n, dvec, n, spart);
  p->launches += 2;
  GP_CUDA(cudaGetLastError());
  std::vector<double> hpart((size_t)nz * k * k + 2 * (size_t)gs);
  GP_CUDA(cudaMemcpyAsync(hpart.data(), gpart, sizeof(double) * hpart.size(), cudaMemcpyDeviceToHost, st));
  GP_CUDA(cudaStreamSynchronize(st));
  const double* hs = hpart.data() + (size_t)nz * k * k;
  double lsq = 0.0, dmin = INFINITY;
  for (int b = 0; b < gs; ++b) { lsq += hs[2 * b]; dmin = std::min(dmin, hs[2 * b + 1]); }
  GP_REQUIRE(!dvec || dmin > 0.0, GP_E_SHAPE, "the CIQ preconditioner needs a per-row noise diagonal > 0");
  const double sig2 = dvec ? 1.0 : (double)p->noise;
  std::vector<double> A((size_t)k * k), V((size_t)k * k), T((size_t)k * k);
  bool finite = std::isfinite(lsq);
  for (int e = 0; e < k * k; ++e) {
    double s = 0.0;
    for (int z = 0; z < nz; ++z) s += hpart[(size_t)z * k * k + e];
    A[e] = s / sig2;
    finite = finite && std::isfinite(A[e]);
  }
  if (!finite) {
    set_error("NaNs encountered in the CIQ preconditioner factor. Attempting to continue without preconditioning.");
    return GP_W_PIVCHOL_NAN;
  }
  // (V, s) = eigh(M^T M), M = D^-1/2 L ; T = diag(h) V^T with h_j = (sqrt(1 + s_j) (1 + sqrt(1 + s_j)))^-1/2 (no 1/s, no subtraction)
  jacobi_eigh(k, A.data(), V.data());
  for (int j = 0; j < k; ++j) {
    const double r1 = sqrt(1.0 + std::max(A[(size_t)j * k + j], 0.0));
    const double h = 1.0 / sqrt(r1 * (1.0 + r1));
    for (int b = 0; b < k; ++b) T[(size_t)j * k + b] = h * V[(size_t)b * k + j];
  }
  GP_CUDA(cudaMemcpyAsync(d_T, T.data(), sizeof(double) * k * k, cudaMemcpyHostToDevice, st));   // pageable: copied before return
  const size_t shu = sizeof(double) * ((size_t)k * k + (size_t)k * 32);
  GP_CHECK(opt_in_smem<usolve_kernel>(p->device, 168 * 1024));   // 128 KB + 32 KB
  usolve_kernel<<<(unsigned)cdiv(n, 32 * WS_BLOCKS), 128, shu, st>>>(Lt, k, n, d_T, dvec, 1.0 / sqrt((double)p->noise), U);
  p->launches += 1;
  GP_CUDA(cudaGetLastError());
  // tr(K - L L^T): the diagonal of a stationary kernel (sum) is its (summed) outputscale, as gp_kdiag fills it; the SKI diagonal
  // w_i^T K_uu w_i varies from row to row and is summed in fp64
  if (p->backend == GP_BACKEND_PRODUCT) GP_CHECK(product_refresh(p));   // the constant diagonal S = prod_f s_f
  double tr_k = (double)n * p->outputscale;
  if (p->kind == GP_POLY || (p->backend == GP_BACKEND_SUM && sum_has_poly(p))) {
    GP_CHECK(dot_diag_sum(p, &tr_k));   // a polynomial diagonal S (|x_i|^2 + c)^p varies from row to row
  } else if (p->backend == GP_BACKEND_SUM) {
    double os_total = 0.0;
    for (const gp_plan* q : p->terms) os_total += q->outputscale;
    tr_k = (double)n * os_total;
  } else if (p->backend == GP_BACKEND_SKI) {
    GP_CHECK(ski_diag_sum(p, &tr_k));
  } else if (p->deriv) {    // s N (1 + c sum_c 1 / l_c^2), c = 1 RBF, 5/3 Matern-5/2
    GP_CHECK(deriv_refresh(p));
    tr_k = deriv_trace(p);
  } else if (p->kron && p->kron->nterm > 1) {   // N sum_q s_q sum_a B_q[a, a]
    const gp_kron_state* ks = p->kron;
    tr_k = 0.0;
    for (int q = 0; q < ks->nterm; ++q) {
      double bt = 0.0;
      for (int a = 0; a < ks->T; ++a) bt += (double)ks->B[((size_t)q * ks->T + a) * ks->T + a];
      tr_k += (double)ks->term[q]->outputscale * (double)ks->term[q]->n2 * bt;
    }
  } else if (p->kron && p->kron->masked) {   // s sum_r B[a_r, a_r] over the observed rows r, a_r = rowmap[r] mod T
    const gp_kron_state* ks = p->kron;
    double bt = 0.0;
    for (int g : ks->obs_r) bt += (double)ks->B[(size_t)(g % ks->T) * ks->T + g % ks->T];
    tr_k = (double)ks->data->outputscale * bt;
  } else if (p->kron) {     // s N sum_a B[a, a]
    const gp_kron_state* ks = p->kron;
    double bt = 0.0;
    for (int a = 0; a < ks->T; ++a) bt += (double)ks->B[(size_t)a * ks->T + a];
    tr_k = (double)ks->data->outputscale * (double)ks->data->n2 * bt;
  } else if (p->tasks) {   // s sum_i B[t_i, t_i]
    const gp_task_state* ts = p->tasks;
    double bt = 0.0;
    for (int a = 0; a < ts->T; ++a) bt += (double)(ts->off1[a + 1] - ts->off1[a]) * (double)ts->B[(size_t)a * ts->T + a];
    tr_k = (double)p->outputscale * bt;
  } else if (p->add_M) {   // N sum_m e_m(s)
    tr_k = (double)n * p->add_diag;
  } else if (p->sm_Q) {   // N S (sum_q w_q)^d
    tr_k = (double)n * p->sm_diag;
  }
  if (trace_resid_out) *trace_resid_out = tr_k - lsq;
  GP_CUDA(cudaStreamSynchronize(st));
  return GP_OK;
}

extern "C" int gp_precond_probes(gp_plan* p, const float* Lt, int k, const float* eps1, const float* eps2, int tp, float* Z) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_CHECK(refuse_settings(p, CALL_PRECOND_PROBES));
  GP_REQUIRE(k >= 1 && tp >= 1 && (size_t)k * tp * 4 <= 40 * 1024, GP_E_SHAPE, "bad probe shape k=%d tp=%d", k, tp);
  int64_t tot = p->row_count * tp;
  probes_kernel<<<(unsigned)cdiv(tot, 256), 256, sizeof(float) * k * tp, p->stream>>>(Lt, k, p->n2, p->row_begin, p->row_count,
                                                                                  eps1, eps2, tp, sqrtf(p->noise), p->noise_diag, Z);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}
