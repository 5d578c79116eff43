// m52grad.cu -- GPs with derivative observations under a Matern-5/2 covariance: the value / gradient operator of
// Matern52KernelGrad (kernels/matern52_kernel_grad.py) over interleaved rows i (d+1) + a, on a plain Matern-5/2 data plan
// (gp_plan_set_deriv_kind).  Geometry, refresh, the split sum and the host reductions are deriv.cu's; this file holds the entries.
//
// Entries.  With D = x_i - x'_j, u_a = D_a / l_a^2, rho = sqrt(5) r (r^2 = sum_c D_c^2 / l_c^2), e = exp(-rho),
// A = (5/3) (1 + rho) e and B = (25/3) e (times the outputscale s):
//     [0, 0] = (1 + rho + rho^2 / 3) e,   [0, b] = A u_b,   [a, 0] = -A u_a,   [a, b] = A delta_ab / l_a^2 - B u_a u_b.
// The data plan packs z = (x - mean) sqrt(10) / l (pack.cu), so rho = sqrt(|dz|^2 / 2) and u_c = dz_c / (sqrt(10) l_c) = dz_c w[c].
// D = 0 gives s and (5/3) s / l_a^2 on the diagonal exactly.
//
// Products.  With h = sum_b u_b v^b per column:  out0 += [0,0] v0 + A h,  out^a += A v^a / l_a^2 - u_a (A v0 + B h): 3 d + 4 FMAs
// per pair and column, one sqrt and one ex2 per pair.  One thread owns one point's d + 1 rows; 64-point tiles of the other side
// and their V block are staged in shared memory; the reduced side is split over CTAs into partials that deriv_finish_kernel sums
// in a fixed order.  No atomics: repeated calls give identical bits.
//
// Gradients (DESIGN 4.16).  For one pair and column, with P = l0 r0, h = sum u_b r^b, g = sum u_a l^a, q = sum l^a r^a / l_a^2:
//     F = sum_ab l_a E_ab r_b = [0,0] P + A (l0 h - g r0 + q) - B g h           (d/ds = sum F)
// and with q_c = (D_c / l_c)^2 = dz_c^2 / 10:  l_c d[0,0]/dl_c = A q_c,  l_c dA/dl_c = B q_c,  l_c dB/dl_c = 5 B q_c / rho,
// l_c du_a/dl_c = -2 delta_ac u_a,  l_c d(1 / l_a^2)/dl_c = -2 delta_ac / l_a^2, so
//     l_c dF/dl_c = q_c [A P + B (l0 h - g r0 + q) - (5 B / rho) g h] - 2 A [u_c (l0 r^c - l^c r0) + r^c l^c / l_c^2]
//                   + 2 B u_c (l^c h + r^c g).
// q_c / rho <= rho / 5 is bounded but 0 / 0 at coincident points (and where |dz|^2 flushes to zero): 5 B / rho is taken as 0 at
// rho = 0, where every q_c is 0 as well.  m52g_grad_kernel sums per thread in fp32 and every CTA in fp64; the host adds the CTA
// partials in a fixed order.
#include <math.h>

#include <algorithm>

#include "gp_common.cuh"

namespace gp {

constexpr float M52_A = 1.6666666f;    // 5 / 3
constexpr float M52_B = 8.3333333f;    // 25 / 3
constexpr float M52_Q = 0.1f;          // q_c = dz_c^2 / 10

// columns per CTA: the RBF kernels' choice (deriv.cu), the accumulators are the same (DP + 1) x TW
template <int DP>
struct M52TW { static constexpr int value = DP <= 4 ? 16 : 4; };
template <int DP>
struct M52GradTW { static constexpr int value = DP <= 4 ? 8 : (DP <= 8 ? 4 : 2); };

// rho, e = exp(-rho), [0, 0], A and B of one pair from |dz|^2
__device__ __forceinline__ void m52g_pair(float s, float* rho, float* k0, float* A, float* B) {
  const float r = sqrt_approx(0.5f * s);
  const float e = ex2_approx(-LOG2E * r);
  *rho = r;
  *k0 = fmaf(fmaf(r, 0.33333334f, 1.f), r, 1.f) * e;
  *A = M52_A * fmaf(r, e, e);
  *B = M52_B * e;
}

// out rows i (d+1) + a of the split's partial, columns [c0, c0 + TW)
// CTAs per SM as the RBF kernel reaches them: DP = 4 three (168 registers; unbounded, ptxas takes 177 and two fit, 1.6x the RBF
// time at d = 2 on H100), with one pair per loop step to stay free of spills; DP = 8 four (126); wider DP unbounded
template <int DP, int TW>
__global__ void __launch_bounds__(DV_TI, DP <= 4 ? 3 : (DP <= 8 ? 4 : 1))
m52g_kmv_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ V16, float* __restrict__ part,
                int64_t n1, int64_t n2, int d, int64_t cols_per_split, int64_t slot_rows, const __grid_constant__ DerivHyp hy,
                const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  constexpr int R = DP + 1;
  __shared__ __align__(16) float zj[DV_TJ][DP];
  __shared__ __align__(16) float vj[DV_TJ][R][TW];
  const int tid = threadIdx.x;
  const int rw = d + 1;
  const int64_t i = (int64_t)blockIdx.x * DV_TI + tid;
  const int split = blockIdx.y;
  const int c0 = blockIdx.z * TW;
  const int64_t j_begin = (int64_t)split * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const bool rv = i < n1;
  float zi[DP];
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? Z1[i * DP + c] : 0.f;
  float acc[R][TW];
#pragma unroll
  for (int a = 0; a < R; ++a)
#pragma unroll
    for (int t = 0; t < TW; ++t) acc[a][t] = 0.f;

  for (int64_t j0 = j_begin; j0 < j_end; j0 += DV_TJ) {
    const int nj = (int)min((int64_t)DV_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < DV_TJ * DP; e += DV_TI) (&zj[0][0])[e] = (e / DP < nj) ? Z2[j0 * DP + e] : 0.f;
    for (int e = tid; e < DV_TJ * R * TW; e += DV_TI) {
      const int jj = e / (R * TW), b = (e / TW) % R, t = e % TW;
      (&vj[0][0][0])[e] = (jj < nj && b < rw) ? V16[((j0 + jj) * rw + b) * TP + c0 + t] : 0.f;
    }
    __syncthreads();
#pragma unroll (DP <= 4 ? 1 : 2)
    for (int jj = 0; jj < DV_TJ; ++jj) {   // staged padding points carry V = 0: they add 0
      float u[DP], al[DP];
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        const float df = zi[c] - zj[jj][c];
        s = fmaf(df, df, s);
        u[c] = df * hy.w[c];
      }
      float rho, k0, A, B;
      m52g_pair(s, &rho, &k0, &A, &B);
#pragma unroll
      for (int c = 0; c < DP; ++c) al[c] = A * hy.il2[c];
#pragma unroll
      for (int t = 0; t < TW; ++t) {
        const float v0 = vj[jj][0][t];
        float h = 0.f;
#pragma unroll
        for (int c = 0; c < DP; ++c) h = fmaf(u[c], vj[jj][1 + c][t], h);
        acc[0][t] = fmaf(k0, v0, fmaf(A, h, acc[0][t]));
        const float m = fmaf(A, v0, B * h);
#pragma unroll
        for (int c = 0; c < DP; ++c) acc[1 + c][t] = fmaf(al[c], vj[jj][1 + c][t], fmaf(-u[c], m, acc[1 + c][t]));
      }
    }
  }
  if (!rv) return;
  float* dst = part + ((int64_t)split * slot_rows + i * rw) * TP + c0;
#pragma unroll
  for (int a = 0; a < R; ++a) {
    if (a < rw) {
#pragma unroll
      for (int t = 0; t < TW; ++t) dst[(int64_t)a * TP + t] = acc[a][t];
    }
  }
}

// gout[blk][0] = sum F ; gout[blk][1 + c] = sum l_c dF/dl_c / s  (c < d), the expansion of the file header
template <int DP, int TW>
__global__ void __launch_bounds__(DV_TI)
m52g_grad_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ L16, const float* __restrict__ R16,
                 int64_t n1, int64_t n2, int d, int64_t cols_per_split, const __grid_constant__ DerivHyp hy, double* __restrict__ gout) {
  constexpr int R = DP + 1;
  __shared__ __align__(16) float zj[DV_TJ][DP];
  __shared__ __align__(16) float rj[DV_TJ][R][TW];
  __shared__ double red[DV_TI];
  const int tid = threadIdx.x;
  const int rw = d + 1;
  const int64_t i = (int64_t)blockIdx.x * DV_TI + tid;
  const int c0 = blockIdx.z * TW;
  const int64_t j_begin = (int64_t)blockIdx.y * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const bool rv = i < n1;
  float zi[DP], li[R][TW];
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? Z1[i * DP + c] : 0.f;
#pragma unroll
  for (int a = 0; a < R; ++a)
#pragma unroll
    for (int t = 0; t < TW; ++t) li[a][t] = (rv && a < rw) ? L16[(i * rw + a) * TP + c0 + t] : 0.f;
  float gk = 0.f, gc[DP];
#pragma unroll
  for (int c = 0; c < DP; ++c) gc[c] = 0.f;
  for (int64_t j0 = j_begin; j0 < j_end; j0 += DV_TJ) {
    const int nj = (int)min((int64_t)DV_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < DV_TJ * DP; e += DV_TI) (&zj[0][0])[e] = (e / DP < nj) ? Z2[j0 * DP + e] : 0.f;
    for (int e = tid; e < DV_TJ * R * TW; e += DV_TI) {
      const int jj = e / (R * TW), b = (e / TW) % R, t = e % TW;
      (&rj[0][0][0])[e] = (jj < nj && b < rw) ? R16[((j0 + jj) * rw + b) * TP + c0 + t] : 0.f;
    }
    __syncthreads();
    for (int jj = 0; jj < nj; ++jj) {
      float u[DP], dz2[DP];
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        const float df = zi[c] - zj[jj][c];
        dz2[c] = df * df;
        s += dz2[c];
        u[c] = df * hy.w[c];
      }
      float rho, k0, A, B;
      m52g_pair(s, &rho, &k0, &A, &B);
      const float q5 = rho > 0.f ? __fdividef(5.f * B, rho) : 0.f;   // 5 B / rho; every q_c is 0 where rho is
      const float m2A = -2.f * A, p2B = 2.f * B;
      float sp = 0.f, sa = 0.f, sb = 0.f;
#pragma unroll
      for (int t = 0; t < TW; ++t) {
        const float l0 = li[0][t], r0 = rj[jj][0][t];
        float h = 0.f, g = 0.f, q = 0.f;
#pragma unroll
        for (int c = 0; c < DP; ++c) {
          h = fmaf(u[c], rj[jj][1 + c][t], h);
          g = fmaf(u[c], li[1 + c][t], g);
          q = fmaf(hy.il2[c] * li[1 + c][t], rj[jj][1 + c][t], q);
        }
        sp = fmaf(l0, r0, sp);
        sa += fmaf(l0, h, fmaf(-g, r0, q));
        sb = fmaf(g, h, sb);
#pragma unroll
        for (int c = 0; c < DP; ++c) {
          const float lc = li[1 + c][t], rc = rj[jj][1 + c][t];
          const float x = fmaf(u[c], fmaf(l0, rc, -lc * r0), hy.il2[c] * lc * rc);
          const float y = u[c] * fmaf(lc, h, rc * g);
          gc[c] = fmaf(m2A, x, fmaf(p2B, y, gc[c]));
        }
      }
      gk += fmaf(k0, sp, fmaf(A, sa, -B * sb));
      const float T = fmaf(A, sp, fmaf(B, sa, -q5 * sb));
#pragma unroll
      for (int c = 0; c < DP; ++c) gc[c] = fmaf(M52_Q * dz2[c], T, gc[c]);
    }
  }
  const int nout = 1 + d;
  const int64_t blk = ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
#pragma unroll
  for (int o = 0; o <= DP; ++o) {   // unrolled: gc is indexed by constants only (no local memory)
    if (o >= nout) break;
    const float v = o == 0 ? gk : gc[o > 0 ? o - 1 : 0];
    __syncthreads();
    red[tid] = (double)v;
    __syncthreads();
    for (int sft = DV_TI / 2; sft > 0; sft >>= 1) {
      if (tid < sft) red[tid] += red[tid + sft];
      __syncthreads();
    }
    if (tid == 0) gout[blk * nout + o] = red[0];
  }
}

// OUT[r][j (d+1) + b] = s E(i a, j b) for row idx[r] = i (d+1) + a; a NaN row for an index outside [0, n1 (d+1)) or non-finite inputs
__global__ void m52g_krows_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int DP, int d, const int64_t* __restrict__ idx,
                                  int64_t nrows, int64_t n2, float os, const __grid_constant__ DerivHyp hy, float* __restrict__ OUT,
                                  int64_t ldo, const int* __restrict__ xbad) {
  extern __shared__ float zs[];
  const int rw = d + 1;
  const int64_t r = blockIdx.y;
  const int64_t v = idx[r];
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v < 0 || v >= nrows || *xbad) {   // CTA-uniform
    if (j < n2)
      for (int b = 0; b < rw; ++b) OUT[r * ldo + j * rw + b] = __int_as_float(0x7fc00000);
    return;
  }
  const int64_t i = v / rw;
  const int a = (int)(v % rw);
  for (int c = threadIdx.x; c < DP; c += blockDim.x) zs[c] = Z1[i * DP + c];
  __syncthreads();
  if (j >= n2) return;
  const float* zj = Z2 + j * DP;
  float s = 0.f;
  for (int c = 0; c < DP; ++c) {
    const float df = zs[c] - zj[c];
    s = fmaf(df, df, s);
  }
  float rho, k0, A, B;
  m52g_pair(s, &rho, &k0, &A, &B);
  k0 *= os; A *= os; B *= os;
  const float ua = a ? (zs[a - 1] - zj[a - 1]) * hy.w[a - 1] : 0.f;
  float* out = OUT + r * ldo + j * rw;
  out[0] = a ? -A * ua : k0;
  for (int b = 1; b < rw; ++b) {
    const float ub = (zs[b - 1] - zj[b - 1]) * hy.w[b - 1];
    out[b] = a ? fmaf(-B * ua, ub, a == b ? A * hy.il2[a - 1] : 0.f) : A * ub;
  }
}

// OUT[i (d+1) + a] = s E(i a, i a): s and (5/3) s / l_a^2 on a square plan (D = 0), A / l_a^2 - B u_a^2 for a cross plan of equal sizes
__global__ void m52g_kdiag_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int DP, int d, int64_t n, float os,
                                  const __grid_constant__ DerivHyp hy, float* __restrict__ OUT, const int* __restrict__ xbad) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int rw = d + 1;
  if (e >= n * rw) return;
  const int64_t i = e / rw;
  const int a = (int)(e % rw);
  float s = 0.f;
  for (int c = 0; c < DP; ++c) {
    const float df = Z1[i * DP + c] - Z2[i * DP + c];
    s = fmaf(df, df, s);
  }
  float rho, k0, A, B;
  m52g_pair(s, &rho, &k0, &A, &B);
  float o = os * k0;
  if (a) {
    const float ua = (Z1[i * DP + a - 1] - Z2[i * DP + a - 1]) * hy.w[a - 1];
    o = os * fmaf(-B * ua, ua, A * hy.il2[a - 1]);
  }
  OUT[e] = *xbad ? __int_as_float(0x7fc00000) : o;
}

template <int DP>
static int m52g_kmv_launch(gp_plan* p, const float* V16, int ncols, const int* done_flag) {
  constexpr int TW = M52TW<DP>::value;
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  const int nchunk = (int)cdiv(ncols, TW);
  const int64_t rows = p->n1;
  GP_CHECK(ds->part.ensure(sizeof(float) * (size_t)ds->nsplit * rows * TP));
  dim3 grid((unsigned)cdiv(q->n1, DV_TI), (unsigned)ds->nsplit, (unsigned)nchunk);
  m52g_kmv_kernel<DP, TW><<<grid, DV_TI, 0, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), V16, ds->part.as<float>(), q->n1, q->n2, q->d,
                                                         ds->cps, rows, ds->hyp, done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return deriv_finish_launch(p, nchunk * TW, done_flag);
}

int m52g_kmv_partials(gp_plan* p, const float* V16, int ncols, const int* done_flag) {
  return deriv_with_dp(p->DP, [&](auto D) { return m52g_kmv_launch<decltype(D)::value>(p, V16, ncols, done_flag); });
}

int m52g_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  dim3 grid((unsigned)cdiv(q->n2, 256), (unsigned)m);
  m52g_krows_kernel<<<grid, 256, sizeof(float) * q->DP, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), q->DP, q->d, idx, p->n1, q->n2,
                                                                     q->outputscale, ds->hyp, OUT, ldo, q->xbad);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int m52g_kdiag(gp_plan* p, float* OUT) {
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  m52g_kdiag_kernel<<<(unsigned)cdiv(p->n1, 256), 256, 0, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), q->DP, q->d, q->n1, q->outputscale,
                                                                      ds->hyp, OUT, q->xbad);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

template <int DP>
static int m52g_grad_launch(gp_plan* p, const float* L16, const float* R16, int ncols, std::vector<double>& tot) {
  constexpr int TW = M52GradTW<DP>::value;
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  const int nout = 1 + q->d;
  const int nchunk = (int)cdiv(ncols, TW);
  dim3 grid((unsigned)cdiv(q->n1, DV_TI), (unsigned)ds->nsplit, (unsigned)nchunk);
  const size_t nblk = (size_t)grid.x * grid.y * grid.z;
  GP_CHECK(ds->gout.ensure(sizeof(double) * nblk * nout));
  m52g_grad_kernel<DP, TW><<<grid, DV_TI, 0, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), L16, R16, q->n1, q->n2, q->d, ds->cps, ds->hyp,
                                                          ds->gout.as<double>());
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return deriv_sum_gout(p, nblk, nout, tot);
}

int m52g_grad(gp_plan* p, const float* L16, const float* R16, int ncols, std::vector<double>& tot) {
  return deriv_with_dp(p->DP, [&](auto D) { return m52g_grad_launch<decltype(D)::value>(p, L16, R16, ncols, tot); });
}

}  // namespace gp
