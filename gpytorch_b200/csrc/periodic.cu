// periodic.cu -- periodic kernels (MacKay 1998, eq. 47; the reference's kernels/periodic_kernel.py, lengthscale not squared):
//
//   K(x, x') = S exp(-2 sum_d sin^2(pi tau_d / p_d) / l_d),   tau = x - x'
//
// is the RBF kernel of unit lengthscale over an embedding of the inputs, exactly: with e_d(x) = (cos, sin)(2 pi x_d / p_d),
// |e_d(x) - e_d(x')|^2 = 2 - 2 cos(2 pi tau_d / p_d) = 4 sin^2(pi tau_d / p_d), so u_d(x) = e_d(x) / sqrt(l_d) gives
// K = S exp(-|u(x) - u(x')|^2 / 2).  The plan therefore packs u into the plain layout of an RBF plan of width 2d (packed_dims)
// and every plain kernel runs on it unchanged: the tensor-core and CUDA-core K.V, rows, the diagonal, the pivoted Cholesky,
// the solvers, kernel-sum terms and the low-rank correction.  Only the packing and the hyper-parameter gradient are new.
//
// Packing (periodic_pack).  Per point and dimension the reduced phase r = x/p - floor(x/p + 1/2) in [-1/2, 1/2) is formed in
// fp64 (x and p are fp32, so x/p is correct to 2^-53 relative) and rounded once to fp32; the plan then stores
// sqrt(log2 e / l_d) (cos 2 pi r, sin 2 pi r) in columns 2c, 2c + 1 of dimension c (the RBF packing constant of pack.cu, so the plain kernels'
// ex2 gives exp).  The error of an entry therefore does not grow with |x|: the reference's fp32 argument pi x / p carries an
// absolute error of order 2^-24 |x / p|, 1e-2 rad at x ~ 1e5.  The rows are not mean-centred: |u|^2 = sum_d log2 e / l_d is the
// same for every point.
//
// Gradient (periodic_bilinear_kernel).  One pass over the pairs with g = L_i . R_j and k = 2^{-|du|^2 / 2} from direct
// differences of the packed rows (exact on the diagonal):
//   dk/dl_d = k 2 sin^2(pi tau_d / p_d) / l_d^2 = k |du_d|^2 / (2 l_d log2 e)
//   dk/dp_d = k 2 pi tau_d sin(2 pi tau_d / p_d) / (l_d p_d^2) = k tau_d (us_i uc_j - uc_i us_j) 2 pi / (p_d^2 log2 e)
// sin(2 pi tau / p) = sin(2 pi (r_i - r_j)) comes from the reduced phases and tau_d is the fp32 difference of the raw inputs.
// The chain rule through u would instead sum du_i/dp (which carries x_i) over i, where translation invariance makes the terms
// cancel: its error grows with |x|.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "gp_common.cuh"

namespace gp {

constexpr int PER_DMAX = 16;   // input dimensions: 2d packed columns keep 3 (2d) + 4 <= KP_MAX
constexpr double PER_LOG2E = 1.4426950408889634;

struct PerPack {
  double inv_p[PER_DMAX];   // 1 / p_d in fp64
  float a[PER_DMAX];        // sqrt(log2 e / l_d)
};

// dimensions whose gradients one CTA of the bilinear kernel accumulates: 2 fp64 sums each, with dF/dS at most 17 per thread
__host__ __device__ constexpr int per_gd(int D) { return D < 8 ? D : 8; }

// ---- packing: one thread per point ---------------------------------------------------------------------------------------------
__global__ void periodic_pack_kernel(const float* __restrict__ X, int64_t n, int64_t ld, int d, int DP, const PerPack pk,
                                     float* __restrict__ Z, int* __restrict__ xbad) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  float* row = Z + r * DP;
  bool bad = false;
  for (int c = 0; c < d; ++c) {
    const float x = X[r * ld + c];
    bad |= !(fabsf(x) <= 3.402823466e38f);
    const double t = (double)x * pk.inv_p[c];
    const float ph = (float)(t - floor(t + 0.5));
    float sn, cs;
    sincospif(2.f * ph, &sn, &cs);   // 2 ph is exact
    row[2 * c] = pk.a[c] * cs;
    row[2 * c + 1] = pk.a[c] * sn;
  }
  for (int c = 2 * d; c < DP; ++c) row[c] = 0.f;
  if (bad) *xbad = 1;
}

// ---- bilinear derivative: grid (row blocks, column splits, dimension groups of GD = per_gd(D)) --------------------------------
//   out[0]          = sum g k                                  (dF/dS)
//   out[1 + k]      = sum g k |du_c|^2                         (dF/dl_c  2 l_c log2 e / S)
//   out[1 + GD + k] = sum g k tau_c (us_i uc_j - uc_i us_j)    (dF/dp_c  p_c^2 log2 e / (2 pi S))
// for the group's dimensions c = blockIdx.z GD + k.  Every pair term is formed in fp32 and added to an fp64 accumulator; the
// block reduction runs in a fixed order (no atomics), so repeated calls return identical bits.
template <int D>
__global__ void __launch_bounds__(SIMT_TI)
periodic_bilinear_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int DP, const float* __restrict__ X1, int64_t ld1,
                         const float* __restrict__ X2, int64_t ld2, const float* __restrict__ L16, const float* __restrict__ R16,
                         int64_t n1, int64_t n2, int64_t cols_per_split, double* __restrict__ gout, int gstride) {
  constexpr int GD = per_gd(D);
  constexpr int NO = 1 + 2 * GD;
  __shared__ __align__(16) float zj[SIMT_TJ][2 * D];
  __shared__ float xj[SIMT_TJ][D];
  __shared__ __align__(16) float rj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int c0 = blockIdx.z * GD;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int64_t j_begin = (int64_t)blockIdx.y * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const bool rv = i < n1;
  float zi[2 * D], gi[GD][2], xi[GD], li[TP];   // gi, xi: the group's columns, so that the pair loop indexes registers statically
#pragma unroll
  for (int c = 0; c < 2 * D; ++c) zi[c] = rv ? Z1[i * DP + c] : 0.f;
#pragma unroll
  for (int k = 0; k < GD; ++k) {
    const bool kv = rv && c0 + k < D;
    xi[k] = kv ? X1[i * ld1 + c0 + k] : 0.f;
    gi[k][0] = kv ? Z1[i * DP + 2 * (c0 + k)] : 0.f;
    gi[k][1] = kv ? Z1[i * DP + 2 * (c0 + k) + 1] : 0.f;
  }
#pragma unroll
  for (int c = 0; c < TP; ++c) li[c] = rv ? L16[i * TP + c] : 0.f;
  double acc[NO];
#pragma unroll
  for (int o = 0; o < NO; ++o) acc[o] = 0.0;
  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < SIMT_TJ * 2 * D; e += SIMT_TI) {
      const int r = e / (2 * D), c = e - r * (2 * D);
      zj[r][c] = r < nj ? Z2[(j0 + r) * DP + c] : 0.f;
    }
    for (int e = tid; e < SIMT_TJ * D; e += SIMT_TI) {
      const int r = e / D, c = e - r * D;
      xj[r][c] = r < nj ? X2[(j0 + r) * ld2 + c] : 0.f;
    }
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) (&rj[0][0])[e] = (e / TP < nj) ? R16[j0 * TP + e] : 0.f;
    __syncthreads();
    for (int jj = 0; jj < nj; ++jj) {
      float g = 0.f;
#pragma unroll
      for (int c = 0; c < TP; ++c) g = fmaf(li[c], rj[jj][c], g);
      float a = 0.f;
#pragma unroll
      for (int c = 0; c < 2 * D; ++c) {
        const float df = zi[c] - zj[jj][c];
        a = fmaf(df, df, a);
      }
      const float gk = g * ex2_approx(-0.5f * a);
      acc[0] += (double)gk;
#pragma unroll
      for (int k = 0; k < GD; ++k) {
        const int c = c0 + k;
        if (c < D) {
          const float uci = gi[k][0], usi = gi[k][1], ucj = zj[jj][2 * c], usj = zj[jj][2 * c + 1];
          const float dc = uci - ucj, ds = usi - usj;
          const float tau = xi[k] - xj[jj][c];
          acc[1 + k] += (double)(gk * fmaf(dc, dc, ds * ds));
          acc[1 + GD + k] += (double)(gk * tau * fmaf(usi, ucj, -uci * usj));
        }
      }
    }
  }
  __shared__ double red[SIMT_TI];
  const int64_t blk = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
#pragma unroll
  for (int o = 0; o < NO; ++o) {
    __syncthreads();
    red[tid] = acc[o];
    __syncthreads();
    for (int sft = SIMT_TI / 2; sft > 0; sft >>= 1) {
      if (tid < sft) red[tid] += red[tid + sft];
      __syncthreads();
    }
    if (tid == 0) gout[blk * gstride + blockIdx.z * NO + o] = red[0];
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------------------
static float per_period(const gp_plan* p, int c) { return p->per_p[p->per_n == 1 ? 0 : c]; }
static float per_ls(const gp_plan* p, int c) { return p->ls[p->ls.size() == 1 ? 0 : c]; }

int periodic_pack(gp_plan* p) {
  const int d = p->d;
  GP_REQUIRE(d <= PER_DMAX && (p->per_n == 1 || p->per_n == d), GP_E_SHAPE,
             "periodic plan: %d periods for data of d=%d columns (1 or d periods, d <= %d)", p->per_n, d, PER_DMAX);
  GP_REQUIRE(p->kind == GP_RBF, GP_E_STATE, "periodic plan: gp_plan_set_hypers must pass the kind GP_RBF");
  GP_REQUIRE(p->tasks == nullptr && p->add_M == 0, GP_E_STATE, "periodic plan: task indices and additive plans are not available");
  cudaStream_t st = p->stream;
  const int DP = p->DP;
  PerPack pk;
  memset(&pk, 0, sizeof(pk));
  for (int c = 0; c < d; ++c) {
    pk.inv_p[c] = 1.0 / (double)per_period(p, c);
    pk.a[c] = (float)sqrt(PER_LOG2E / (double)per_ls(p, c));
  }
  GP_CHECK(p->mean.ensure(sizeof(float) * (d + 4)));
  p->xbad = reinterpret_cast<int*>(p->mean.as<float>() + d);
  GP_CUDA(cudaMemsetAsync(p->xbad, 0, sizeof(int), st));
  const float* X2 = p->same ? p->X1 : p->X2;
  const int64_t ld2 = p->same ? p->ld1 : p->ld2;
  GP_CHECK(p->Z2.ensure(sizeof(float) * p->n2 * DP));
  periodic_pack_kernel<<<(unsigned)cdiv(p->n2, 256), 256, 0, st>>>(X2, p->n2, ld2, d, DP, pk, p->Z2.as<float>(), p->xbad);
  p->launches++;
  if (!p->same) {
    GP_CHECK(p->Z1.ensure(sizeof(float) * p->n1 * DP));
    periodic_pack_kernel<<<(unsigned)cdiv(p->n1, 256), 256, 0, st>>>(p->X1, p->n1, p->ld1, d, DP, pk, p->Z1.as<float>(), p->xbad);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  if (p->backend == GP_BACKEND_TCGEN05) {   // the plain tensor-core tiles of the 2d embedding columns
    const int64_t padA = p->rows_pad, padB = p->ntile_j * TILE_J;
    GP_CHECK(p->XA.ensure(sizeof(float) * padA * p->KP));
    GP_CHECK(p->XB.ensure(sizeof(float) * padB * p->KP));
    GP_CHECK(pack_tc_rows(p, p->same ? p->Z2.as<float>() : p->Z1.as<float>(), p->row_count, padA, true, p->XA.as<float>()));
    GP_CHECK(pack_tc_rows(p, p->Z2.as<float>(), p->n2, padB, false, p->XB.as<float>()));
    GP_CHECK(p->Vtiles.ensure(sizeof(float) * p->ntile_j * (2 * TILE_J * TP + TILE_J * TP / 2)));
  }
  p->nparts = p->nsplit;
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// grad_ls = [dF/dl (1 or d) | dF/dp (per_n)], *grad_os = dF/dS; a shared parameter's gradient is the sum over the dimensions
int periodic_bilinear_grad(gp_plan* p, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  const int d = p->d;
  GP_REQUIRE(d >= 1 && d <= PER_DMAX, GP_E_SHAPE, "periodic plan: d=%d > %d", d, PER_DMAX);
  const int GD = per_gd(d), NO = 1 + 2 * GD;
  const int ngrp = (int)cdiv(d, GD), nout = ngrp * NO;
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
  const float* Z1 = p->same ? p->Z2.as<float>() : p->Z1.as<float>();
  const float* X2 = p->same ? p->X1 : p->X2;
  const int64_t ld2 = p->same ? p->ld1 : p->ld2;
  for (int c0 = 0; c0 < s; c0 += TP) {
    const int tc = std::min(TP, s - c0);
    GP_CHECK(to_v16(p, Lf + c0, ldl, tc, p->row_count, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, Rt + c0, ldr, tc, p->n2, p->misc3.as<float>()));
#define GP_PER_BL(DV)                                                                                                          \
  case DV:                                                                                                                     \
    periodic_bilinear_kernel<DV><<<grid, SIMT_TI, 0, p->stream>>>(Z1, p->Z2.as<float>(), p->DP, p->X1, p->ld1, X2, ld2,      \
                                                                  p->misc2.as<float>(), p->misc3.as<float>(), p->row_count,  \
                                                                  p->n2, cps, gout, nout);                                   \
    break;
    switch (d) {
      GP_PER_BL(1) GP_PER_BL(2) GP_PER_BL(3) GP_PER_BL(4) GP_PER_BL(5) GP_PER_BL(6) GP_PER_BL(7) GP_PER_BL(8)
      GP_PER_BL(9) GP_PER_BL(10) GP_PER_BL(11) GP_PER_BL(12) GP_PER_BL(13) GP_PER_BL(14) GP_PER_BL(15) GP_PER_BL(16)
      default:
        set_error("periodic plan: no compiled case for d=%d", d);
        return GP_E_SHAPE;
    }
#undef GP_PER_BL
    p->launches++;
    GP_CUDA(cudaGetLastError());
    GP_CHECK(sum_partials_double(p, gout, nblk, nout, nout, gsum));
    GP_CUDA(cudaMemcpyAsync(hbuf.data(), gsum, sizeof(double) * nout, cudaMemcpyDeviceToHost, p->stream));
    GP_CUDA(cudaStreamSynchronize(p->stream));
    for (int o = 0; o < nout; ++o) total[o] += hbuf[o];
  }
  const double S = p->outputscale;
  const int nls = (int)p->ls.size();
  for (int c = 0; c < nls; ++c) grad_ls[c] = 0.0;
  for (int c = 0; c < p->per_n; ++c) grad_ls[nls + c] = 0.0;
  *grad_os = 0.0;
  for (int c = 0; c < d; ++c) {
    const int base = (c / GD) * NO, k = c % GD;
    const double l = per_ls(p, c), per = per_period(p, c);
    grad_ls[nls == 1 ? 0 : c] += S * total[base + 1 + k] / (2.0 * l * PER_LOG2E);
    grad_ls[nls + (p->per_n == 1 ? 0 : c)] += S * total[base + 1 + GD + k] * 2.0 * M_PI / (per * per * PER_LOG2E);
  }
  *grad_os = total[0];   // every group sums the same g k: group 0's
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_periodic(gp_plan* p, const float* period, int n_period, int d) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  if (period == nullptr || n_period == 0) {   // back to a plain plan
    if (p->per_n == 0) return GP_OK;
    p->per_n = 0;
    p->per_p.clear();
    return (p->data_set && p->hypers_set) ? pack_inputs(p) : GP_OK;
  }
  GP_REQUIRE(p->data_set, GP_E_STATE, "periodic plan: call gp_plan_set_data first");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "a SKI plan cannot become a periodic plan");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel-sum plan cannot become a periodic plan");
  GP_CHECK(refuse_settings(p, CALL_SET_PERIODIC));
  GP_CHECK(refuse_compact(p, "gp_plan_set_periodic"));
  GP_REQUIRE(p->row_begin == 0 && p->row_count == p->n1 && !(p->comm && p->comm->world > 1), GP_E_STATE,
             "a periodic plan is not available on a row-sharded plan");
  GP_REQUIRE(d >= 1 && d <= PER_DMAX, GP_E_SHAPE, "a periodic plan takes 1 <= d <= %d input dimensions (got d=%d)", PER_DMAX, d);
  GP_REQUIRE(d == p->d, GP_E_SHAPE, "periodic plan: parameters for d=%d, data of d=%d columns", d, p->d);
  GP_REQUIRE(n_period == 1 || n_period == d, GP_E_SHAPE, "periodic plan: %d periods for d=%d (1 or d)", n_period, d);
  for (int c = 0; c < n_period; ++c)
    GP_REQUIRE(period[c] > 0.f && isfinite(period[c]), GP_E_SHAPE, "period[%d]=%g must be positive", c, period[c]);
  GP_REQUIRE(!p->hypers_set || p->kind == GP_RBF, GP_E_STATE,
             "gp_plan_set_periodic needs the kind GP_RBF from gp_plan_set_hypers (the plan's kind is %d)", p->kind);
  GP_CUDA(cudaSetDevice(p->device));
  // all or nothing: when the pack fails the plan keeps its previous setting (and packing), so that callers which size the
  // gradient output by the setting they asked for never see a plan in the other state
  const int old_n = p->per_n;
  const std::vector<float> old_p = p->per_p;
  p->per_n = n_period;
  p->per_p.assign(period, period + n_period);
  if (!p->hypers_set) return GP_OK;
  const int st = pack_inputs(p);
  if (st != GP_OK) {
    p->per_n = old_n;
    p->per_p = old_p;
    pack_inputs(p);   // the previous packing; the error reported is the first one
  }
  return st;
}
