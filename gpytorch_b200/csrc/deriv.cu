// deriv.cu -- GPs with derivative observations: the RBF value / gradient operator of RBFKernelGrad (kernels/rbf_kernel_grad.py:
// 60-115; examples/08_Advanced_Usage/Simple_GP_Regression_Derivative_Information_{1d,2d}.ipynb) over interleaved rows i (d+1) + a
// (a = 0: f(x_i), a = 1..d: df/dx_a at x_i), built on a plain RBF data plan without ever storing the N (d+1) x N (d+1) matrix.
//
// Entries.  With D = x_i - x'_j, u_a = D_a / l_a^2 and k = exp(-|D / l|^2 / 2) (s k with the outputscale):
//     [0, 0] = k,   [0, b] = k u_b,   [a, 0] = -k u_a,   [a, b] = k (delta_ab / l_a^2 - u_a u_b).
// D is formed by direct differences of the data plan's packed rows z = (x - mean) sqrt(log2 e) / l (DESIGN 4.10: no cancellation),
// u_c = dz_c / (sqrt(log2 e) l_c); D = 0 gives s and s / l_a^2 on the diagonal exactly, without a special case.
//
// Products.  With h_ij = v0_j + sum_b u_b v^b_j per column:  out0_i = sum_j k h,  out^a_i = (1 / l_a^2) sum_j k v^a_j - sum_j k u_a h.
// deriv_kmv_kernel: one thread owns one point's d + 1 output rows for TW columns; 64-point tiles of the other side and their
// (d + 1) x TW block of V are staged in shared memory (broadcast reads).  The reduced side is split over CTAs into partials that
// deriv_finish_kernel sums in a fixed order into the parent's partial slot 0; the parent's finish kernels (outputscale, noise or
// per-row noise, CG done flag) then run unchanged on n = N (d + 1).  No atomics: repeated calls give identical bits.
//
// Gradients.  For one pair and column, with g = l0 - sum_a u_a l_a (L side) and h as above, sum_ab l_a E_ab r_b = k F with
// F = g h + sum_a l_a r_a / l_a^2, so d/ds = sum k F and (DESIGN 4.14)
//     l_c d/dl_c = s sum k [ (dz_c^2 / log2 e) F - 2 u_c (g r_c - l_c h) - 2 l_c r_c / l_c^2 ].
// deriv_grad_kernel evaluates these per thread in fp32 over its columns and reduces every CTA in fp64; the host adds the CTA
// partials in a fixed order.
//
// Matern-5/2 (gp_plan_set_deriv_kind(..., GP_MATERN52)): the value / gradient operator of Matern52KernelGrad
// (kernels/matern52_kernel_grad.py) over the same interleaved rows, on a plain Matern-5/2 data plan.
//
// Entries.  With D = x_i - x'_j, u_a = D_a / l_a^2, rho = sqrt(5) r (r^2 = sum_c D_c^2 / l_c^2), e = exp(-rho),
// A = (5/3) (1 + rho) e and B = (25/3) e (times the outputscale s):
//     [0, 0] = (1 + rho + rho^2 / 3) e,   [0, b] = A u_b,   [a, 0] = -A u_a,   [a, b] = A delta_ab / l_a^2 - B u_a u_b.
// The data plan packs z = (x - mean) sqrt(10) / l (pack.cu), so rho = sqrt(|dz|^2 / 2) and u_c = dz_c / (sqrt(10) l_c) = dz_c w[c].
// D = 0 gives s and (5/3) s / l_a^2 on the diagonal exactly.
//
// Products.  With h = sum_b u_b v^b per column:  out0 += [0,0] v0 + A h,  out^a += A v^a / l_a^2 - u_a (A v0 + B h): 3 d + 4 FMAs
// per pair and column, one sqrt and one ex2 per pair.
//
// Gradients (DESIGN 4.16).  For one pair and column, with P = l0 r0, h = sum u_b r^b, g = sum u_a l^a, q = sum l^a r^a / l_a^2:
//     F = sum_ab l_a E_ab r_b = [0,0] P + A (l0 h - g r0 + q) - B g h           (d/ds = sum F)
// and with q_c = (D_c / l_c)^2 = dz_c^2 / 10:  l_c d[0,0]/dl_c = A q_c,  l_c dA/dl_c = B q_c,  l_c dB/dl_c = 5 B q_c / rho,
// l_c du_a/dl_c = -2 delta_ac u_a,  l_c d(1 / l_a^2)/dl_c = -2 delta_ac / l_a^2, so
//     l_c dF/dl_c = q_c [A P + B (l0 h - g r0 + q) - (5 B / rho) g h] - 2 A [u_c (l0 r^c - l^c r0) + r^c l^c / l_c^2]
//                   + 2 B u_c (l^c h + r^c g).
// q_c / rho <= rho / 5 is bounded but 0 / 0 at coincident points (and where |dz|^2 flushes to zero): 5 B / rho is taken as 0 at
// rho = 0, where every q_c is 0 as well.
//
// One kernel per job serves both kinds: deriv_kmv_kernel, deriv_grad_kernel, deriv_krows_kernel and deriv_kdiag_kernel stage,
// index and reduce; the kind's DerivTable (deriv_table.cuh) supplies the pair coefficients, the entry, the product's per-column
// and the gradient's per-pair update.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "gp_common.cuh"
#include "deriv_table.cuh"

namespace gp {

static const float* deriv_z1(const gp_plan* q) { return q->same ? q->Z2.as<float>() : q->Z1.as<float>(); }

// out rows i (d+1) + a of the split's partial, columns [c0, c0 + TW)
template <class K, int DP, int TW>
__global__ void __launch_bounds__(DV_TI, K::min_blocks(DP))
deriv_kmv_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ V16, float* __restrict__ part,
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
#pragma unroll (K::unroll(DP))
    for (int jj = 0; jj < DV_TJ; ++jj) {   // staged padding points carry V = 0: they add 0
      float u[DP];
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        const float df = zi[c] - zj[jj][c];
        s = fmaf(df, df, s);
        u[c] = df * hy.w[c];
      }
      const auto p = K::pair(s);
      float kl[DP];
#pragma unroll
      for (int c = 0; c < DP; ++c) kl[c] = K::delta_coef(p) * hy.il2[c];
#pragma unroll
      for (int t = 0; t < TW; ++t) K::template kmv_column<DP, TW>(p, u, kl, vj[jj], t, acc);
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

// parent slot 0 [rows][16] = sum over splits in order (columns >= ncols: 0)
__global__ void deriv_finish_kernel(const float* __restrict__ part, int nsplit, int64_t rows, int ncols, float* __restrict__ out,
                                    const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * TP) return;
  const int c = (int)(idx % TP);
  float s = 0.f;
  if (c < ncols)
    for (int sp = 0; sp < nsplit; ++sp) s += part[(int64_t)sp * rows * TP + idx];
  out[idx] = s;
}

// gout[blk][0] = sum_pairs d/ds, gout[blk][1 + c] = sum_pairs l_c d/dl_c / s (c < d): the kind's grad_pair per pair
template <class K, int DP, int TW>
__global__ void __launch_bounds__(DV_TI)
deriv_grad_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ L16, const float* __restrict__ R16,
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
      K::template grad_pair<DP, TW>(K::pair(s), u, dz2, li, rj[jj], hy, gk, gc);
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
template <class K>
__global__ void deriv_krows_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int DP, int d, const int64_t* __restrict__ idx,
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
  const auto pr = K::pair(s).scaled(os);
  const float ua = a ? (zs[a - 1] - zj[a - 1]) * hy.w[a - 1] : 0.f;
  float* out = OUT + r * ldo + j * rw;
  out[0] = K::entry(pr, a, 0, ua, 0.f, hy);
  for (int b = 1; b < rw; ++b) out[b] = K::entry(pr, a, b, ua, (zs[b - 1] - zj[b - 1]) * hy.w[b - 1], hy);
}

// OUT[i (d+1) + a] = s E(i a, i a): s and DIAG s / l_a^2 on a square plan (D = 0), the full entry for a cross plan of equal sizes
template <class K>
__global__ void deriv_kdiag_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, int DP, int d, int64_t n, float os,
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
  const float ua = a ? (Z1[i * DP + a - 1] - Z2[i * DP + a - 1]) * hy.w[a - 1] : 0.f;
  OUT[e] = *xbad ? __int_as_float(0x7fc00000) : K::entry(K::pair(s).scaled(os), a, a, ua, ua, hy);
}

static int deriv_check_data(const gp_plan* p, const gp_plan* q) {
  GP_REQUIRE(q->data_set && q->hypers_set, GP_E_STATE, "derivative plan: the data plan needs set_data + set_hypers");
  GP_REQUIRE(q->backend == GP_BACKEND_TCGEN05 || q->backend == GP_BACKEND_SIMT, GP_E_SHAPE,
             "derivative plan: the data plan must be a plain kernel plan (not SKI, not a kernel sum, not Kronecker or derivative)");
  if (p->deriv->kind == GP_MATERN52)
    GP_REQUIRE(q->kind == GP_MATERN52, GP_E_SHAPE, "Matern-5/2 derivative plan: the data plan must be a Matern-5/2 plan (kind=%d)", q->kind);
  else
    GP_REQUIRE(q->kind == GP_RBF, GP_E_SHAPE, "derivative observations are available for the RBF kernel only (kind=%d)", q->kind);
  GP_CHECK(refuse_settings(q, CALL_DERIV_DATA_REFRESH));
  GP_REQUIRE(q->row_begin == 0 && q->row_count == q->n1 && !(q->comm && q->comm->world > 1), GP_E_SHAPE,
             "derivative plan: a row-sharded data plan is not available");
  GP_REQUIRE(q->device == p->device && q->stream == p->stream, GP_E_STATE, "derivative plan: the data plan must live on the same device and stream");
  GP_REQUIRE(q->d >= 1 && q->d <= DERIV_DMAX, GP_E_SHAPE, "derivative observations support d <= %d input dimensions (d=%d)", DERIV_DMAX, q->d);
  GP_REQUIRE(q->n1 * (q->d + 1) < ((int64_t)1 << 31) && q->n2 * (q->d + 1) < ((int64_t)1 << 31), GP_E_SHAPE,
             "derivative plan: N (d + 1) must stay below 2^31");
  return GP_OK;
}

// operator geometry from the data plan: N1 (d+1) x N2 (d+1) rows, one partial slot; the derivative kernel's own column split
static void deriv_geometry(gp_plan* p) {
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  const int rw = q->d + 1;
  p->backend = GP_BACKEND_DERIV;
  p->n1 = q->n1 * rw;
  p->n2 = q->n2 * rw;
  p->same = q->same;
  p->d = q->d;
  p->row_begin = 0;
  p->row_count = p->n1;
  p->rows_pad = cdiv(p->row_count, 2 * TILE_I) * 2 * TILE_I;
  p->ntile_i = p->rows_pad / TILE_I;
  p->ntile_j = cdiv(p->n2, TILE_J);
  p->DP = q->DP;
  p->KP = q->KP;
  p->nsplit = 1;
  p->nparts = 1;
  // about two CTAs per SM before the column chunks multiply them, at least 256 points per split; independent of the number of
  // columns, so a column's result does not depend on how many columns a call carries
  const int64_t rb = cdiv(q->n1, DV_TI);
  const int64_t ns = std::max<int64_t>(1, std::min<int64_t>({cdiv(2 * (int64_t)p->n_sm, rb), cdiv(q->n2, 256), (int64_t)32}));
  ds->cps = cdiv(cdiv(q->n2, ns), DV_TJ) * DV_TJ;
  ds->nsplit = (int)cdiv(q->n2, ds->cps);
}

int deriv_refresh(gp_plan* p) {
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  GP_CHECK(deriv_check_data(p, q));
  // d as well: N (d + 1) alone can stay the same while the points, the padded width and the column split change
  GP_REQUIRE(q->d == p->d && p->n1 == q->n1 * (q->d + 1) && p->n2 == q->n2 * (q->d + 1) && p->same == q->same, GP_E_STATE,
             "derivative plan: the data plan changed its size; call gp_plan_set_deriv again");
  p->kind = q->kind;
  p->outputscale = q->outputscale;   // the finish kernels scale the unscaled product by the data plan's s
  p->xbad = q->xbad;
  DerivHyp h;
  memset(&h, 0, sizeof(h));
  const double rc = sqrt(deriv_with_kind(ds->kind, [](auto K) { return decltype(K)::PACK; }));
  for (int c = 0; c < q->d; ++c) {
    const double l = q->ls.size() == 1 ? q->ls[0] : q->ls[c];
    h.w[c] = (float)(1.0 / (rc * l));
    h.il2[c] = (float)(1.0 / (l * l));
  }
  if (!ds->hyp_set || memcmp(&h, &ds->hyp, sizeof(h)) != 0) {
    GP_CHECK(ds->hypd.ensure(sizeof(DerivHyp)));
    ds->hyp = h;
    GP_CUDA(cudaMemcpyAsync(ds->hypd.p, &ds->hyp, sizeof(DerivHyp), cudaMemcpyHostToDevice, p->stream));
    GP_CUDA(cudaStreamSynchronize(p->stream));   // the next refresh may rewrite ds->hyp
    ds->hyp_set = true;
  }
  return GP_OK;
}

int deriv_pack(gp_plan* p) {
  GP_CHECK(deriv_check_data(p, p->deriv->data));
  deriv_geometry(p);
  GP_CHECK(deriv_refresh(p));
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  return GP_OK;
}

// the split partials of the first ncols columns, summed in order into the parent's partial slot 0
static int deriv_finish_launch(gp_plan* p, int ncols, const int* done_flag) {
  gp_deriv_state* ds = p->deriv;
  const int64_t rows = p->n1;
  deriv_finish_kernel<<<(unsigned)cdiv(rows * TP, 256), 256, 0, p->stream>>>(ds->part.as<float>(), ds->nsplit, rows, ncols,
                                                                            p->partial.as<float>(), done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// tot[o] += the CTA partials of ds->gout, in order
static int deriv_sum_gout(gp_plan* p, size_t nblk, int nout, std::vector<double>& tot) {
  std::vector<double> h(nblk * nout);
  GP_CUDA(cudaMemcpyAsync(h.data(), p->deriv->gout.p, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));
  for (size_t b = 0; b < nblk; ++b)
    for (int o = 0; o < nout; ++o) tot[o] += h[b * nout + o];
  return GP_OK;
}

// f(integral_constant<DP>) for the padded widths the product and gradient kernels are built for
template <class F>
static int deriv_with_dp(int DP, F&& f) {
  switch (DP) {
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
    case 12: return f(std::integral_constant<int, 12>{});
    case 16: return f(std::integral_constant<int, 16>{});
  }
  set_error("derivative plan: unsupported padded width DP=%d", DP);
  return GP_E_SHAPE;
}

template <class K, int DP>
static int deriv_kmv_launch(gp_plan* p, const float* V16, int ncols, const int* done_flag) {
  constexpr int TW = K::kmv_tw(DP);
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  const int nchunk = (int)cdiv(ncols, TW);
  const int64_t rows = p->n1;
  GP_CHECK(ds->part.ensure(sizeof(float) * (size_t)ds->nsplit * rows * TP));
  dim3 grid((unsigned)cdiv(q->n1, DV_TI), (unsigned)ds->nsplit, (unsigned)nchunk);
  deriv_kmv_kernel<K, DP, TW><<<grid, DV_TI, 0, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), V16, ds->part.as<float>(), q->n1, q->n2,
                                                             q->d, ds->cps, rows, ds->hyp, done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return deriv_finish_launch(p, nchunk * TW, done_flag);
}

int deriv_kmv_partials(gp_plan* p, const float* V16, const int* done_flag) {
  GP_CHECK(deriv_refresh(p));
  const int ncols = p->kron_cols;
  return deriv_with_kind(p->deriv->kind, [&](auto K) {
    return deriv_with_dp(p->DP, [&](auto D) { return deriv_kmv_launch<decltype(K), decltype(D)::value>(p, V16, ncols, done_flag); });
  });
}

int deriv_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "rows of a derivative plan: at most 65535 rows per call (m=%lld)", (long long)m);
  GP_CHECK(deriv_refresh(p));
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  dim3 grid((unsigned)cdiv(q->n2, 256), (unsigned)m);
  deriv_with_kind(ds->kind, [&](auto K) {
    deriv_krows_kernel<decltype(K)><<<grid, 256, sizeof(float) * q->DP, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), q->DP, q->d, idx,
                                                                                    p->n1, q->n2, q->outputscale, ds->hyp, OUT, ldo, q->xbad);
  });
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int deriv_kdiag(gp_plan* p, float* OUT) {
  GP_CHECK(deriv_refresh(p));
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  GP_REQUIRE(q->same || q->n1 == q->n2, GP_E_SHAPE, "diagonal of a %lld x %lld cross-covariance is undefined", (long long)p->n1, (long long)p->n2);
  deriv_with_kind(ds->kind, [&](auto K) {
    deriv_kdiag_kernel<decltype(K)><<<(unsigned)cdiv(p->n1, 256), 256, 0, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), q->DP, q->d, q->n1,
                                                                                       q->outputscale, ds->hyp, OUT, q->xbad);
  });
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

template <class K, int DP>
static int deriv_grad_launch(gp_plan* p, const float* L16, const float* R16, int ncols, std::vector<double>& tot) {
  constexpr int TW = K::grad_tw(DP);
  gp_deriv_state* ds = p->deriv;
  const gp_plan* q = ds->data;
  const int nout = 1 + q->d;
  const int nchunk = (int)cdiv(ncols, TW);
  dim3 grid((unsigned)cdiv(q->n1, DV_TI), (unsigned)ds->nsplit, (unsigned)nchunk);
  const size_t nblk = (size_t)grid.x * grid.y * grid.z;
  GP_CHECK(ds->gout.ensure(sizeof(double) * nblk * nout));
  deriv_grad_kernel<K, DP, TW><<<grid, DV_TI, 0, p->stream>>>(deriv_z1(q), q->Z2.as<float>(), L16, R16, q->n1, q->n2, q->d, ds->cps,
                                                              ds->hyp, ds->gout.as<double>());
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return deriv_sum_gout(p, nblk, nout, tot);
}

int deriv_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  GP_CHECK(deriv_refresh(p));
  const gp_plan* q = p->deriv->data;
  const int d = q->d;
  std::vector<double> tot(1 + d, 0.0);
  GP_CHECK(p->misc2.ensure(sizeof(float) * p->n1 * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * p->n2 * TP));
  for (int c0 = 0; c0 < s; c0 += TP) {
    const int tc = std::min(TP, s - c0);
    GP_CHECK(to_v16(p, L + c0, ldl, tc, p->n1, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, R + c0, ldr, tc, p->n2, p->misc3.as<float>()));
    GP_CHECK(deriv_with_kind(p->deriv->kind, [&](auto K) {
      return deriv_with_dp(p->DP, [&](auto D) {
        return deriv_grad_launch<decltype(K), decltype(D)::value>(p, p->misc2.as<float>(), p->misc3.as<float>(), tc, tot);
      });
    }));
  }
  int bad = 0;
  GP_CUDA(cudaMemcpyAsync(&bad, q->xbad, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));
  const double os = q->outputscale;
  *grad_os = bad ? NAN : tot[0];
  if (q->ls.size() > 1) {
    for (int c = 0; c < d; ++c) grad_ls[c] = bad ? NAN : os * tot[1 + c] / (double)q->ls[c];
  } else {
    double sum = 0.0;
    for (int c = 0; c < d; ++c) sum += tot[1 + c];
    grad_ls[0] = bad ? NAN : os * sum / (double)q->ls[0];
  }
  return GP_OK;
}

double deriv_trace(const gp_plan* p) {
  const gp_deriv_state* ds = p->deriv;
  const double f = deriv_with_kind(ds->kind, [](auto K) { return decltype(K)::DIAG; });   // the derivative rows' diagonal is f s / l_c^2
  double t = 1.0;
  for (int c = 0; c < ds->data->d; ++c) t += f * (double)ds->hyp.il2[c];
  return (double)ds->data->outputscale * (double)ds->data->n2 * t;
}

static void deriv_release(gp_plan* p) {
  gp_deriv_state* ds = p->deriv;
  gp::DevBuf* bufs[] = {&ds->part, &ds->gout, &ds->hypd};
  for (auto* b : bufs) b->release();
  delete ds;
  p->deriv = nullptr;
}

// gp_plan_set_deriv (RBF) and gp_plan_set_deriv_kind: `call` and `data_role` name the C call in the refusals
static int deriv_set(gp_plan* p, gp_plan* data, int kind, CallId call, CallId data_role) {
  GP_CUDA(cudaSetDevice(p->device));
  if (data == nullptr) {
    if (p->deriv) {
      GP_CUDA(cudaStreamSynchronize(p->stream));
      deriv_release(p);
      p->backend_req = GP_BACKEND_AUTO;
      p->backend = GP_BACKEND_SIMT;
      p->data_set = false;   // the rows belonged to the data plan: gp_plan_set_data again
    }
    return GP_OK;
  }
  GP_REQUIRE(data != p, GP_E_STATE, "a derivative plan cannot be its own data plan");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "a SKI plan cannot become a derivative plan");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel-sum plan cannot become a derivative plan");
  GP_CHECK(refuse_settings(p, call));
  GP_CHECK(refuse_settings(data, data_role));
  GP_REQUIRE(!(p->comm && p->comm->world > 1), GP_E_SHAPE, "a derivative plan is not available on a row-sharded plan");
  gp_deriv_state* ds = p->deriv ? p->deriv : new gp_deriv_state();
  gp_plan* old = ds->data;
  const int old_kind = ds->kind;
  ds->data = data;
  ds->kind = kind;
  p->deriv = ds;
  const int st = deriv_check_data(p, data);
  if (st != GP_OK) {
    if (old) { ds->data = old; ds->kind = old_kind; }
    else deriv_release(p);
    return st;
  }
  p->backend_req = GP_BACKEND_DERIV;
  deriv_geometry(p);
  p->data_set = true;
  return p->hypers_set ? deriv_pack(p) : GP_OK;   // without the noise yet: packed by gp_plan_set_hypers
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_deriv(gp_plan* p, gp_plan* data) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  return deriv_set(p, data, GP_RBF, CALL_SET_DERIV, CALL_DERIV_DATA);
}

extern "C" int gp_plan_set_deriv_kind(gp_plan* p, gp_plan* data, int kind) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(kind == GP_RBF || kind == GP_MATERN52, GP_E_SHAPE,
             "derivative observations are available for the RBF and Matern-5/2 kernels (kind=%d)", kind);
  return deriv_set(p, data, kind, CALL_SET_DERIV_KIND, CALL_DERIV_KIND_DATA);
}
