// kmv_simt.cu -- fp32 CUDA-core fused kernel-matmul, row extraction, diagonal and the
// bilinear hyper-parameter gradient.
//
// The SIMT K.V kernel is the bring-up / cross-check path for the tensor-core kernel (kmv_tc.cu) and
// the backend for d > 41.  It evaluates a_ij = -0.5 |z_i - z_j|^2 by direct differences (no
// cancellation), so it is also the more accurate of the two.
// Reference semantics: LazyEvaluatedKernelTensor._matmul (lazy/lazy_evaluated_kernel_tensor.py:245-276),
// _getitem (:136-243), _diagonal (:107-133), _bilinear_derivative (:69-105).
#include "gp_common.cuh"
#include "simt_pass.cuh"
#include "ski_rows.cuh"

namespace gp {

// grid (row blocks, nsplit); 128 threads, one output row each; partial[split][row][16]
template <int KIND, int DP>
__device__ __forceinline__ void kmv_simt_body(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ V16,
                                              float* __restrict__ partial, int64_t n1, int64_t n2, int64_t rows_pad,
                                              int64_t cols_per_split, int same, int64_t row_begin, const int* __restrict__ done_flag,
                                              CovParam cp) {
  if (done_flag && *done_flag) return;
  __shared__ __align__(16) float zj[SIMT_TJ][DP];
  __shared__ __align__(16) float vj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int split = blockIdx.y;
  const int64_t j_begin = (int64_t)split * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  float zi[DP];
  const bool rv = i < n1;
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? Z1[i * DP + c] : 0.f;
  float acc[TP];
#pragma unroll
  for (int c = 0; c < TP; ++c) acc[c] = 0.f;
  const int64_t gi = i + row_begin;

  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < SIMT_TJ * DP; e += SIMT_TI) {
      int jj = e / DP;
      (&zj[0][0])[e] = (jj < nj) ? Z2[j0 * DP + e] : 0.f;
    }
    for (int e = tid; e < SIMT_TJ * TP; e += SIMT_TI) {
      int jj = e / TP;
      (&vj[0][0])[e] = (jj < nj) ? V16[j0 * TP + e] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int jj = 0; jj < SIMT_TJ; ++jj) {
      float a;
      if constexpr (is_poly_code(KIND)) {   // a = x_i . x_j + c: every entry, the diagonal too, from the raw inputs
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < DP; ++c) s = fmaf(zi[c], zj[jj][c], s);
        a = s + cp.offset;
      } else {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < DP; ++c) {
          float df = zi[c] - zj[jj][c];
          s = fmaf(df, df, s);
        }
        a = -0.5f * s;
        if (same && (j0 + jj) == gi) a = 0.f;  // exact diagonal (kernel.py:44-45)
      }
      float k = cov_from_arg<KIND>(a, cp);
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
template <int KIND, int DP>
__global__ void __launch_bounds__(SIMT_TI)
kmv_simt_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ V16,
                float* __restrict__ partial, int64_t n1, int64_t n2, int64_t rows_pad, int64_t cols_per_split,
                int same, int64_t row_begin, const int* __restrict__ done_flag) {
  kmv_simt_body<KIND, DP>(Z1, Z2, V16, partial, n1, n2, rows_pad, cols_per_split, same, row_begin, done_flag, CovParam{});
}
// the RQ kernel with its per-plan alpha
template <int DP>
__global__ void __launch_bounds__(SIMT_TI)
rq_simt_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ V16,
               float* __restrict__ partial, int64_t n1, int64_t n2, int64_t rows_pad, int64_t cols_per_split,
               int same, int64_t row_begin, const int* __restrict__ done_flag, CovParam cp) {
  kmv_simt_body<RQ_K, DP>(Z1, Z2, V16, partial, n1, n2, rows_pad, cols_per_split, same, row_begin, done_flag, cp);
}
// the polynomial kernel with its per-plan power and offset
template <int DP>
__global__ void __launch_bounds__(SIMT_TI)
poly_simt_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ V16,
                 float* __restrict__ partial, int64_t n1, int64_t n2, int64_t rows_pad, int64_t cols_per_split,
                 int same, int64_t row_begin, const int* __restrict__ done_flag, CovParam cp) {
  kmv_simt_body<POLY_K, DP>(Z1, Z2, V16, partial, n1, n2, rows_pad, cols_per_split, same, row_begin, done_flag, cp);
}

struct SimtLaunch {
  const float* Z1;
  const float* Z2;
  const float* V16;
  float* partial;
  int64_t n2, cps, row_begin;
  int nsplit;
};

template <int KIND>
static int launch_simt_kind(gp_plan* p, const SimtLaunch& a, const int* done_flag) {
  int64_t rows_pad = p->rows_pad;
  dim3 grid((unsigned)cdiv(p->row_count, SIMT_TI), (unsigned)a.nsplit);
  const bool ok = with_width<4, 8, 12, 16, 24, 32, 48, 64, 96, 128>(p->DP, [&](auto w) {
    constexpr int D = decltype(w)::value;
    if constexpr (KIND == POLY_K)
      poly_simt_kernel<D><<<grid, SIMT_TI, 0, p->stream>>>(a.Z1, a.Z2, a.V16, a.partial, p->row_count, a.n2, rows_pad, a.cps,
                                                           p->same ? 1 : 0, a.row_begin, done_flag, cov_param(p));
    else if constexpr (KIND == RQ_K)
      rq_simt_kernel<D><<<grid, SIMT_TI, 0, p->stream>>>(a.Z1, a.Z2, a.V16, a.partial, p->row_count, a.n2, rows_pad, a.cps,
                                                         p->same ? 1 : 0, a.row_begin, done_flag, cov_param(p));
    else
      kmv_simt_kernel<KIND, D><<<grid, SIMT_TI, 0, p->stream>>>(a.Z1, a.Z2, a.V16, a.partial, p->row_count, a.n2, rows_pad, a.cps,
                                                                p->same ? 1 : 0, a.row_begin, done_flag);
  });
  if (!ok) {
    set_error("unsupported DP=%d", p->DP);
    return GP_E_SHAPE;
  }
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

static int launch_simt_any(gp_plan* p, int kind, const SimtLaunch& a, const int* done_flag) {
  switch (rq_code(p, kind)) {
    case GP_RBF: return launch_simt_kind<GP_RBF>(p, a, done_flag);
    case GP_MATERN12: return launch_simt_kind<GP_MATERN12>(p, a, done_flag);
    case GP_MATERN32: return launch_simt_kind<GP_MATERN32>(p, a, done_flag);
    case GP_MATERN52: return launch_simt_kind<GP_MATERN52>(p, a, done_flag);
    case RQ_K: return launch_simt_kind<RQ_K>(p, a, done_flag);
    case POLY_K: return launch_simt_kind<POLY_K>(p, a, done_flag);
  }
  set_error("bad kernel kind %d", kind);
  return GP_E_SHAPE;
}

int kmv_simt_launch(gp_plan* p, const float* V16, const int* done_flag) {
  const float* Z1 = p->same ? p->Z2.as<float>() + p->row_begin * p->DP : p->Z1.as<float>();
  const SimtLaunch a{Z1, p->Z2.as<float>(), V16, partial_ptr(p), p->n2, p->tiles_per_split * SIMT_TJ, p->row_begin, p->nsplit};
  return launch_simt_any(p, p->kind, a, done_flag);
}

int kmv_simt_launch_cols(gp_plan* p, int kind, const float* Z1, const float* Z2, const float* V16, float* partial, int64_t n2,
                         int64_t cols_per_split, int nsplit, int64_t diag_row_begin, const int* done_flag) {
  const SimtLaunch a{Z1, Z2, V16, partial, n2, cols_per_split, diag_row_begin, nsplit};
  return launch_simt_any(p, kind, a, done_flag);
}

static int kmv_partials_base(gp_plan* p, const float* V16, const int* done_flag) {
  if (p->kron) return kron_kmv_partials(p, V16, done_flag);
  if (p->deriv) return deriv_kmv_partials(p, V16, done_flag);
  if (p->tasks) return tasks_kmv_partials(p, V16, p->kind, done_flag);
  if (p->backend == GP_BACKEND_SKI) return ski_kmv_partials(p, V16, done_flag);
  if (p->compact) return compact_kmv_partials(p, V16, done_flag);
  if (p->backend == GP_BACKEND_PRODUCT) {
    GP_CHECK(product_refresh(p));   // before the V tiles are packed: a re-packed factor can change the backend
    if (p->prod_tc) GP_CHECK(pack_v_tiles(p, V16));
    return product_kmv_launch(p, V16, done_flag);
  }
  if (p->backend == GP_BACKEND_SUM) {
    if (p->sum_any_tc) GP_CHECK(pack_v_tiles(p, V16));
    return sum_kmv_launch(p, V16, done_flag);
  }
  if (p->backend == GP_BACKEND_TCGEN05) {
    GP_CHECK(pack_v_tiles(p, V16));
    return kmv_tc_launch(p, done_flag);
  }
  if (p->add_M) return additive_kmv_launch(p, V16, done_flag);
  if (p->sm_Q) return spectral_kmv_launch(p, V16, done_flag);
  return kmv_simt_launch(p, V16, done_flag);
}

// the backend's slots, then the low-rank slot (lowrank.cu) when the plan has one
int kmv_partials(gp_plan* p, const float* V16, const int* done_flag) {
  GP_CHECK(kmv_partials_base(p, V16, done_flag));
  return lowrank_partials(p, V16, done_flag);
}

// OUT[r, c] = os * sum_s partial[s][r][c] + noise * V16[row_begin + r][c]
__global__ void kmv_finish_user_kernel(const float* __restrict__ partial, int nsplit, int64_t rows, int64_t rows_pad,
                                       float os, const float* __restrict__ pscale, float noise_add, const float* __restrict__ dvec, const float* __restrict__ V16,
                                       int64_t row_begin, float* __restrict__ OUT, int64_t ldo, int t, const int* __restrict__ xbad) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * TP) return;
  int64_t r = idx / TP;
  int c = (int)(idx % TP);
  if (c >= t) return;
  float s = 0.f;
  if (pscale) {   // kernel sum: slot sp belongs to the term with outputscale pscale[sp]
    for (int sp = 0; sp < nsplit; ++sp) s = fmaf(pscale[sp], partial[((int64_t)sp * rows_pad + r) * TP + c], s);
  } else {
    for (int sp = 0; sp < nsplit; ++sp) s += partial[((int64_t)sp * rows_pad + r) * TP + c];
    s *= os;
  }
  float o = s;
  if (dvec) o = fmaf(dvec[row_begin + r], V16[(row_begin + r) * TP + c], o);
  else if (noise_add != 0.f) o = fmaf(noise_add, V16[(row_begin + r) * TP + c], o);
  if (*xbad) o = __int_as_float(0x7fc00000);
  OUT[r * ldo + c] = o;
}

int kmv_finish_user(gp_plan* p, const float* V16, float* OUT, int64_t ldo, int t, int add_noise) {
  int64_t rows_pad = p->rows_pad;
  int64_t tot = p->row_count * TP;
  float na = (add_noise && p->same) ? p->noise : 0.f;
  const float* dv = (add_noise && p->same) ? p->noise_diag : nullptr;
  kmv_finish_user_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, p->stream>>>(p->partial.as<float>(), nslots(p), p->row_count,
                                                                          rows_pad, kernel_scale(p), part_scale_ptr(p), na, dv, V16, p->row_begin,
                                                                          OUT, ldo, t, p->xbad);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// ---- rows and diagonals: os * k(x1_i, x2_j) of one pair of packed rows of width DP ---------------------------------------
template <int KIND>
struct PlainEntry {
  static constexpr bool XBAD = false;
  const float* Z1;
  const float* Z2;
  int ld;   // DP
  float os;
  int same;
  int64_t row_begin;
  CovParam cp;
  __host__ __device__ int width() const { return ld; }
  __device__ __forceinline__ float entry(const float* za, const float* zb, int64_t i, int64_t j) const {
    float a;
    if constexpr (is_poly_code(KIND)) {   // also the square diagonal S (|x_i|^2 + c)^p (Z1 = Z2)
      a = poly_arg(za, zb, ld, cp.offset);
    } else {
      float s = 0.f;
      for (int c = 0; c < ld; ++c) {
        float df = za[c] - zb[c];
        s = fmaf(df, df, s);
      }
      a = -0.5f * s;
      if (same && (i + row_begin) == j) a = 0.f;
    }
    return os * cov_from_arg<KIND>(a, cp);
  }
};

template <bool XB>
__global__ void fill_kernel(float* __restrict__ OUT, int64_t n, float v, const int* __restrict__ xbad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if constexpr (XB)
    OUT[i] = *xbad ? __int_as_float(0x7fc00000) : v;
  else
    OUT[i] = v;
}
template __global__ void fill_kernel<false>(float* __restrict__, int64_t, float, const int* __restrict__);
template __global__ void fill_kernel<true>(float* __restrict__, int64_t, float, const int* __restrict__);

// the diagonal of a square kernel sum with a polynomial term, term by term in term order: OUT[i] (+)= os_t k_t(x_i, x_i), the
// constant os_t for a stationary term, os_t (|x_i|^2 + c_t)^p_t for a polynomial one (Z: its packed rows)
__global__ void sum_diag_term_kernel(const float* __restrict__ Z, int DP, int64_t n, float os, CovParam cp, int first,
                                     float* __restrict__ OUT) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = Z ? os * cov_from_arg<POLY_K>(poly_arg(Z + i * DP, Z + i * DP, DP, cp.offset), cp) : os;
  OUT[i] = first ? v : OUT[i] + v;
}

// ---- bilinear derivative: sum_ij (Lf_i . Rt_j) dk_ij/dtheta ---------------------------------
// grid (row blocks, col splits); per-thread row, staged columns; outputs per block partial sums
//   gout[block][0]      = sum_ij w_ij k_ij                 (-> d/d outputscale)
//   gout[block][1 + c]  = sum_ij w_ij g_ij (z_ic-z_jc)^2   (ARD)  or  gout[block][1] = sum w_ij g_ij (scalar l)
//   RQ: gout[block][1 + n_ls] = sum_ij w_ij dk_ij/dalpha    (n_ls = d (ARD) or 1)
template <int KIND, int DP, bool ARD>
__global__ void __launch_bounds__(SIMT_TI)
bilinear_kernel(const float* __restrict__ Z1, const float* __restrict__ Z2, const float* __restrict__ L16,
                const float* __restrict__ R16, int64_t n1, int64_t n2, int64_t cols_per_split, int same,
                int64_t row_begin, int d, double* __restrict__ gout, int gstride, CovParam cp) {
  constexpr bool RQ = KIND == RQ_K;
  constexpr bool POLY = KIND == POLY_K;   // g = dk/dc, one output beside dF/dS (ARD is not used)
  __shared__ __align__(16) float zj[SIMT_TJ][DP];
  __shared__ __align__(16) float rj[SIMT_TJ][TP];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int64_t j_begin = (int64_t)blockIdx.y * cols_per_split;
  const int64_t j_end = min(n2, j_begin + cols_per_split);
  const bool rv = i < n1;
  float zi[DP], li[TP];
#pragma unroll
  for (int c = 0; c < DP; ++c) zi[c] = rv ? Z1[i * DP + c] : 0.f;
#pragma unroll
  for (int c = 0; c < TP; ++c) li[c] = rv ? L16[i * TP + c] : 0.f;
  constexpr int NG = ARD ? DP : 1;
  float gk = 0.f, gl[NG], ga = 0.f;
#pragma unroll
  for (int c = 0; c < NG; ++c) gl[c] = 0.f;
  const int64_t gi = i + row_begin;
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
      float s = 0.f;
      float df2[DP];
      float a;
      if constexpr (POLY) {
#pragma unroll
        for (int c = 0; c < DP; ++c) s = fmaf(zi[c], zj[jj][c], s);
        a = s + cp.offset;
      } else {
#pragma unroll
        for (int c = 0; c < DP; ++c) {
          float df = zi[c] - zj[jj][c];
          df2[c] = df * df;
          s += df2[c];
        }
        a = -0.5f * s;
        if (same && (j0 + jj) == gi) a = 0.f;
      }
      float k;
      float g = dcov_from_arg<KIND>(a, &k, cp);
      gk = fmaf(w, k, gk);
      if (RQ) ga = fmaf(w, -k * rq_phi(rq_t(a, cp)), ga);
      if (ARD && !POLY) {
        // dk/dl_c = g * (z_ic - z_jc)^2 / (s * l_c)   (g/l is the scalar-lengthscale derivative)
        float gs = (s > 0.f) ? w * g / s : 0.f;
#pragma unroll
        for (int c = 0; c < NG; ++c) gl[c] = fmaf(gs, df2[c], gl[c]);
      } else {
        gl[0] = fmaf(w, g, gl[0]);
      }
    }
  }
  // block reduction in double
  __shared__ double red[SIMT_TI];
  const int nls = ARD ? d : 1;
  const int nout = 1 + nls + (RQ ? 1 : 0);
  const int64_t blk = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
  for (int o = 0; o < nout; ++o) {
    float v = (o == 0) ? gk : 0.f;
    if (o > 0) {
#pragma unroll
      for (int c = 0; c < NG; ++c)
        if (c == o - 1) v = gl[c];
    }
    if (RQ && o == 1 + nls) v = ga;   // after the loop: an ARD thread holds DP >= d + 1 (padding) accumulators
    __syncthreads();
    block_sum_store<SIMT_TI>(red, (double)v, gout + blk * gstride + o);
  }
}

// xbad: non-finite inputs make every gradient NaN, as in the reference (the covariance clamps would otherwise treat every pair
// as distance 0 and return finite sums)
__global__ void sum_partials_double_kernel(const double* __restrict__ in, int64_t nblk, int stride, int nout,
                                           double* __restrict__ out, const int* __restrict__ xbad) {
  int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= nout) return;
  double s = 0.0;
  for (int64_t b = 0; b < nblk; ++b) s += in[b * stride + o];
  out[o] = *xbad ? __longlong_as_double(0x7ff8000000000000LL) : s;
}

// tensor-core path of the bilinear derivative: gout[block][o] = sum_{r,c} L16[r][c] * sum_split partial[split][r][c]
__global__ void bilin_dot_kernel(const float* __restrict__ partial, int nsplit, int64_t rows, int64_t rows_pad,
                                 const float* __restrict__ L16, double* __restrict__ gout, int gstride, int o) {
  __shared__ double red[256];
  double acc = 0.0;
  for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < rows * TP; e += (int64_t)gridDim.x * 256) {
    float s = 0.f;
    for (int sp = 0; sp < nsplit; ++sp) s += partial[(int64_t)sp * rows_pad * TP + e];
    acc += (double)L16[e] * (double)s;
  }
  block_sum_store<256>(red, acc, gout + (int64_t)blockIdx.x * gstride + o);
}

int sum_partials_double(gp_plan* p, const double* in, int64_t nblk, int stride, int nout, double* out) {
  sum_partials_double_kernel<<<(unsigned)cdiv(nout, 64), 64, 0, p->stream>>>(in, nblk, stride, nout, out, p->xbad);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

struct BilinLaunch {
  const float* Z1;
  const float* Z2;
  int64_t n2, row_begin;
};

template <int KIND, bool ARD>
static int launch_bilinear(gp_plan* p, const BilinLaunch& a, const float* L16, const float* R16, double* gout, int gstride, dim3 grid,
                           int64_t cps) {
  // DP <= 64: gp_bilinear_grad refuses wider plans before any launch
  with_width<4, 8, 12, 16, 24, 32, 48, 64>(p->DP, [&](auto w) {
    bilinear_kernel<KIND, decltype(w)::value, ARD><<<grid, SIMT_TI, 0, p->stream>>>(
        a.Z1, a.Z2, L16, R16, p->row_count, a.n2, cps, p->same ? 1 : 0, a.row_begin, p->d, gout, gstride, cov_param(p));
  });
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// the SIMT derivative launch split of gp_bilinear_grad over n2 columns
void bilinear_split(const gp_plan* p, int64_t n2, dim3* grid, int64_t* cps) {
  int64_t ntj = cdiv(n2, SIMT_TJ);
  int nsp = (int)std::min<int64_t>(ntj, std::max<int64_t>(1, (2 * p->n_sm) / std::max<int64_t>(1, cdiv(p->row_count, SIMT_TI))));
  *cps = cdiv(ntj, nsp) * SIMT_TJ;
  nsp = (int)cdiv(n2, *cps);
  *grid = dim3((unsigned)cdiv(p->row_count, SIMT_TI), (unsigned)nsp);
}

template <bool ARD>
static int launch_bilinear_any(gp_plan* p, const BilinLaunch& a, const float* L16, const float* R16, double* gout, int gstride,
                               dim3 grid, int64_t cps) {
  switch (p->kind) {
    case GP_RBF: return launch_bilinear<GP_RBF, ARD>(p, a, L16, R16, gout, gstride, grid, cps);
    case GP_MATERN12: return launch_bilinear<GP_MATERN12, ARD>(p, a, L16, R16, gout, gstride, grid, cps);
    case GP_MATERN32: return launch_bilinear<GP_MATERN32, ARD>(p, a, L16, R16, gout, gstride, grid, cps);
    case GP_RQ: return launch_bilinear<RQ_K, ARD>(p, a, L16, R16, gout, gstride, grid, cps);
    case GP_POLY: return launch_bilinear<POLY_K, false>(p, a, L16, R16, gout, gstride, grid, cps);
    default: return launch_bilinear<GP_MATERN52, ARD>(p, a, L16, R16, gout, gstride, grid, cps);
  }
}

// f(std::integral_constant<int, KIND>()) for the covariance code of a plain plan's rows and diagonal
template <class F>
static void with_plain_kind(int kind, F&& f) {
  switch (kind) {
    case GP_RBF: return f(std::integral_constant<int, GP_RBF>());
    case GP_MATERN12: return f(std::integral_constant<int, GP_MATERN12>());
    case GP_MATERN32: return f(std::integral_constant<int, GP_MATERN32>());
    case GP_RQ: return f(std::integral_constant<int, RQ_K>());
    case GP_POLY: return f(std::integral_constant<int, POLY_K>());
    case GP_PPOLY: return f(std::integral_constant<int, PP_K>());
    default: return f(std::integral_constant<int, GP_MATERN52>());
  }
}

bool sum_has_poly(const gp_plan* p) {
  for (const gp_plan* t : p->terms)
    if (t->kind == GP_POLY) return true;
  return false;
}

// per-row diagonal of a square kernel sum with a polynomial term: the terms' diagonals added in term order
int sum_kdiag_terms(gp_plan* p, float* OUT) {
  const unsigned g = (unsigned)cdiv(p->row_count, 256);
  for (size_t t = 0; t < p->terms.size(); ++t) {
    const gp_plan* q = p->terms[t];
    const float* Z = q->kind == GP_POLY ? q->Z2.as<float>() + p->row_begin * q->DP : nullptr;
    sum_diag_term_kernel<<<g, 256, 0, p->stream>>>(Z, q->DP, p->row_count, q->outputscale, cov_param(q), t == 0 ? 1 : 0, OUT);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int64_t bilinear_blocks(const gp_plan* p, int64_t n2) {
  dim3 grid;
  int64_t cps;
  bilinear_split(p, n2, &grid, &cps);
  return (int64_t)grid.x * grid.y;
}

int bilinear_launch_cols(gp_plan* p, bool ard, const float* Z1, const float* Z2, const float* L16, const float* R16, int64_t n2,
                         int64_t diag_row_begin, double* gout, int gstride, int64_t* nblk_out) {
  dim3 grid;
  int64_t cps;
  bilinear_split(p, n2, &grid, &cps);
  *nblk_out = (int64_t)grid.x * grid.y;
  const BilinLaunch a{Z1, Z2, n2, diag_row_begin};
  return ard ? launch_bilinear_any<true>(p, a, L16, R16, gout, gstride, grid, cps)
             : launch_bilinear_any<false>(p, a, L16, R16, gout, gstride, grid, cps);
}

}  // namespace gp

using namespace gp;

static int krows_base(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);

extern "C" int gp_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(p->backend != GP_BACKEND_SUM || p->lr_U, GP_E_SHAPE, "row extraction of a kernel sum: call gp_krows on every term and add");
  GP_REQUIRE(m >= 0 && ldo >= p->n2, GP_E_SHAPE, "bad krows shape");
  if (m == 0) return GP_OK;
  if (p->backend == GP_BACKEND_PRODUCT) return product_krows(p, idx, m, OUT, ldo);
  if (p->kron) return kron_krows(p, idx, m, OUT, ldo);
  if (p->deriv) return deriv_krows(p, idx, m, OUT, ldo);
  if (p->lr_U) {   // rows of the operator the plan multiplies: s K - U U^T
    GP_CHECK(p->backend == GP_BACKEND_SUM ? sum_krows(p, idx, m, OUT, ldo) : krows_base(p, idx, m, OUT, ldo));
    return lowrank_krows(p, idx, m, OUT, ldo);
  }
  GP_CHECK(krows_base(p, idx, m, OUT, ldo));
  return p->tasks ? tasks_krows_scale(p, idx, m, OUT, ldo) : GP_OK;
}

static int krows_base(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  if (p->backend == GP_BACKEND_SKI) return ski_krows(p, idx, m, OUT, ldo);   // separable entries (ski_rows.cuh)
  if (p->add_M) return additive_krows(p, idx, m, OUT, ldo);
  if (p->sm_Q) return spectral_krows(p, idx, m, OUT, ldo);
  const float* Z1 = p->same ? p->Z2.as<float>() + p->row_begin * p->DP : p->Z1.as<float>();
  int st = GP_OK;
  with_plain_kind(p->kind, [&](auto k) {
    const PlainEntry<decltype(k)::value> src{Z1, p->Z2.as<float>(), p->DP, p->outputscale, p->same, p->row_begin, cov_param(p)};
    st = launch_krows(p, src, idx, m, OUT, ldo);
  });
  return st;
}

static int kdiag_base(gp_plan* p, float* OUT);

extern "C" int gp_kdiag(gp_plan* p, float* OUT) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(p->backend != GP_BACKEND_SUM || p->lr_U, GP_E_SHAPE, "diagonal of a kernel sum: call gp_kdiag on every term and add");
  if (p->backend == GP_BACKEND_PRODUCT) {   // square: the constant S = prod_f s_f (kdiag_base); cross: the factors' diagonals
    GP_CHECK(product_refresh(p));
    if (!p->same) return product_kdiag_cross(p, OUT);
  }
  if (p->kron) return kron_kdiag(p, OUT);
  if (p->deriv) return deriv_kdiag(p, OUT);
  if (p->lr_U) {   // diag(s K) - sum_j U_ij^2
    if (p->backend == GP_BACKEND_SUM && sum_has_poly(p)) {
      GP_CHECK(sum_kdiag_terms(p, OUT));   // a polynomial term's diagonal is not constant
    } else if (p->backend == GP_BACKEND_SUM) {
      // a low-rank plan is square: every stationary term contributes its constant outputscale, added in term order
      float os = 0.f;
      for (gp_plan* t : p->terms) os += t->outputscale;
      fill_kernel<false><<<(unsigned)cdiv(p->row_count, 256), 256, 0, p->stream>>>(OUT, p->row_count, os, nullptr);
      p->launches++;
    } else {
      GP_CHECK(kdiag_base(p, OUT));
    }
    return lowrank_kdiag(p, OUT);
  }
  GP_CHECK(kdiag_base(p, OUT));
  return p->tasks ? tasks_kdiag_scale(p, OUT) : GP_OK;
}

static int kdiag_base(gp_plan* p, float* OUT) {
  if (p->backend == GP_BACKEND_SKI) return ski_kdiag(p, OUT);   // not constant: w_i^T K_uu w_i (ski_rows.cuh)
  if (p->add_M) return additive_kdiag(p, OUT);   // square: the constant sum_m e_m(s); cross: per pair
  if (p->sm_Q) return spectral_kdiag(p, OUT);    // square: the constant S (sum_q w_q)^d; cross: per pair
  if (p->same && p->kind == GP_POLY) {   // a dot-product kernel: S (|x_i|^2 + c)^p, row by row
    const float* Z = p->Z2.as<float>() + p->row_begin * p->DP;
    return launch_kdiag(p, OUT, nullptr, PlainEntry<POLY_K>{Z, Z, p->DP, p->outputscale, 0, 0, cov_param(p)});
  }
  // stationary kernels: k(x,x) = outputscale on a square plan (lazy_evaluated_kernel_tensor.py:107-133 evaluates
  // kernel(diag=True)), per pair on a cross plan
  int st = GP_OK;
  with_plain_kind(p->kind, [&](auto k) {
    const PlainEntry<decltype(k)::value> src{p->Z1.as<float>(), p->Z2.as<float>(), p->DP, p->outputscale, 0, 0, cov_param(p)};
    st = launch_kdiag(p, OUT, &p->outputscale, src);
  });
  return st;
}

extern "C" int gp_bilinear_grad(gp_plan* p, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr, int s,
                                double* grad_ls, double* grad_os) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_CHECK(refuse_settings(p, CALL_BILINEAR_GRAD));
  GP_REQUIRE(p->backend != GP_BACKEND_SUM, GP_E_SHAPE, "gradients of a kernel sum: call gp_bilinear_grad on every term");
  GP_REQUIRE(s >= 1, GP_E_SHAPE, "s must be >= 1");
  GP_REQUIRE(Lf && Rt, GP_E_SHAPE, "gp_bilinear_grad: null factor");
  // a single row is read at offset 0 only, so it may carry any row stride
  GP_REQUIRE((ldl >= s || p->row_count == 1) && (ldr >= s || p->n2 == 1), GP_E_SHAPE,
             "gp_bilinear_grad: leading dimensions must be >= s (ldl=%lld, ldr=%lld, s=%d)", (long long)ldl, (long long)ldr, s);
  if (p->backend == GP_BACKEND_PRODUCT) return product_bilinear_grad(p, Lf, ldl, Rt, ldr, s, grad_ls, grad_os);
  if (p->compact) return compact_bilinear_grad(p, Lf, ldl, Rt, ldr, s, grad_ls, grad_os);
  if (p->kron) return kron_bilinear_grad(p, Lf, ldl, Rt, ldr, s, grad_ls, grad_os);
  if (p->deriv) return deriv_bilinear_grad(p, Lf, ldl, Rt, ldr, s, grad_ls, grad_os);
  if (p->add_M) return additive_bilinear_grad(p, Lf, ldl, Rt, ldr, s, grad_ls, grad_os);
  if (p->sm_Q) return spectral_bilinear_grad(p, Lf, ldl, Rt, ldr, s, grad_ls, grad_os);
  if (p->per_n) return periodic_bilinear_grad(p, Lf, ldl, Rt, ldr, s, grad_ls, grad_os);
  // before any launch: the SIMT derivative kernel is instantiated up to DP = 64
  GP_REQUIRE(p->backend == GP_BACKEND_SKI || p->DP <= 64, GP_E_SHAPE, "bilinear gradient supports d <= 64 (d=%d)", p->d);
  bool ard = p->ls.size() > 1;
  if (p->backend == GP_BACKEND_SKI) {
    // interpolated operator: everything happens on the grid (ski.cu); one sweep per 16 columns
    std::vector<double> tot(1 + p->d, 0.0);
    GP_CHECK(v16_chunks(p, Lf, ldl, Rt, ldr, s, p->row_count,
                        [&](const float* L16, const float* R16) { return ski_bilinear(p, L16, R16, tot.data()); }));
    *grad_os = tot[0];
    if (ard) {
      for (int c = 0; c < p->d; ++c) grad_ls[c] = p->outputscale * tot[1 + c] / (double)p->ls[c];
    } else {
      double sum = 0.0;
      for (int c = 0; c < p->d; ++c) sum += tot[1 + c];
      grad_ls[0] = p->outputscale * sum / (double)p->ls[0];
    }
    return GP_OK;
  }
  const bool rq = p->kind == GP_RQ;   // one more output: dF/dalpha
  const bool poly = p->kind == GP_POLY;   // [dF/dc] and dF/dS: no lengthscale (ARD does not apply)
  if (poly) ard = false;
  const int nls = ard ? p->d : 1;
  const int nout = 1 + nls + (rq ? 1 : 0);
  std::vector<double> total(nout, 0.0);
  if (p->tasks && (ard || p->backend != GP_BACKEND_TCGEN05)) {
    // K o B on the SIMT derivative kernel: one pass per column task with B folded into the rows (tasks.cu)
    GP_CHECK(v16_chunks(p, Lf, ldl, Rt, ldr, s, p->row_count,
                        [&](const float* L16, const float* R16) { return tasks_bilinear(p, L16, R16, ard, total); }));
  } else if (!ard && p->backend == GP_BACKEND_TCGEN05) {
    // scalar lengthscale on the tensor-core backend: sum_ij (L_i . R_j) f_ij = sum_i L_i . (F R)_i, i.e. two launches of
    // the fused K.V kernel (f = k, then f = g = l dk/dl through the derivative kinds) + a dot product with L; an RQ plan adds a
    // third (f = dk/dalpha).  ARD needs d weighted sums per pair and stays on the SIMT kernel.
    const int dot_blocks = (int)std::min<int64_t>(bilinear_blocks(p, p->n2), 2 * p->n_sm);
    GP_CHECK(bilinear_sweep(p, Lf, ldl, Rt, ldr, s, p->row_count, dot_blocks, nout, [&](const float* L16, const float* R16, double* gout) -> int {
      if (!p->tasks) GP_CHECK(pack_v_tiles(p, R16));
      for (int pass = 0; pass < nout; ++pass) {
        const int kind = pass == 0 ? p->kind : poly ? POLY_DC : !rq ? GP_DERIV + p->kind : pass == 1 ? RQ_DL : RQ_DA;
        // a multitask plan runs both passes on K o B (tasks.cu), combined into slot 0 in user row order
        GP_CHECK(p->tasks ? tasks_kmv_partials(p, R16, kind, nullptr) : kmv_tc_launch_kind(p, kind, nullptr));
        bilin_dot_kernel<<<dot_blocks, 256, 0, p->stream>>>(p->partial.as<float>(), p->nparts, p->row_count, p->rows_pad, L16, gout, nout,
                                                            pass);
        p->launches++;
      }
      GP_CUDA(cudaGetLastError());
      return GP_OK;
    }, total));
  } else {
    dim3 grid;
    int64_t cps;
    bilinear_split(p, p->n2, &grid, &cps);
    const BilinLaunch a{p->same ? p->Z2.as<float>() + p->row_begin * p->DP : p->Z1.as<float>(), p->Z2.as<float>(), p->n2, p->row_begin};
    GP_CHECK(bilinear_sweep(p, Lf, ldl, Rt, ldr, s, p->row_count, (int64_t)grid.x * grid.y, nout,
                            [&](const float* L16, const float* R16, double* gout) -> int {
                              return ard ? launch_bilinear_any<true>(p, a, L16, R16, gout, nout, grid, cps)
                                         : launch_bilinear_any<false>(p, a, L16, R16, gout, nout, grid, cps);
                            }, total));
  }
  // d/d outputscale of os*k = k ; d/dl: scalar -> sum w g / l ; ARD -> sum w g dz_c^2/s / l_c ; both times os
  *grad_os = total[0];
  if (poly)
    grad_ls[0] = p->outputscale * total[1];   // dF/dc = S sum_ij w_ij p a_ij^(p-1)
  else if (ard)
    for (int c = 0; c < p->d; ++c) grad_ls[c] = p->outputscale * total[1 + c] / (double)p->ls[c];
  else
    grad_ls[0] = p->outputscale * total[1] / (double)p->ls[0];
  if (rq) grad_ls[nls] = p->outputscale * total[1 + nls];   // [dF/dl | dF/dalpha]
  return GP_OK;
}
