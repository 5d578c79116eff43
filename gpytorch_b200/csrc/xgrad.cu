// xgrad.cu -- input gradients of kernel products and dense kernel blocks: dF/dX1, dF/dX2 for
//   product form  F = sum_ic G_ic (K V)_ic = sum_ij w_ij k_ij,  w_ij = G_i . V_j
//   dense form    F = sum_ij W_ij k_ij
// (the test-input gradient of an exact-GP posterior; the reference gets it from autograd through the slow branch of
// RBFKernel.forward / MaternKernel.forward, kernels/rbf_kernel.py:68-85, kernels/matern_kernel.py:86-107).
//
// Math, in the packed units of pack.cu (z = (x - mean) sqrt(C) / l, a = -|z_i - z_j|^2 / 2, k = s f(a)):
//   dk_ij/dx_ic = -s q_ij (z_ic - z_jc) sqrt(C) / l_c,   q = f'(a)  (hcov_from_arg, gp_common.cuh)
// so  DX1_i = -s sqrt(C)/l (.) sum_j w_ij q_ij (z_i - z_j)  and DX2_j the same with the roles swapped.  On a square plan both
// arguments are the same points: DX_i = -s sqrt(C)/l (.) sum_j (w_ij + w_ji) q_ij (z_i - z_j).  A pair at distance 0 contributes 0
// (the clamps of kernels/kernel.py:52-60 give the same; the stationary diagonal has zero input gradient).
// Polynomial plans (DESIGN 4.21) are not of the difference form: over the raw inputs (scale 1, no centring) a = x_i . x_j + c and
//   dk_ij/dx_i = s q_ij x_j,   q = p a^(p-1)  (hcov_from_arg<POLY_K>)
// so the kernel accumulates -w q x_j (the finish kernel's sign turns it back) and no pair is masked: on a square plan the diagonal
// pair adds (w_ii + w_ii) q_ii x_i, the derivative of k(x_i, x_i) = (|x_i|^2 + c)^p through both of its arguments.
//
// One kernel, two roles: a thread owns the row that receives the gradient ("own" side, Zo) and streams staged 64-row tiles of the
// other side (Zt), forming z_i - z_j by direct differences as kmv_simt_kernel does (no cancellation).  The reduced side is split
// over CTAs (blockIdx.y), each split writing partials [nsplit][rows][DP] that xgrad_finish_kernel sums in split order: no atomics,
// repeated calls are bit-identical, and m = 1 own row still spreads over every SM.
//   product form: w_ij = L_i . R_j over TW packed columns (L = G, R = V for DX1; L = V, R = G for DX2; L = [G | V], R = [V | G]
//                 on a square plan).  Columns are processed in chunks of TW = 8 (t <= 8, after doubling on a square plan) or
//                 TW = 32; every chunk evaluates each pair's q once and adds into the same partials.
//   dense form:   w_ij read from W with the role's strides (+ the transposed entry on a square plan).
// The cost is ~ n1 n2 (t + 3 DP) FMAs + 1 ex2 (+ 1 sqrt for Matern) per pair and chunk: far below a training K.V at Bayesian-
// optimisation sizes, so FP32 SIMT suffices (DESIGN.md section 4.10 says why no tensor-core path was built).
#include "gp_common.cuh"

namespace gp {

template <int KIND, int DP, int TW>
__global__ void __launch_bounds__(SIMT_TI)
xgrad_kernel(const float* __restrict__ Zo, const float* __restrict__ Zt, int64_t no, int64_t nt,
             const float* __restrict__ Lo, const float* __restrict__ Rt, const float* __restrict__ W, int64_t sr, int64_t sc,
             int sym, int64_t cols_per_split, int accumulate, float* __restrict__ partial, CovParam cp) {
  constexpr int TWS = TW > 0 ? TW : 1;
  __shared__ __align__(16) float zj[SIMT_TJ][DP];
  __shared__ __align__(16) float rj[SIMT_TJ][TWS];
  const int tid = threadIdx.x;
  const int64_t i = (int64_t)blockIdx.x * SIMT_TI + tid;
  const int split = blockIdx.y;
  const int64_t j_begin = (int64_t)split * cols_per_split;
  const int64_t j_end = min(nt, j_begin + cols_per_split);
  const bool rv = i < no;
  float zi[DP], li[TWS], acc[DP];
#pragma unroll
  for (int c = 0; c < DP; ++c) {
    zi[c] = rv ? Zo[i * DP + c] : 0.f;
    acc[c] = 0.f;
  }
#pragma unroll
  for (int c = 0; c < TWS; ++c) li[c] = (TW > 0 && rv) ? Lo[i * TWS + c] : 0.f;

  for (int64_t j0 = j_begin; j0 < j_end; j0 += SIMT_TJ) {
    const int nj = (int)min((int64_t)SIMT_TJ, j_end - j0);
    __syncthreads();
    for (int e = tid; e < SIMT_TJ * DP; e += SIMT_TI) (&zj[0][0])[e] = (e / DP < nj) ? Zt[j0 * DP + e] : 0.f;
    if (TW > 0)
      for (int e = tid; e < SIMT_TJ * TWS; e += SIMT_TI) (&rj[0][0])[e] = (e / TWS < nj) ? Rt[j0 * TWS + e] : 0.f;
    __syncthreads();
    if (!rv) continue;
#pragma unroll 2
    for (int jj = 0; jj < nj; ++jj) {
      float w = 0.f;
      if (TW > 0) {
#pragma unroll
        for (int c = 0; c < TWS; ++c) w = fmaf(li[c], rj[jj][c], w);
      } else {
        const int64_t j = j0 + jj;
        w = W[i * sr + j * sc];
        if (sym) w += W[j * sr + i * sc];
      }
      if constexpr (KIND == POLY_K) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < DP; ++c) s = fmaf(zi[c], zj[jj][c], s);
        const float wq = -w * hcov_from_arg<KIND>(s + cp.offset, cp);
#pragma unroll
        for (int c = 0; c < DP; ++c) acc[c] = fmaf(wq, zj[jj][c], acc[c]);
        continue;
      }
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        float df = zi[c] - zj[jj][c];
        s = fmaf(df, df, s);
      }
      const float a = -0.5f * s;
      // distance 0 (coinciding points, the diagonal of a square plan) contributes 0; a NaN argument fails the test too and is
      // reported through the plan's xbad flag by the finish kernel
      const float wq = (a < 0.f) ? w * hcov_from_arg<KIND>(a, cp) : 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) acc[c] = fmaf(wq, zi[c] - zj[jj][c], acc[c]);
    }
  }
  if (!rv) return;
  float4* dst = reinterpret_cast<float4*>(partial + ((int64_t)split * no + i) * DP);
#pragma unroll
  for (int q = 0; q < DP / 4; ++q) {
    float4 v = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
    if (accumulate) {
      const float4 o = dst[q];
      v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
    }
    dst[q] = v;
  }
}

// OUT[r][c] = -s scale_c sum_split partial[split][r][c]  (splits in order), NaN when the packed inputs held a non-finite value
__global__ void xgrad_finish_kernel(const float* __restrict__ partial, int nsplit, int64_t rows, int DP, int d,
                                    const float* __restrict__ scale, float os, const int* __restrict__ xbad,
                                    float* __restrict__ OUT, int64_t ld) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * d) return;
  const int64_t r = idx / d;
  const int c = (int)(idx % d);
  float s = 0.f;
  for (int sp = 0; sp < nsplit; ++sp) s += partial[((int64_t)sp * rows + r) * DP + c];
  float o = -os * scale[c] * s;
  if (*xbad) o = __int_as_float(0x7fc00000);
  OUT[r * ld + c] = o;
}

// out[r][c] = column c0 + c of the virtual block [A | B] (ta + tb columns; zero beyond)
__global__ void xgrad_pack_kernel(const float* __restrict__ A, int64_t lda, int ta, const float* __restrict__ B, int64_t ldb,
                                  int tb, int c0, int64_t n, int tw, float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * tw) return;
  const int64_t r = idx / tw;
  const int c = c0 + (int)(idx % tw);
  out[idx] = (c < ta) ? A[r * lda + c] : (c < ta + tb ? B[r * ldb + (c - ta)] : 0.f);
}

struct XgArgs {
  const float *Zo, *Zt;
  int64_t no, nt;
  const float *Lo, *Rt, *W;
  int64_t sr, sc;
  int sym, accumulate;
  int64_t cps;
  float* partial;
};

template <int KIND, int TW>
static int launch_xgrad(gp_plan* p, dim3 grid, const XgArgs& a) {
#define GP_XG_CASE(D)                                                                                                     \
  case D:                                                                                                                 \
    xgrad_kernel<KIND, D, TW><<<grid, SIMT_TI, 0, p->stream>>>(a.Zo, a.Zt, a.no, a.nt, a.Lo, a.Rt, a.W, a.sr, a.sc, a.sym, \
                                                               a.cps, a.accumulate, a.partial, cov_param(p));             \
    break;
  switch (p->DP) {
    GP_XG_CASE(4) GP_XG_CASE(8) GP_XG_CASE(12) GP_XG_CASE(16) GP_XG_CASE(24) GP_XG_CASE(32) GP_XG_CASE(48) GP_XG_CASE(64)
    default:
      set_error("input gradients support d <= 64 (DP=%d)", p->DP);
      return GP_E_SHAPE;
  }
#undef GP_XG_CASE
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

template <int TW>
static int launch_xgrad_kind(gp_plan* p, dim3 grid, const XgArgs& a) {
  switch (p->kind) {
    case GP_RBF: return launch_xgrad<GP_RBF, TW>(p, grid, a);
    case GP_MATERN12: return launch_xgrad<GP_MATERN12, TW>(p, grid, a);
    case GP_MATERN32: return launch_xgrad<GP_MATERN32, TW>(p, grid, a);
    case GP_MATERN52: return launch_xgrad<GP_MATERN52, TW>(p, grid, a);
    case GP_RQ: return launch_xgrad<RQ_K, TW>(p, grid, a);
    case GP_POLY: return launch_xgrad<POLY_K, TW>(p, grid, a);
  }
  set_error("bad kernel kind %d", p->kind);
  return GP_E_SHAPE;
}

// the right-hand factor of w_ij as a virtual block [A | B] of ta + tb columns (B only on a square plan)
struct XgSide {
  const float* A;
  int64_t lda;
  const float* B;
  int64_t ldb;
};

// one role: OUT [no][d] = gradient w.r.t. the own rows.  Product form when W == nullptr (L, R over tw = ta + tb columns), dense
// form otherwise (w_ij = W[i sr + j sc] (+ W[j sr + i sc] when sym)).
static int xgrad_role(gp_plan* p, const float* Zo, int64_t no, const float* Zt, int64_t nt, XgSide L, XgSide R, int ta, int tb,
                      const float* W, int64_t sr, int64_t sc, int sym, float* OUT, int64_t ld) {
  // splits of the reduced side: about 4 CTAs of 128 threads per SM, each split at least one 64-row tile
  const int64_t row_blocks = cdiv(no, SIMT_TI);
  const int64_t ntj = cdiv(nt, SIMT_TJ);
  int nsp = (int)std::min<int64_t>(ntj, std::max<int64_t>(1, cdiv(4 * (int64_t)p->n_sm, row_blocks)));
  const int64_t cps = cdiv(ntj, nsp) * SIMT_TJ;
  nsp = (int)cdiv(nt, cps);
  const dim3 grid((unsigned)row_blocks, (unsigned)nsp);
  GP_CHECK(p->misc.ensure(sizeof(float) * (size_t)nsp * no * p->DP));
  XgArgs a{Zo, Zt, no, nt, nullptr, nullptr, W, sr, sc, sym, 0, cps, p->misc.as<float>()};
  if (W) {
    GP_CHECK(launch_xgrad_kind<0>(p, grid, a));
  } else {
    const int tw_all = ta + tb;
    const int TW = tw_all <= 8 ? 8 : 32;
    GP_CHECK(p->misc2.ensure(sizeof(float) * no * TW));
    GP_CHECK(p->misc3.ensure(sizeof(float) * nt * TW));
    a.Lo = p->misc2.as<float>();
    a.Rt = p->misc3.as<float>();
    for (int c0 = 0; c0 < tw_all; c0 += TW) {
      xgrad_pack_kernel<<<(unsigned)cdiv(no * TW, 256), 256, 0, p->stream>>>(L.A, L.lda, ta, L.B, L.ldb, tb, c0, no, TW, p->misc2.as<float>());
      xgrad_pack_kernel<<<(unsigned)cdiv(nt * TW, 256), 256, 0, p->stream>>>(R.A, R.lda, ta, R.B, R.ldb, tb, c0, nt, TW, p->misc3.as<float>());
      p->launches += 2;
      a.accumulate = c0 > 0;
      GP_CHECK(TW == 8 ? launch_xgrad_kind<8>(p, grid, a) : launch_xgrad_kind<32>(p, grid, a));
    }
  }
  xgrad_finish_kernel<<<(unsigned)cdiv(no * p->d, 256), 256, 0, p->stream>>>(p->misc.as<float>(), nsp, no, p->DP, p->d,
                                                                             p->scale.as<float>(), p->outputscale, p->xbad, OUT, ld);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

static int xgrad_check(gp_plan* p, CallId call, float* DX1, int64_t ld1, float* DX2, int64_t ld2) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_CHECK(refuse_settings(p, call));
  const char* what = CALL_ROWS[call].name;
  GP_CHECK(refuse_compact(p, what));
  GP_REQUIRE(p->backend != GP_BACKEND_SUM, GP_E_SHAPE, "%s of a kernel sum: call it on every term", what);
  GP_REQUIRE(p->backend != GP_BACKEND_SKI, GP_E_SHAPE, "%s is not available on a SKI plan", what);
  GP_REQUIRE(p->row_begin == 0 && p->row_count == p->n1 && !(p->comm && p->comm->world > 1), GP_E_SHAPE,
             "%s is not available on a row-sharded plan", what);
  GP_REQUIRE(p->DP <= 64, GP_E_SHAPE, "%s supports d <= 64 (d=%d)", what, p->d);
  GP_REQUIRE(!(p->same && DX2), GP_E_SHAPE, "%s: on a square plan DX1 receives the total gradient and DX2 must be NULL", what);
  GP_REQUIRE((!DX1 || ld1 >= p->d) && (!DX2 || ld2 >= p->d), GP_E_SHAPE, "%s: output leading dimension below d=%d", what, p->d);
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_kmv_input_grad(gp_plan* p, const float* G, int64_t ldg, const float* V, int64_t ldv, int t, float* DX1,
                                 int64_t ld1, float* DX2, int64_t ld2) {
  GP_CHECK(xgrad_check(p, CALL_KMV_INPUT_GRAD, DX1, ld1, DX2, ld2));
  GP_REQUIRE(t >= 1 && ldg >= t && ldv >= t && G && V, GP_E_SHAPE, "gp_kmv_input_grad: bad shape t=%d ldg=%lld ldv=%lld", t,
             (long long)ldg, (long long)ldv);
  GP_CUDA(cudaSetDevice(p->device));
  const float* Z2 = p->Z2.as<float>();
  if (p->same) {   // both arguments move: w_ij + w_ji = [G_i | V_i] . [V_j | G_j]
    if (!DX1) return GP_OK;
    return xgrad_role(p, Z2, p->n2, Z2, p->n2, XgSide{G, ldg, V, ldv}, XgSide{V, ldv, G, ldg}, t, t, nullptr, 0, 0, 0, DX1, ld1);
  }
  const float* Z1 = p->Z1.as<float>();
  if (DX1) GP_CHECK(xgrad_role(p, Z1, p->n1, Z2, p->n2, XgSide{G, ldg, nullptr, 0}, XgSide{V, ldv, nullptr, 0}, t, 0, nullptr, 0, 0, 0, DX1, ld1));
  if (DX2) GP_CHECK(xgrad_role(p, Z2, p->n2, Z1, p->n1, XgSide{V, ldv, nullptr, 0}, XgSide{G, ldg, nullptr, 0}, t, 0, nullptr, 0, 0, 0, DX2, ld2));
  return GP_OK;
}

extern "C" int gp_kdense_input_grad(gp_plan* p, const float* W, int64_t ldw, float* DX1, int64_t ld1, float* DX2, int64_t ld2) {
  GP_CHECK(xgrad_check(p, CALL_KDENSE_INPUT_GRAD, DX1, ld1, DX2, ld2));
  GP_REQUIRE(W && ldw >= p->n2, GP_E_SHAPE, "gp_kdense_input_grad: bad W (ldw=%lld, n2=%lld)", (long long)ldw, (long long)p->n2);
  GP_CUDA(cudaSetDevice(p->device));
  const float* Z2 = p->Z2.as<float>();
  const XgSide none{nullptr, 0, nullptr, 0};
  if (p->same) {
    if (!DX1) return GP_OK;
    return xgrad_role(p, Z2, p->n2, Z2, p->n2, none, none, 0, 0, W, ldw, 1, 1, DX1, ld1);
  }
  const float* Z1 = p->Z1.as<float>();
  if (DX1) GP_CHECK(xgrad_role(p, Z1, p->n1, Z2, p->n2, none, none, 0, 0, W, ldw, 1, 0, DX1, ld1));
  if (DX2) GP_CHECK(xgrad_role(p, Z2, p->n2, Z1, p->n1, none, none, 0, 0, W, 1, ldw, 0, DX2, ld2));
  return GP_OK;
}
