// simt_pass.cuh -- what the CUDA-core (SIMT) kernel families share: the fixed-order fp64 block reduction of the gradient kernels,
// row extraction, the cross diagonal and the constant square diagonal over per-family entry sources, the compile-time width
// dispatch, and the host sweep of a bilinear gradient over 16-column chunks.
//
// An entry source is a small struct passed by value: Z1, Z2 (packed rows), ld (their row stride), width() (host and device:
// the columns a row kernel stages in shared memory) and entry(za, zb, i, j) -> K(x1_i, x2_j) from two packed rows.  XBAD says
// whether the cross diagonal returns NaN for non-finite inputs (the plain kinds do not).
#pragma once
#include <algorithm>
#include <type_traits>
#include <vector>

#include "gp_common.cuh"

namespace gp {

// *dst = sum over the CTA's NT threads of v, in a fixed tree order through red (NT doubles of shared memory).  A caller that
// reduces several values in turn puts a __syncthreads() before each call: red is reused.
template <int NT>
__device__ __forceinline__ void block_sum_store(double* red, double v, double* dst) {
  const int tid = threadIdx.x;
  red[tid] = v;
  __syncthreads();
  for (int sft = NT / 2; sft > 0; sft >>= 1) {
    if (tid < sft) red[tid] += red[tid + sft];
    __syncthreads();
  }
  if (tid == 0) *dst = red[0];
}

// rows: OUT[r][j] = K(x1[idx[r]], x2[j]); grid (column blocks, m), dynamic shared memory of width() floats.  An out-of-range
// row index (CTA-uniform) gives a NaN row instead of an out-of-bounds read.  Non-finite inputs: every entry is NaN in the reference
// (mean-centring spreads it), while the covariance clamps would turn it into a constant
template <class Src>
__global__ void krows_kernel(const Src src, const int64_t* __restrict__ idx, int64_t n1_local, int64_t n2, float* __restrict__ OUT,
                             int64_t ldo, const int* __restrict__ xbad) {
  extern __shared__ float zi[];
  const int64_t r = blockIdx.y;
  const int64_t i = idx[r];
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 0 || i >= n1_local || *xbad) {
    if (j < n2) OUT[r * ldo + j] = __int_as_float(0x7fc00000);
    return;
  }
  for (int c = threadIdx.x; c < src.width(); c += blockDim.x) zi[c] = src.Z1[i * src.ld + c];
  __syncthreads();
  if (j >= n2) return;
  OUT[r * ldo + j] = src.entry(zi, src.Z2 + j * src.ld, i, j);
}

// diagonal of a cross-covariance K(x1, x2) (n1 == n2): OUT[i] = K(x1_i, x2_i)  (kernel(x1, x2, diag=True)); NaN for non-finite
// inputs when the source says so
template <class Src>
__global__ void kdiag_cross_kernel(const Src src, int64_t n, float* __restrict__ OUT, const int* __restrict__ xbad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if constexpr (Src::XBAD)
    OUT[i] = *xbad ? __int_as_float(0x7fc00000) : src.entry(src.Z1 + i * src.ld, src.Z2 + i * src.ld, i, i);
  else
    OUT[i] = src.entry(src.Z1 + i * src.ld, src.Z2 + i * src.ld, i, i);
}

// a constant diagonal: OUT[i] = v; with XB, NaN for non-finite inputs (kmv_simt.cu instantiates both)
template <bool XB>
__global__ void fill_kernel(float* __restrict__ OUT, int64_t n, float v, const int* __restrict__ xbad);

// ---- host ----------------------------------------------------------------------------------------------------------------------
// f(std::integral_constant<int, W>()) for the W of the list equal to w; false when none is (the caller reports the error)
template <int... W, class F>
bool with_width(int w, F&& f) {
  return ((w == W ? (f(std::integral_constant<int, W>()), true) : false) || ...);
}

template <class Src>
int launch_krows(gp_plan* p, const Src& src, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  krows_kernel<Src><<<dim3((unsigned)cdiv(p->n2, 256), (unsigned)m), 256, sizeof(float) * src.width(), p->stream>>>(
      src, idx, p->row_count, p->n2, OUT, ldo, p->xbad);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// the diagonal: on a square plan the constant *square_value when one is given, else the source's entries (x1_i, x2_i) (a cross
// plan needs n1 == n2).  NaN for non-finite inputs as Src::XBAD says
template <class Src>
int launch_kdiag(gp_plan* p, float* OUT, const float* square_value, const Src& src) {
  if (p->same && square_value) {
    fill_kernel<Src::XBAD><<<(unsigned)cdiv(p->row_count, 256), 256, 0, p->stream>>>(OUT, p->row_count, *square_value, p->xbad);
  } else {
    GP_REQUIRE(p->same || p->n1 == p->n2, GP_E_SHAPE,
               "diagonal of a %lld x %lld cross-covariance is undefined (kernel(x1, x2, diag=True) needs equal sizes)", (long long)p->n1,
               (long long)p->n2);
    const int64_t n = p->same ? p->row_count : p->n1;
    kdiag_cross_kernel<Src><<<(unsigned)cdiv(n, 256), 256, 0, p->stream>>>(src, n, OUT, p->xbad);
  }
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// f(L16, R16) for every chunk of 16 columns of the factors L [rows][s] and R [n2][s], converted to fp32 rows of 16 in misc2 / misc3
template <class F>
int v16_chunks(gp_plan* p, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr, int s, int64_t rows, F&& f) {
  GP_CHECK(p->misc2.ensure(sizeof(float) * rows * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * p->n2 * TP));
  for (int c0 = 0; c0 < s; c0 += TP) {
    const int tc = std::min(TP, s - c0);
    GP_CHECK(to_v16(p, Lf + c0, ldl, tc, rows, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, Rt + c0, ldr, tc, p->n2, p->misc3.as<float>()));
    GP_CHECK(f(p->misc2.as<float>(), p->misc3.as<float>()));
  }
  return GP_OK;
}

// total[o] = sum over the 16-column chunks of sum_b gout[b][o]: launch(L16, R16, gout) writes nblk rows of nout block partials
// per chunk, summed in fixed order on the device (NaN when an input is not finite) and accumulated on the host in chunk order
template <class F>
int bilinear_sweep(gp_plan* p, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr, int s, int64_t rows, int64_t nblk, int nout,
                   F&& launch, std::vector<double>& total) {
  GP_CHECK(p->misc.ensure(sizeof(double) * (nblk * nout + nout)));
  double* gout = p->misc.as<double>();
  double* gsum = gout + nblk * nout;
  total.assign(nout, 0.0);
  std::vector<double> h(nout);
  return v16_chunks(p, Lf, ldl, Rt, ldr, s, rows, [&](const float* L16, const float* R16) -> int {
    GP_CHECK(launch(L16, R16, gout));
    GP_CHECK(sum_partials_double(p, gout, nblk, nout, nout, gsum));
    GP_CUDA(cudaMemcpyAsync(h.data(), gsum, sizeof(double) * nout, cudaMemcpyDeviceToHost, p->stream));
    GP_CUDA(cudaStreamSynchronize(p->stream));
    for (int o = 0; o < nout; ++o) total[o] += h[o];
    return GP_OK;
  });
}

}  // namespace gp
