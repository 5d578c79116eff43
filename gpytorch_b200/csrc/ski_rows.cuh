// ski_rows.cuh -- single entries of the SKI operator (ski.cu) from its separable form, without a product with the operator:
//   K_ski(i, j) = s prod_k a_k(i, j),   a_k(i, j) = sum_{a,b<4} w_ik[a] T_k[f_ik + a, f_jk + b] w_jk[b]
// (T_0 x ... x T_{d-1} is a Kronecker product and the cubic interpolation is a product of 1-D weights, so every kind -- the
// Materns included -- factorises per dimension).  f_ik / w_ik are the first node and the 4 weights of ski_interp_kernel in the
// caller's row order, T_k the G_k x G_k factor of ski_toeplitz_kernel.  A row i is evaluated through
//   u_k = T_k[:, f_ik : f_ik + 4] w_ik   (one G_k-vector per dimension, sum_k G_k <= 512 floats, staged in shared memory)
//   a_k(i, j) = sum_b w_jk[b] u_k[f_jk + b]                 (4 FMAs per dimension and entry)
// and the diagonal with the same operations in the same order, so that ski_diag_entry(i) == ski_entry(u of row i, i) bit for bit.
#pragma once
#include "gp_common.cuh"

namespace gp {

constexpr int SKI_U_MAX = 512;   // sum_k G_k: d <= 4, G_k <= 128

struct SkiRows {
  int d;
  int G[4];
  int toff[4];        // offset of T_k in T
  int uoff[4];        // offset of u_k in the staged vector
  int usum;           // sum_k G_k
  float os;           // outputscale
  const float* T;     // the factors back to back
  const int* first;   // [n][d]
  const float* wts;   // [n][d][4]
};

int ski_rows_args(const gp_plan* p, SkiRows* s);                                        // ski.cu
int ski_kdiag(gp_plan* p, float* OUT);                                                  // OUT[n] = diag K_ski
int ski_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);     // OUT[r] = K_ski[idx[r], :]
int ski_diag_sum(gp_plan* p, double* out);                                              // sum_i K_ski(i, i) in fp64

#if defined(__CUDACC__)
// The loops over the dimensions are unrolled to the compile-time bound 4 so that the fields of s are only ever indexed by constants
// (a run-time index would copy the struct to local memory).
// u[uoff[k] + g] = sum_a T_k[g][f_ik + a] w_ik[a] for every k and g; the caller synchronises the CTA before reading u
__device__ __forceinline__ void ski_stage_u(const SkiRows& s, int64_t i, float* u, int tid, int nthr) {
  for (int e = tid; e < s.usum; e += nthr) {
    int k = 0, G = s.G[0], toff = s.toff[0], uoff = s.uoff[0];
#pragma unroll
    for (int q = 1; q < 4; ++q)
      if (q < s.d && e >= s.uoff[q]) { k = q; G = s.G[q]; toff = s.toff[q]; uoff = s.uoff[q]; }
    const int g = e - uoff;
    const int f = s.first[i * s.d + k];
    const float4 w = *reinterpret_cast<const float4*>(s.wts + (i * s.d + k) * 4);
    const float* tr = s.T + toff + (int64_t)g * G + f;
    float v = tr[0] * w.x;
    v = fmaf(tr[1], w.y, v);
    v = fmaf(tr[2], w.z, v);
    v = fmaf(tr[3], w.w, v);
    u[e] = v;
  }
}

// K_ski(i, j) from the staged u of row i
__device__ __forceinline__ float ski_entry(const SkiRows& s, const float* u, int64_t j) {
  float v = s.os;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k >= s.d) break;
    const int f = s.first[j * s.d + k];
    const float4 w = *reinterpret_cast<const float4*>(s.wts + (j * s.d + k) * 4);
    const float* uk = u + s.uoff[k] + f;
    float a = uk[0] * w.x;
    a = fmaf(uk[1], w.y, a);
    a = fmaf(uk[2], w.z, a);
    a = fmaf(uk[3], w.w, a);
    v *= a;
  }
  return v;
}

// K_ski(i, i): u_k[f + b] = sum_a T_k[f + b][f + a] w[a] formed on the fly, 16 FMAs per dimension
__device__ __forceinline__ float ski_diag_entry(const SkiRows& s, int64_t i) {
  float v = s.os;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k >= s.d) break;
    const int f = s.first[i * s.d + k];
    const float4 w = *reinterpret_cast<const float4*>(s.wts + (i * s.d + k) * 4);
    const float wb[4] = {w.x, w.y, w.z, w.w};
    float a = 0.f;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const float* tr = s.T + s.toff[k] + (int64_t)(f + b) * s.G[k] + f;
      float ub = tr[0] * w.x;
      ub = fmaf(tr[1], w.y, ub);
      ub = fmaf(tr[2], w.z, ub);
      ub = fmaf(tr[3], w.w, ub);
      a = (b == 0) ? ub * wb[0] : fmaf(ub, wb[b], a);
    }
    v *= a;
  }
  return v;
}
#endif

}  // namespace gp
