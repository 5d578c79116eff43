// ski_rows.cuh -- single entries of the SKI operator (ski.cu) from its separable form, without a product with the operator:
//   K_ski(i, j) = s prod_k a_k(i, j),   a_k(i, j) = sum_{a,b<4} w_ik[a] T_k[f_ik + a, f_jk + b] w_jk[b]
// (T_0 x ... x T_{d-1} is a Kronecker product and the cubic interpolation is a product of 1-D weights, so every kind -- the
// Materns included -- factorises per dimension).  f_ik / w_ik are the first node and the 4 weights of ski_interp_kernel in the
// caller's row order; T_k is Toeplitz and read from its generating column, T_k[a][b] = t_k[|a - b|] (ski_toeplitz_col_kernel,
// bit-identical to the dense factor).  A row i is evaluated through
//   u_k = T_k[:, f_ik : f_ik + 4] w_ik   (one G_k-vector per dimension)
//   a_k(i, j) = sum_b w_jk[b] u_k[f_jk + b]                 (4 FMAs per dimension and entry)
// with u staged in shared memory when sum_k G_k <= SKI_U_MAX (`staged`); on larger grids the 4 entries u_k[f_jk + b] an entry needs
// are formed on the fly with the same operations in the same order, so both forms give the same bits.  The diagonal uses the same
// operations in the same order too, so that ski_diag_entry(i) == ski_entry(u of row i, i, i) bit for bit.
#pragma once
#include "gp_common.cuh"

namespace gp {

constexpr int SKI_U_MAX = 512;   // sum_k G_k staged in shared memory (every grid with G_k <= 128)

struct SkiRows {
  int d;
  int G[4];
  int coff[4];        // offset of t_k in tc
  int uoff[4];        // offset of u_k in the staged vector
  int usum;           // sum_k G_k
  int staged;         // usum <= SKI_U_MAX: the callers stage u (usum floats of shared memory); 0: entries form it on the fly
  float os;           // outputscale
  const float* tc;    // the generating columns back to back
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
// u_k[g] = sum_a T_k[g][f + a] w[a] = sum_a t_k[|g - f - a|] w[a], in a fixed order
__device__ __forceinline__ float ski_u_value(const float* t, int g, int f, float4 w) {
  float v = t[abs(g - f)] * w.x;
  v = fmaf(t[abs(g - f - 1)], w.y, v);
  v = fmaf(t[abs(g - f - 2)], w.z, v);
  v = fmaf(t[abs(g - f - 3)], w.w, v);
  return v;
}

// u[uoff[k] + g] = u_k[g] for every k and g (staged plans only; a no-op otherwise); the caller synchronises the CTA before reading u
__device__ __forceinline__ void ski_stage_u(const SkiRows& s, int64_t i, float* u, int tid, int nthr) {
  if (!s.staged) return;
  for (int e = tid; e < s.usum; e += nthr) {
    int k = 0, coff = s.coff[0], uoff = s.uoff[0];
#pragma unroll
    for (int q = 1; q < 4; ++q)
      if (q < s.d && e >= s.uoff[q]) { k = q; coff = s.coff[q]; uoff = s.uoff[q]; }
    const int f = s.first[i * s.d + k];
    const float4 w = *reinterpret_cast<const float4*>(s.wts + (i * s.d + k) * 4);
    u[e] = ski_u_value(s.tc + coff, e - uoff, f, w);
  }
}

// K_ski(i, j) from the staged u of row i (or from row i's interpolation data when the plan is not staged)
__device__ __forceinline__ float ski_entry(const SkiRows& s, const float* u, int64_t i, int64_t j) {
  float v = s.os;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (k >= s.d) break;
    const int f = s.first[j * s.d + k];
    const float4 w = *reinterpret_cast<const float4*>(s.wts + (j * s.d + k) * 4);
    float uk[4];
    if (s.staged) {
#pragma unroll
      for (int b = 0; b < 4; ++b) uk[b] = u[s.uoff[k] + f + b];
    } else {
      const int fi = s.first[i * s.d + k];
      const float4 wi = *reinterpret_cast<const float4*>(s.wts + (i * s.d + k) * 4);
#pragma unroll
      for (int b = 0; b < 4; ++b) uk[b] = ski_u_value(s.tc + s.coff[k], f + b, fi, wi);
    }
    float a = uk[0] * w.x;
    a = fmaf(uk[1], w.y, a);
    a = fmaf(uk[2], w.z, a);
    a = fmaf(uk[3], w.w, a);
    v *= a;
  }
  return v;
}

// K_ski(i, i): u_k[f + b] = sum_a t_k[|b - a|] w[a] formed on the fly, 16 FMAs per dimension
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
      const float ub = ski_u_value(s.tc + s.coff[k], f + b, f, w);
      a = (b == 0) ? ub * wb[0] : fmaf(ub, wb[b], a);
    }
    v *= a;
  }
  return v;
}
#endif

}  // namespace gp
