// deriv_table.cuh -- the block table of the derivative-observation operator per covariance kind (deriv.cu, and the entry source
// of the pivoted Cholesky in pivchol.cu).  A table holds everything that depends on the kind: the per-pair coefficients from
// |dz|^2, the block entry E(a, b), the product's per-column and the gradient's per-pair update, and the constants of the packing,
// the diagonal and the kernels' shapes.  deriv.cu's kernels are one skeleton over a table; the derivations are in its header.
#pragma once

#include "gp_common.cuh"

namespace gp {

constexpr float DV_LN2 = 0.69314718f;   // 1 / log2 e: dz_c^2 / log2 e = D_c^2 / l_c^2
constexpr float M52_A = 1.6666666f;     // 5 / 3
constexpr float M52_B = 8.3333333f;     // 25 / 3
constexpr float M52_Q = 0.1f;           // q_c = dz_c^2 / 10

template <int KIND>
struct DerivTable;

template <>
struct DerivTable<GP_RBF> {
  static constexpr double PACK = 1.4426950408889634;   // z = (x - mean) sqrt(PACK) / l (pack.cu): w[c] = 1 / (sqrt(PACK) l_c)
  static constexpr double DIAG = 1.0;                  // the derivative rows' diagonal is DIAG s / l_a^2
  // columns per CTA: (DP + 1) x TW accumulators per thread in the product (DP = 8 with 8 columns takes 201 registers and ran
  // d = 5 at 6.7 TFLOP/s, with 4 columns 127 registers and 14.5 TFLOP/s, DESIGN 4.14); the gradient holds (DP + 1) x TW of L
  // instead, and half the columns keep it out of local memory
  static constexpr int kmv_tw(int DP) { return DP <= 4 ? 16 : 4; }
  static constexpr int grad_tw(int DP) { return DP <= 4 ? 8 : (DP <= 8 ? 4 : 2); }
  static constexpr int min_blocks(int) { return 0; }   // the product's __launch_bounds__: unbounded
  static constexpr int unroll(int) { return 2; }       // pairs per step of the product's loop

  struct Pair {
    float k;
    __device__ __forceinline__ Pair scaled(float os) const { return {os * k}; }
  };
  static __device__ __forceinline__ Pair pair(float s) { return {ex2_approx(fminf(-0.5f * s, 0.f))}; }

  // E(a, b) of one pair: [0, 0] = k, [0, b] = k u_b, [a, 0] = -k u_a, [a, b] = k (delta_ab / l_a^2 - u_a u_b)
  static __device__ __forceinline__ float entry(const Pair& p, int a, int b, float ua, float ub, const DerivHyp& hy) {
    const float k = p.k;
    return a == 0 ? (b == 0 ? k : k * ub) : (b == 0 ? -k * ua : k * ((a == b ? hy.il2[a - 1] : 0.f) - ua * ub));
  }

  // the coefficient of delta_ab / l_a^2 in E(a, b)
  static __device__ __forceinline__ float delta_coef(const Pair& p) { return p.k; }

  // acc += E V in column t of one staged point v, kl[c] = k / l_c^2:  h = v0 + sum_b u_b v^b,  acc0 += k h,
  // acc^a += k v^a / l_a^2 - u_a k h
  template <int DP, int TW>
  static __device__ __forceinline__ void kmv_column(const Pair& p, const float (&u)[DP], const float (&kl)[DP], const float (&v)[DP + 1][TW],
                                                    int t, float (&acc)[DP + 1][TW]) {
    const float k = p.k;
    float h = v[0][t];
#pragma unroll
    for (int c = 0; c < DP; ++c) h = fmaf(u[c], v[1 + c][t], h);
    const float kh = k * h;
    acc[0][t] += kh;
#pragma unroll
    for (int c = 0; c < DP; ++c) acc[1 + c][t] = fmaf(kl[c], v[1 + c][t], fmaf(-u[c], kh, acc[1 + c][t]));
  }

  // gk += k F ; gc[c] += k [ (dz_c^2 / log2 e) F - 2 u_c (g r_c - l_c h) - 2 il2_c l_c r_c ] over the TW columns of one pair
  template <int DP, int TW>
  static __device__ __forceinline__ void grad_pair(const Pair& p, const float (&u)[DP], const float (&dz2)[DP], const float (&li)[DP + 1][TW],
                                                   const float (&r)[DP + 1][TW], const DerivHyp& hy, float& gk, float (&gc)[DP]) {
    const float k = p.k;
    float fs = 0.f, hc[DP];
#pragma unroll
    for (int c = 0; c < DP; ++c) hc[c] = 0.f;
#pragma unroll
    for (int t = 0; t < TW; ++t) {
      float h = r[0][t], g = li[0][t], q = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        h = fmaf(u[c], r[1 + c][t], h);
        g = fmaf(-u[c], li[1 + c][t], g);
        q = fmaf(hy.il2[c] * li[1 + c][t], r[1 + c][t], q);
      }
      fs += fmaf(g, h, q);
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        const float lr = li[1 + c][t] * r[1 + c][t];
        hc[c] = fmaf(-2.f * u[c], fmaf(g, r[1 + c][t], -li[1 + c][t] * h), fmaf(-2.f * hy.il2[c], lr, hc[c]));
      }
    }
    gk = fmaf(k, fs, gk);
#pragma unroll
    for (int c = 0; c < DP; ++c) gc[c] = fmaf(k, fmaf(DV_LN2 * dz2[c], fs, hc[c]), gc[c]);
  }
};

template <>
struct DerivTable<GP_MATERN52> {
  static constexpr double PACK = 10.0;
  static constexpr double DIAG = 5.0 / 3.0;
  // columns per CTA: the RBF table's, the accumulators are the same (DP + 1) x TW
  static constexpr int kmv_tw(int DP) { return DP <= 4 ? 16 : 4; }
  static constexpr int grad_tw(int DP) { return DP <= 4 ? 8 : (DP <= 8 ? 4 : 2); }
  // CTAs per SM as the RBF product reaches them: DP = 4 three (168 registers; unbounded, ptxas takes 177 and two fit, 1.6x the
  // RBF time at d = 2 on H100), with one pair per loop step to stay free of spills; DP = 8 four (126); wider DP unbounded
  static constexpr int min_blocks(int DP) { return DP <= 4 ? 3 : (DP <= 8 ? 4 : 1); }
  static constexpr int unroll(int DP) { return DP <= 4 ? 1 : 2; }

  // rho, [0, 0] = k0 = (1 + rho + rho^2 / 3) e, A = (5/3) (1 + rho) e and B = (25/3) e with e = exp(-rho)
  struct Pair {
    float rho, k0, A, B;
    __device__ __forceinline__ Pair scaled(float os) const { return {rho, k0 * os, A * os, B * os}; }
  };
  static __device__ __forceinline__ Pair pair(float s) {
    const float r = sqrt_approx(0.5f * s);
    const float e = ex2_approx(-LOG2E * r);
    return {r, fmaf(fmaf(r, 0.33333334f, 1.f), r, 1.f) * e, M52_A * fmaf(r, e, e), M52_B * e};
  }

  // E(a, b) of one pair: [0, 0] = k0, [0, b] = A u_b, [a, 0] = -A u_a, [a, b] = A delta_ab / l_a^2 - B u_a u_b
  static __device__ __forceinline__ float entry(const Pair& p, int a, int b, float ua, float ub, const DerivHyp& hy) {
    return a == 0 ? (b == 0 ? p.k0 : p.A * ub) : (b == 0 ? -p.A * ua : fmaf(-p.B * ua, ub, a == b ? p.A * hy.il2[a - 1] : 0.f));
  }

  static __device__ __forceinline__ float delta_coef(const Pair& p) { return p.A; }

  // acc += E V in column t of one staged point v, al[c] = A / l_c^2:  h = sum_b u_b v^b,  acc0 += k0 v0 + A h,
  // acc^a += A v^a / l_a^2 - u_a (A v0 + B h)
  template <int DP, int TW>
  static __device__ __forceinline__ void kmv_column(const Pair& p, const float (&u)[DP], const float (&al)[DP], const float (&v)[DP + 1][TW],
                                                    int t, float (&acc)[DP + 1][TW]) {
    const float k0 = p.k0, A = p.A, B = p.B;
    const float v0 = v[0][t];
    float h = 0.f;
#pragma unroll
    for (int c = 0; c < DP; ++c) h = fmaf(u[c], v[1 + c][t], h);
    acc[0][t] = fmaf(k0, v0, fmaf(A, h, acc[0][t]));
    const float m = fmaf(A, v0, B * h);
#pragma unroll
    for (int c = 0; c < DP; ++c) acc[1 + c][t] = fmaf(al[c], v[1 + c][t], fmaf(-u[c], m, acc[1 + c][t]));
  }

  // gk += F ; gc[c] += l_c dF/dl_c / s over the TW columns of one pair, the expansion of deriv.cu's header
  template <int DP, int TW>
  static __device__ __forceinline__ void grad_pair(const Pair& p, const float (&u)[DP], const float (&dz2)[DP], const float (&li)[DP + 1][TW],
                                                   const float (&r)[DP + 1][TW], const DerivHyp& hy, float& gk, float (&gc)[DP]) {
    const float rho = p.rho, k0 = p.k0, A = p.A, B = p.B;
    const float q5 = rho > 0.f ? __fdividef(5.f * B, rho) : 0.f;   // 5 B / rho; every q_c is 0 where rho is
    const float m2A = -2.f * A, p2B = 2.f * B;
    float sp = 0.f, sa = 0.f, sb = 0.f;
#pragma unroll
    for (int t = 0; t < TW; ++t) {
      const float l0 = li[0][t], r0 = r[0][t];
      float h = 0.f, g = 0.f, q = 0.f;
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        h = fmaf(u[c], r[1 + c][t], h);
        g = fmaf(u[c], li[1 + c][t], g);
        q = fmaf(hy.il2[c] * li[1 + c][t], r[1 + c][t], q);
      }
      sp = fmaf(l0, r0, sp);
      sa += fmaf(l0, h, fmaf(-g, r0, q));
      sb = fmaf(g, h, sb);
#pragma unroll
      for (int c = 0; c < DP; ++c) {
        const float lc = li[1 + c][t], rc = r[1 + c][t];
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
};

// f(DerivTable<kind>{}) for a plan's kind (GP_RBF or GP_MATERN52): the one place a runtime kind selects its table
template <class F>
inline auto deriv_with_kind(int kind, F&& f) {
  return kind == GP_MATERN52 ? f(DerivTable<GP_MATERN52>{}) : f(DerivTable<GP_RBF>{});
}

}  // namespace gp
