// kmv_tc.cu -- the fused kernel-matmul  out = K(X1,X2) V  on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces (reference, paths relative to the gpytorch package):
//   sq_dist GEMM + exp over N^2          kernels/kernel.py:26-49, functions/rbf_covariance.py:14-19
//   Matern poly*exp passes               functions/matern_covariance.py:21-47
//   dense K @ V inside linear_cg         lazy/lazy_evaluated_kernel_tensor.py:245-276 (chunked form)
// The N x N matrix K never exists in HBM: per 64 x 64 tile it lives in the registers of one warpgroup.
//
// One CTA per SM owns one work unit = (128-row tile of K) x (a contiguous range of 64-column tiles).  Per column tile j
// each consumer warpgroup computes, for its 64 rows:
//   GEMM1  S  = A_i . B_j^T     wgmma m64n64k8 tf32, both operands in shared memory (3xTF32 split operands packed by
//                               pack.cu so that S_ij = -0.5|z_i - z_j|^2 directly); S lands in 32 fp32 registers per thread
//   EPI    P  = cov(S)          ex2 / sqrt on the MUFU, in registers; P = P_hi + P_lo, both tf32 (P_hi: P with the low 13
//                               bits cleared, P_lo: the exact fp32 residual), each in its own 32 registers
//   GEMM2  O  = P_hi [V_hi;V_lo] (m64n32k8) + P_lo V_hi (m64n16k8), A operand from registers, B = V^T tiles in shared memory;
//          a fresh accumulator per tile, folded into fp32 registers after every tile
// P_hi / P_lo are the register A operand of GEMM2 in the layout of the GEMM1 accumulator.  That works because pack.cu stores
// the columns of every 8-column group of XB in the order 0 4 1 5 2 6 3 7: a thread's accumulator pair (2t, 2t+1) then holds
// the columns (t, t+4) the tf32 A fragment expects, and the V tiles keep their natural row order.
//
// Warp specialisation (384 threads):
//   warpgroup 0   producer: one thread issues the bulk copies (cp.async.bulk, mbarrier complete_tx) of the A tile and of
//                 the B / V tiles, pre-packed in HBM in the wgmma K-major no-swizzle layout, into an NS-deep shared-memory
//                 ring; it refills a stage once both consumers have released it.
//   warpgroups 1-2 consumers, rows [64 c, +64) of the tile for consumer c.  In its turn on the tensor core a consumer runs
//                 GEMM2 of tile j - 1 (two chains, one wait), then issues GEMM1 of tile j (one chain) and hands the tensor
//                 core to the other consumer (named barriers 1 and 2) before it waits for S and runs the MUFU-bound epilogue.
//                 So one consumer's epilogue overlaps the other's 21+ wgmmas.
// Every wgmma chain is issued back to back (no per-instruction wait) at <= 128 registers per thread: each chain starts
// with a write-only wgmma, so no accumulator is kept live across tiles; P and P_hi are stored in the A-fragment order, so
// P_lo is formed in P's registers (S's) once the P_hi chain has been issued.  ptxas checks the register need of the
// wgmma pipeline against the kernel's launch count (128), not against a warpgroup's setmaxnreg count: a consumer that
// keeps P_lo in 32 registers of its own, so that GEMM2 of tile j - 1 and GEMM1 of tile j go out as one batch with one
// wait, needs 153 registers; with a setmaxnreg 40 / 168 split under the 128 launch count ptxas serialises it (C7512) and
// it runs 1.7-2.3x slower than this kernel; compiled at 168 registers per thread it is no faster (H100: level with this
// kernel for RBF and C2 Matern-3/2, 2-10 % slower for the other Matern cases).
//
// The same pipeline (tc_pipeline) also runs the product of two tensor-core factors (product_tc_kernel, product.cu): a second
// GEMM1 operand with its own A tile and its own B tile per stage, a second GEMM1 chain in the same batch (S_b into hi, dead once
// GEMM2 of the previous tile has read P_hi, so the live set stays s, hi, o1, o2, acc) and the product covariance in the
// epilogue.  What a kernel computes per entry is its covariance source (TcOne, TcRq, TcPoly, TcProduct); the protocol exists once.
// A source also says whether the exact diagonal of a square plan is forced to a = 0 (the stationary kinds) or not (TcPoly, whose
// a_ii = |x_i|^2 + c comes out of GEMM1 like any other entry).
#include "gp_common.cuh"
#include "tc_ptx.cuh"

namespace gp {

using namespace ptx;

constexpr int TC_THREADS = 384;                     // producer warpgroup + 2 consumer warpgroups
constexpr int V_TF32_BYTES = 2 * TILE_J * TP * 4;   // [64/4][32 rows: V_hi(16) | V_lo(16)][4 tf32] = 8192
constexpr int V_TILE_BYTES = V_TILE_FLOATS * 4;                 // pitch of the packed V tiles in HBM (pack.cu)
static_assert(V_TILE_BYTES == V_TF32_BYTES + TILE_J * TP * 2, "packed V tile layout");
constexpr int MAX_NS = 12;
constexpr uint32_t TURN_BAR0 = 1;                   // named barriers 1, 2: consumer 0's / 1's turn on the tensor core

struct TcBars {
  uint64_t a_full;
  uint64_t b_full[MAX_NS];
  uint64_t b_empty[MAX_NS];   // 256 arrivals: every consumer thread, after its warpgroup's GEMM2 has read the stage
};

template <int KIND>
__device__ __forceinline__ float cov_tc(float a) {
  // RBF: k = 2^a with NO clamp of a at 0: a = -0.5|z_i - z_j|^2 can only come out > 0 through rounding for (near-)duplicate
  // points.  GEMM1 forms a = z_i.z_j + n_i + n_j, so that rounding is up to (1 + KP/4) 2^-21 (|z_i|^2 + |z_j|^2), a few 1e-6
  // for unit-cube data but more for inputs spanning many lengthscales (DESIGN 4.1); k then exceeds 1 by as much relative,
  // which the entry bound of tests/kmv_oracle.py allows for.  The exact diagonal is forced to a = 0 in diagonal tiles.
  return (KIND == GP_RBF) ? ex2_approx(a) : cov_from_arg<KIND>(a, CovParam{});
}

// Covariance sources of the pipeline.  TWO: a second GEMM1 operand (S_b into hi); pair(a, b): the covariance of one entry from
// its GEMM1 results (b = S_b, read only when TWO); EXACT_DIAG: a square plan's diagonal entries are evaluated at a = 0.
template <int KIND>
struct TcOne {   // one operand of kind KIND (GP_DERIV + kind: l dk/dl for gp_bilinear_grad)
  static constexpr bool TWO = false;
  static constexpr bool EXACT_DIAG = true;
  __device__ __forceinline__ float pair(float a, float) const { return cov_tc<KIND>(a); }
};
template <int KIND>
struct TcRq {    // the RQ kernel: KIND = RQ_K (k), RQ_DL (l dk/dl) or RQ_DA (dk/dalpha); lg2 + ex2 per entry
  static constexpr bool TWO = false;
  static constexpr bool EXACT_DIAG = true;
  CovParam cp;
  __device__ __forceinline__ float pair(float a, float) const { return cov_from_arg<KIND>(a, cp); }
};
template <int KIND>
struct TcPoly {  // the polynomial kernel: KIND = POLY_K (a^p) or POLY_DC (p a^(p-1)), a = x_i.x_j + c from GEMM1; FMA pipe only
  static constexpr bool TWO = false;
  static constexpr bool EXACT_DIAG = false;
  CovParam cp;
  __device__ __forceinline__ float pair(float a, float) const { return cov_from_arg<KIND>(a, cp); }
};
template <bool RBF_A, bool RBF_B>
struct TcProduct {   // k_a k_b = poly_a poly_b ex2(e_a + e_b): one ex2 per entry (cov_poly_exp, gp_common.cuh)
  static constexpr bool TWO = true;
  static constexpr bool EXACT_DIAG = true;
  CovPoly ca, cb;
  __device__ __forceinline__ float pair(float a, float b) const {
    float pa, ea, pb, eb;
    cov_poly_exp<false>(RBF_A, ca, a, &pa, &ea);
    cov_poly_exp<false>(RBF_B, cb, b, &pb, &eb);
    return (pa * pb) * ex2_approx(ea + eb);
  }
};

// The pipeline of both entries.  KPa: width of the first operand (XA, XB); with Src::TWO the second (XAb, XBb, KPb) has its own A
// tile beside the first and its own B tile in every stage: [A_a | A_b | NS x (B_a | B_b | V) | bars], else [A | NS x (B | V) | bars].
template <class Src>
__device__ __forceinline__ void tc_pipeline(const Src src, const float* __restrict__ XA, const float* __restrict__ XAb,
                                            const float* __restrict__ XB, const float* __restrict__ XBb, const float* __restrict__ Vt,
                                            float* __restrict__ partial, int KPa, int KPb, int NS, int64_t ntile_j,
                                            int64_t tiles_per_split, int64_t rows_pad, int same, int64_t row_begin,
                                            const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;  // CTA-uniform, before any barrier exists
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t it = blockIdx.x;
  const int split = blockIdx.y;
  const int64_t jt0 = (int64_t)split * tiles_per_split;
  const int64_t jt1 = min(ntile_j, jt0 + tiles_per_split);
  const int T = (int)max((int64_t)0, jt1 - jt0);

  const uint32_t aa_bytes = (uint32_t)KPa * TILE_I * 4, ab_bytes = Src::TWO ? (uint32_t)KPb * TILE_I * 4 : 0u;
  const uint32_t ba_bytes = (uint32_t)KPa * TILE_J * 4, bb_bytes = Src::TWO ? (uint32_t)KPb * TILE_J * 4 : 0u;
  const uint32_t b_bytes = ba_bytes + bb_bytes;
  const uint32_t stage_bytes = b_bytes + V_TF32_BYTES;
  uint8_t* sA = smem;
  uint8_t* sStage = smem + aa_bytes + ab_bytes;
  TcBars* bars = reinterpret_cast<TcBars*>(sStage + (size_t)NS * stage_bytes);

  if (threadIdx.x == 0) {
    mbar_init(smem_u32(&bars->a_full), 1);
    for (int s = 0; s < MAX_NS; ++s) {
      mbar_init(smem_u32(&bars->b_full[s]), 1);
      mbar_init(smem_u32(&bars->b_empty[s]), 256);
    }
    fence_mbar_init();
  }
  __syncthreads();   // the last CTA-wide barrier: the roles below never meet all 384 threads again
  if (T == 0) return;

  if (warp < 4) {
    // ---- producer ----
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(smem_u32(&bars->a_full), aa_bytes + ab_bytes);
      bulk_g2s(smem_u32(sA), XA + it * (int64_t)TILE_I * KPa, aa_bytes, smem_u32(&bars->a_full));
      if constexpr (Src::TWO) bulk_g2s(smem_u32(sA + aa_bytes), XAb + it * (int64_t)TILE_I * KPb, ab_bytes, smem_u32(&bars->a_full));
      int s = 0;
      uint32_t par = 0;   // phase of b_empty[s] the consumers complete when they release the stage's previous tile
      for (int u = 0; u < T; ++u) {
        if (u >= NS) mbar_wait(smem_u32(&bars->b_empty[s]), par);
        const uint32_t full = smem_u32(&bars->b_full[s]);
        uint8_t* st = sStage + (size_t)s * stage_bytes;
        const int64_t jt = jt0 + u;
        mbar_arrive_expect_tx(full, stage_bytes);
        bulk_g2s(smem_u32(st), XB + jt * (int64_t)TILE_J * KPa, ba_bytes, full);
        if constexpr (Src::TWO) bulk_g2s(smem_u32(st + ba_bytes), XBb + jt * (int64_t)TILE_J * KPb, bb_bytes, full);
        // only the tf32 part of the packed V tile: the products run in tf32 (P_lo is multiplied by V_hi)
        bulk_g2s(smem_u32(st + b_bytes), reinterpret_cast<const uint8_t*>(Vt) + jt * (int64_t)V_TILE_BYTES, V_TF32_BYTES, full);
        if (++s == NS) {
          s = 0;
          if (u >= NS) par ^= 1;
        }
      }
    }
    return;
  }

  // ---- consumers ----
  // accumulator fragment of wgmma m64nN (fp32): register i of thread (warp wq of the warpgroup, lane = 4 g + t) holds row
  // 16 wq + g + 8 ((i >> 1) & 1) and column position 8 (i >> 2) + 2 t + (i & 1); with the XB column order of pack.cu the
  // position 2 t + e of an 8-column group is column t + 4 e of the tile.
  const int wg = (warp >> 2) - 1;   // consumer 0 / 1
  const int wq = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  const int64_t rloc0 = it * TILE_I + wg * 64 + wq * 16 + g;   // local (padded) rows rloc0 and rloc0 + 8 of this thread
  const int64_t diag_off = row_begin + it * TILE_I + wg * 64 - jt0 * TILE_J;   // first global row of this warpgroup - jt0 * 64
  const uint64_t aa_desc0 = gmma_desc(smem_u32(sA) + (uint32_t)wg * 8 * 128, TILE_I * 16, 128);
  const uint64_t ab_desc0 = gmma_desc(smem_u32(sA + aa_bytes) + (uint32_t)wg * 8 * 128, TILE_I * 16, 128);   // Src::TWO only
  constexpr uint64_t A_KSTEP = (2 * TILE_I * 16) >> 4, B_KSTEP = (2 * TILE_J * 16) >> 4, V_KSTEP = (2 * 2 * TP * 16) >> 4;
  const int ksteps_a = KPa / 8, ksteps_b = KPb / 8;
  const uint32_t my_turn = TURN_BAR0 + wg, other_turn = TURN_BAR0 + (wg ^ 1);

  float acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = 0.f;
  float s[32], o1[16], o2[8];   // s: S (S_a) of the current tile, then P, then P_lo
  float hi[32];                 // P_hi (tf32 bit pattern); with Src::TWO first S_b of the current tile, dead once GEMM2 has read P_hi

  auto stage_addr = [&](int sb) { return smem_u32(sStage + (size_t)sb * stage_bytes); };
  // GEMM1 of the tile in stage sb into s; with Src::TWO a second chain, S_b into hi, in the same batch
  auto issue_gemm1 = [&](int sb) {
    const uint64_t ba_desc0 = gmma_desc(stage_addr(sb), TILE_J * 16, 128);
    const uint64_t bb_desc0 = gmma_desc(stage_addr(sb) + ba_bytes, TILE_J * 16, 128);
    wgmma_m64n64k8_ss_first(s, aa_desc0, ba_desc0);
#pragma unroll 1
    for (int ks = 1; ks < ksteps_a; ++ks) wgmma_m64n64k8_ss(s, aa_desc0 + ks * A_KSTEP, ba_desc0 + ks * B_KSTEP, 1u);
    if constexpr (Src::TWO) {
      wgmma_m64n64k8_ss_first(hi, ab_desc0, bb_desc0);
#pragma unroll 1
      for (int ks = 1; ks < ksteps_b; ++ks) wgmma_m64n64k8_ss(hi, ab_desc0 + ks * A_KSTEP, bb_desc0 + ks * B_KSTEP, 1u);
    }
  };
  // GEMM2 of the tile in stage sb into a fresh o1 / o2, as two chains: P_hi [V_hi;V_lo] (P_hi in hi), then P_lo V_hi with
  // P_lo = P - P_hi formed in place of P (in s) once the first chain has read P_hi.  Two chains keep P, P_hi, P_lo and O
  // within the register budget of 384-thread CTAs.
  auto run_gemm2 = [&](int sb) {
    const uint64_t v_desc0 = gmma_desc(stage_addr(sb) + b_bytes, 2 * TP * 16, 128);   // rows 0-15 V_hi, 16-31 V_lo
    fence_regs(o1);
    wgmma_fence();
    wgmma_m64n32k8_rs_first(o1, __float_as_uint(hi[0]), __float_as_uint(hi[1]), __float_as_uint(hi[2]), __float_as_uint(hi[3]), v_desc0);
#pragma unroll
    for (int jb = 1; jb < TILE_J / 8; ++jb)
      wgmma_m64n32k8_rs(o1, __float_as_uint(hi[4 * jb]), __float_as_uint(hi[4 * jb + 1]), __float_as_uint(hi[4 * jb + 2]),
                        __float_as_uint(hi[4 * jb + 3]), v_desc0 + jb * V_KSTEP, 1u);
    wgmma_commit();
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = s[i] - hi[i];
    fence_regs(s);
    fence_regs(o2);
    wgmma_fence();
    wgmma_m64n16k8_rs_first(o2, __float_as_uint(s[0]), __float_as_uint(s[1]), __float_as_uint(s[2]), __float_as_uint(s[3]), v_desc0);
#pragma unroll
    for (int jb = 1; jb < TILE_J / 8; ++jb)
      wgmma_m64n16k8_rs(o2, __float_as_uint(s[4 * jb]), __float_as_uint(s[4 * jb + 1]), __float_as_uint(s[4 * jb + 2]),
                        __float_as_uint(s[4 * jb + 3]), v_desc0 + jb * V_KSTEP, 1u);
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(s);
    if constexpr (Src::TWO) fence_regs(hi);
    fence_regs(o1);
    fence_regs(o2);
  };
  // covariance P of tile u (S in s, S_b in hi) and its tf32 part P_hi (the fp32 residual P_lo is formed in run_gemm2)
  auto epilogue = [&](int u) {
    const int64_t d = diag_off - (int64_t)u * TILE_J;   // first row of this warpgroup - first column of the tile
    if (Src::EXACT_DIAG && same && d > -64 && d < TILE_J) {
      const int dr = (int)d + wq * 16 + g - t;           // global row of register 0 - global column of register 0
#pragma unroll
      for (int i = 0; i < 32; ++i)   // a_ii = 0 exactly (kernel.py:44-45 fills the diagonal with 0), for both operands
        if (dr + 8 * ((i >> 1) & 1) - 8 * (i >> 2) - 4 * (i & 1) == 0) {
          s[i] = 0.f;
          if constexpr (Src::TWO) hi[i] = 0.f;
        }
    }
    // P goes back into s, P_hi into hi, both in the tf32 A-fragment order (registers 4 jb + {0, 2, 1, 3} of the accumulator)
#pragma unroll
    for (int jb = 0; jb < TILE_J / 8; ++jb) {
      float pv[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) pv[k] = src.pair(s[4 * jb + k], hi[4 * jb + k]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        s[4 * jb + k] = pv[(k >> 1) | ((k & 1) << 1)];   // k = 0 1 2 3 <- accumulator register 0 2 1 3
        hi[4 * jb + k] = __uint_as_float(__float_as_uint(s[4 * jb + k]) & 0xFFFFE000u);
      }
    }
  };
  // O of the previous tile (stage sb): release the stage, fold into acc.  Long accumulation chains inside the tensor core
  // drift, hence a fresh GEMM2 accumulator per tile.
  auto fold = [&](int sb) {
    mbar_arrive(smem_u32(&bars->b_empty[sb]));   // this thread's share of the stage has been read
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] += o1[c] + o1[c + 8] + o2[c];
  };
  auto issue_gemm1_batch = [&](int sb) {
    fence_regs(s);
    if constexpr (Src::TWO) fence_regs(hi);
    wgmma_fence();
    issue_gemm1(sb);
    wgmma_commit();
  };
  auto wait_gemm1 = [&]() {
    wgmma_wait_all();
    fence_regs(s);
    if constexpr (Src::TWO) fence_regs(hi);
  };

  mbar_wait(smem_u32(&bars->a_full), 0);
  if (wg == 1) named_bar_arrive(TURN_BAR0, 256);   // consumer 0 takes the first turn

  // turn 0: GEMM1 of tile 0
  mbar_wait(smem_u32(&bars->b_full[0]), 0);
  named_bar_sync(my_turn, 256);
  issue_gemm1_batch(0);
  named_bar_arrive(other_turn, 256);
  wait_gemm1();
  epilogue(0);

  // turns 1 .. T - 1: GEMM2 of tile u - 1, then GEMM1 of tile u
  int sb_prev = 0, sb = 1;   // NS >= 2 (launch_tc_kind, product_tc_launch)
  uint32_t par = 0;
#pragma unroll 1
  for (int u = 1; u < T; ++u) {
    mbar_wait(smem_u32(&bars->b_full[sb]), par);
    named_bar_sync(my_turn, 256);
    run_gemm2(sb_prev);
    fold(sb_prev);
    issue_gemm1_batch(sb);
    named_bar_arrive(other_turn, 256);
    wait_gemm1();
    epilogue(u);
    sb_prev = sb;
    if (++sb == NS) { sb = 0; par ^= 1; }
  }

  // last turn: GEMM2 of tile T - 1; consumer 1 has no one to hand the tensor core to
  named_bar_sync(my_turn, 256);
  run_gemm2(sb_prev);
  if (wg == 0) named_bar_arrive(other_turn, 256);
  fold(sb_prev);

  // columns 2 t, 2 t + 1 (c even) and 8 + 2 t, 9 + 2 t of rows rloc0 (c & 2 == 0) and rloc0 + 8
#pragma unroll
  for (int c = 0; c < 8; c += 2) {
    const int64_t row = rloc0 + 8 * ((c >> 1) & 1);
    float2* dst = reinterpret_cast<float2*>(partial + ((int64_t)split * rows_pad + row) * TP + 8 * (c >> 2) + 2 * t);
    *dst = make_float2(acc[c], acc[c + 1]);
  }
}

template <int KIND>
__global__ void __maxnreg__(128)
kmv_tc_kernel(const float* __restrict__ XA, const float* __restrict__ XB, const float* __restrict__ Vt,
              float* __restrict__ partial, int KP, int NS, int64_t ntile_j, int64_t tiles_per_split,
              int64_t rows_pad, int same, int64_t row_begin, const int* __restrict__ done_flag) {
  tc_pipeline(TcOne<KIND>{}, XA, nullptr, XB, nullptr, Vt, partial, KP, 0, NS, ntile_j, tiles_per_split, rows_pad, same, row_begin,
              done_flag);
}

// the RQ kernel (CODE = RQ_K, RQ_DL or RQ_DA) with its per-plan alpha
template <int CODE>
__global__ void __maxnreg__(128)
rq_tc_kernel(const float* __restrict__ XA, const float* __restrict__ XB, const float* __restrict__ Vt,
             float* __restrict__ partial, int KP, int NS, int64_t ntile_j, int64_t tiles_per_split,
             int64_t rows_pad, int same, int64_t row_begin, const int* __restrict__ done_flag, CovParam cp) {
  tc_pipeline(TcRq<CODE>{cp}, XA, nullptr, XB, nullptr, Vt, partial, KP, 0, NS, ntile_j, tiles_per_split, rows_pad, same, row_begin,
              done_flag);
}

// the polynomial kernel (CODE = POLY_K or POLY_DC) with its per-plan power
template <int CODE>
__global__ void __maxnreg__(128)
poly_tc_kernel(const float* __restrict__ XA, const float* __restrict__ XB, const float* __restrict__ Vt,
               float* __restrict__ partial, int KP, int NS, int64_t ntile_j, int64_t tiles_per_split,
               int64_t rows_pad, int same, int64_t row_begin, const int* __restrict__ done_flag, CovParam cp) {
  tc_pipeline(TcPoly<CODE>{cp}, XA, nullptr, XB, nullptr, Vt, partial, KP, 0, NS, ntile_j, tiles_per_split, rows_pad, same,
              row_begin, done_flag);
}

// two factors of a kernel product (product.cu), each from its own packed tiles XA_f / XB_f of width KP_f
template <bool RBF_A, bool RBF_B>
__global__ void __maxnreg__(128)
product_tc_kernel(const float* __restrict__ XAa, const float* __restrict__ XAb, const float* __restrict__ XBa,
                  const float* __restrict__ XBb, const float* __restrict__ Vt, float* __restrict__ partial, int KPa, int KPb, int NS,
                  int64_t ntile_j, int64_t tiles_per_split, int64_t rows_pad, int same, int64_t row_begin, CovPoly ca, CovPoly cb,
                  const int* __restrict__ done_flag) {
  tc_pipeline(TcProduct<RBF_A, RBF_B>{ca, cb}, XAa, XAb, XBa, XBb, Vt, partial, KPa, KPb, NS, ntile_j, tiles_per_split, rows_pad, same,
              row_begin, done_flag);
}

static int tc_smem_bytes(int KP, int* ns_out) {
  const int a_bytes = KP * TILE_I * 4;
  const int stage = KP * TILE_J * 4 + V_TF32_BYTES;
  // one CTA per SM: the whole 227 KB opt-in shared memory
  const int budget = 226 * 1024 - a_bytes - (int)sizeof(TcBars);
  int ns = budget / stage;
  if (ns > MAX_NS) ns = MAX_NS;
  *ns_out = ns;
  return a_bytes + ns * stage + (int)sizeof(TcBars);
}

struct TcLaunch {
  const float* XA;
  const float* XB;
  const float* Vt;
  float* partial;
  int64_t ntile_j, tiles_per_split, row_begin;
  int nsplit;
};

template <int KIND>
static int launch_tc_kind(gp_plan* p, const TcLaunch& a, const int* done_flag) {
  int ns = 0;
  int smem_bytes = tc_smem_bytes(p->KP, &ns);
  GP_REQUIRE(ns >= 2, GP_E_SHAPE, "tensor-core path: smem ring too small for KP=%d", p->KP);
  dim3 grid((unsigned)p->ntile_i, (unsigned)a.nsplit);
  if constexpr (is_poly_code(KIND)) {
    GP_CHECK(opt_in_smem<poly_tc_kernel<KIND>>(p->device, 227 * 1024));
    poly_tc_kernel<KIND><<<grid, TC_THREADS, smem_bytes, p->stream>>>(
        a.XA, a.XB, a.Vt, a.partial, p->KP, ns, a.ntile_j, a.tiles_per_split, p->rows_pad, p->same ? 1 : 0, a.row_begin, done_flag,
        cov_param(p));
  } else if constexpr (is_rq_code(KIND)) {
    GP_CHECK(opt_in_smem<rq_tc_kernel<KIND>>(p->device, 227 * 1024));
    rq_tc_kernel<KIND><<<grid, TC_THREADS, smem_bytes, p->stream>>>(
        a.XA, a.XB, a.Vt, a.partial, p->KP, ns, a.ntile_j, a.tiles_per_split, p->rows_pad, p->same ? 1 : 0, a.row_begin, done_flag,
        cov_param(p));
  } else {
    GP_CHECK(opt_in_smem<kmv_tc_kernel<KIND>>(p->device, 227 * 1024));
    kmv_tc_kernel<KIND><<<grid, TC_THREADS, smem_bytes, p->stream>>>(
        a.XA, a.XB, a.Vt, a.partial, p->KP, ns, a.ntile_j, a.tiles_per_split, p->rows_pad, p->same ? 1 : 0, a.row_begin, done_flag);
  }
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

static int launch_tc_any(gp_plan* p, int kind, const TcLaunch& a, const int* done_flag) {
  if (p->kind == GP_RQ) {   // the plan's kind first: GP_RQ is the number of GP_DERIV + GP_RBF
    switch (rq_code(p, kind)) {
      case RQ_K: return launch_tc_kind<RQ_K>(p, a, done_flag);
      case RQ_DL: return launch_tc_kind<RQ_DL>(p, a, done_flag);
      case RQ_DA: return launch_tc_kind<RQ_DA>(p, a, done_flag);
    }
    set_error("bad kernel code %d for a rational quadratic plan", kind);
    return GP_E_SHAPE;
  }
  if (p->kind == GP_POLY) {   // GP_POLY is the number of GP_DERIV + GP_MATERN12
    switch (rq_code(p, kind)) {
      case POLY_K: return launch_tc_kind<POLY_K>(p, a, done_flag);
      case POLY_DC: return launch_tc_kind<POLY_DC>(p, a, done_flag);
    }
    set_error("bad kernel code %d for a polynomial plan", kind);
    return GP_E_SHAPE;
  }
  switch (kind) {
    case GP_RBF: return launch_tc_kind<GP_RBF>(p, a, done_flag);
    case GP_MATERN12: return launch_tc_kind<GP_MATERN12>(p, a, done_flag);
    case GP_MATERN32: return launch_tc_kind<GP_MATERN32>(p, a, done_flag);
    case GP_MATERN52: return launch_tc_kind<GP_MATERN52>(p, a, done_flag);
    case GP_DERIV + GP_RBF: return launch_tc_kind<GP_DERIV + GP_RBF>(p, a, done_flag);
    case GP_DERIV + GP_MATERN12: return launch_tc_kind<GP_DERIV + GP_MATERN12>(p, a, done_flag);
    case GP_DERIV + GP_MATERN32: return launch_tc_kind<GP_DERIV + GP_MATERN32>(p, a, done_flag);
    case GP_DERIV + GP_MATERN52: return launch_tc_kind<GP_DERIV + GP_MATERN52>(p, a, done_flag);
  }
  set_error("bad kernel kind %d", kind);
  return GP_E_SHAPE;
}

int kmv_tc_launch_kind(gp_plan* p, int kind, const int* done_flag) {
  const TcLaunch a{p->XA.as<float>(), p->XB.as<float>(), vtiles_ptr(p), partial_ptr(p), p->ntile_j, p->tiles_per_split,
                   p->row_begin, p->nsplit};
  return launch_tc_any(p, kind, a, done_flag);
}

int kmv_tc_launch_cols(gp_plan* p, int kind, const float* XA, const float* XB, const float* Vt, float* partial, int64_t ntile_j,
                       int64_t tiles_per_split, int nsplit, int64_t diag_row_begin, const int* done_flag) {
  const TcLaunch a{XA, XB, Vt, partial, ntile_j, tiles_per_split, diag_row_begin, nsplit};
  return launch_tc_any(p, kind, a, done_flag);
}

// p->KP = KP_a + KP_b (product_pack), so the ring holds stages of both B tiles beside both A tiles
template <bool RA, bool RB>
static int launch_product_tc_kind(gp_plan* p, const int* done_flag) {
  const gp_plan* a = p->factors[0];
  const gp_plan* b = p->factors[1];
  int ns = 0;
  int smem_bytes = tc_smem_bytes(p->KP, &ns);
  GP_REQUIRE(ns >= 2, GP_E_SHAPE, "kernel product: smem ring too small for KP=%d", p->KP);
  GP_CHECK((opt_in_smem<product_tc_kernel<RA, RB>>(p->device, 227 * 1024)));
  dim3 grid((unsigned)p->ntile_i, (unsigned)p->nsplit);
  product_tc_kernel<RA, RB><<<grid, TC_THREADS, smem_bytes, p->stream>>>(
      a->XA.as<float>(), b->XA.as<float>(), a->XB.as<float>(), b->XB.as<float>(), p->Vtiles.as<float>(), p->partial.as<float>(), a->KP,
      b->KP, ns, p->ntile_j, p->tiles_per_split, p->rows_pad, p->same ? 1 : 0, p->row_begin, cov_poly_of(a->kind), cov_poly_of(b->kind),
      done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int product_tc_launch(gp_plan* p, const int* done_flag) {
  const bool ra = p->factors[0]->kind == GP_RBF, rb = p->factors[1]->kind == GP_RBF;
  return ra ? (rb ? launch_product_tc_kind<true, true>(p, done_flag) : launch_product_tc_kind<true, false>(p, done_flag))
            : (rb ? launch_product_tc_kind<false, true>(p, done_flag) : launch_product_tc_kind<false, false>(p, done_flag));
}
int kmv_tc_launch(gp_plan* p, const int* done_flag) {
  if (p->backend == GP_BACKEND_SUM) return sum_kmv_launch(p, nullptr, done_flag);   // all terms on tensor cores (plan_is_tc)
  if (p->backend == GP_BACKEND_PRODUCT) return product_kmv_launch(p, nullptr, done_flag);   // two tensor-core factors (plan_is_tc)
  return kmv_tc_launch_kind(p, p->kind, done_flag);
}

}  // namespace gp
