// gp_common.cuh -- shared declarations for libgpbbmm (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/gp_bbmm.h"
#include "plan_settings.h"

#ifndef __CUDA_ARCH_FEAT_SM90_ALL
#if defined(__CUDA_ARCH__)
#error "libgpbbmm is written for sm_90a only: compile with -gencode arch=compute_90a,code=sm_90a"
#endif
#endif

namespace gp {

// ---- compile-time geometry ------------------------------------------------------------
constexpr int TP = 16;         // padded column count of every [N, t] block (t <= 16)
constexpr int TILE_I = 128;    // rows of K per CTA tile (two wgmma M = 64 warpgroups)
constexpr int TILE_J = 64;     // columns of K per pipeline step (wgmma N of GEMM1, K of GEMM2)
constexpr int KP_MAX = 128;    // max padded augmented feature width of the tensor-core path (3d+4 <= 128)
constexpr int SIMT_TI = 128;   // rows per CTA in the SIMT kernel
constexpr int SIMT_TJ = 64;    // staged columns per step in the SIMT kernel
// one packed 64-row tile of V (pack.cu): [64/4][32][4] tf32 (V_hi | V_lo) + [64/8][16][8] bf16
constexpr int V_TILE_FLOATS = (2 * TILE_J * TP * 4 + TILE_J * TP * 2) / 4;   // 2560
constexpr float LOG2E = 1.4426950408889634f;

// ---- error plumbing -----------------------------------------------------------------------
void set_error(const char* fmt, ...);
#define GP_CUDA(call)                                                                     \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess) {                                                             \
      gp::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return GP_E_CUDA;                                                                   \
    }                                                                                     \
  } while (0)
#define GP_CHECK(st)              \
  do {                            \
    int s__ = (st);               \
    if (s__ != GP_OK) return s__; \
  } while (0)
#define GP_REQUIRE(cond, code, ...) \
  do {                              \
    if (!(cond)) {                  \
      gp::set_error(__VA_ARGS__);   \
      return (code);                \
    }                               \
  } while (0)

// grow-only device buffer owned by a plan
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return GP_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
      return GP_E_CUDA;
    }
    cap = want;
    return GP_OK;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

// on-device scalar state of one mBCG run (SURVEY.md Appendix A.2)
struct CgState {
  double gamma[2][TP];    // residual_inner_prod, double-buffered by iteration parity
  float alpha[TP];
  float beta[TP];
  float rhs_norm[TP];
  float rnorm[TP];
  int conv[TP];           // has_converged
  int rhs_zero[TP];
  float prev_ar[TP];      // prev_alpha_reciprocal
  float prev_beta[TP];
  int update_tridiag;
  int last_tridiag_iter;
  int done;               // set once the stop rule fires; later launches become no-ops
  int iters;              // iterations executed when done was set
  int tol_reached;
  int nan_flag;
};

// ---- pinned host scratch (gp_plan::pinned): one fixed byte offset per user ------------------------------------------------
constexpr size_t PINNED_BYTES = 32768;
constexpr size_t PIN_DONE_RING = 0;     // int[2]: look-ahead done flags of the mBCG / msMINRES loops (rowpass.cuh)
constexpr size_t PIN_CG_STATE = 64;     // CgState read back after mBCG (cg.cu)
constexpr size_t PIN_PC_STATE = 2048;   // PcState read back after the pivoted Cholesky (pivchol.cu)
constexpr size_t PIN_PRECOND = 3072;    // log det, tail, fail flag of gp_precond_build (pivchol.cu)
constexpr size_t PIN_SLQ = 3200;        // 64 per-probe log-dets + fail flag (slq.cu)
constexpr size_t PIN_SCALARS = 4096;    // gp_mll: 64 inv-quad partials (api.cu); gp_lanczos: 2 scalars, then from +64 the k + 1
                                        // Gram-Schmidt coefficients of step k, which run past the end for num_iter >= 3578
constexpr size_t PIN_CIQ_TW = 8192;     // tau | w of CIQ, 2 Q <= 64 doubles (minres.cu)
constexpr size_t PIN_CIQ_OUT = 12288;   // msMINRES read-back: residuals, iterations, flags (minres.cu)
static_assert(PIN_DONE_RING + 2 * sizeof(int) <= PIN_CG_STATE, "done ring overlaps the CgState slot");
static_assert(PIN_CG_STATE + sizeof(CgState) <= PIN_PC_STATE, "CgState overflows its pinned slot");
static_assert(PIN_PRECOND + 2 * sizeof(double) + sizeof(int) <= PIN_SLQ, "gp_precond_build read-back overflows its pinned slot");
static_assert(PIN_SLQ + 64 * sizeof(double) + sizeof(int) <= PIN_SCALARS, "SLQ read-back overflows its pinned slot");
static_assert(PIN_SCALARS + 64 * sizeof(double) <= PIN_CIQ_TW, "gp_mll read-back overflows its pinned slot");

// Raises KERNEL's dynamic shared-memory limit to `bytes` on `device` the first time any thread asks for it there (plans are
// driven from several host threads at once); later calls return the first call's result.
template <auto KERNEL>
int opt_in_smem(int device, int bytes) {
  static std::once_flag once[64];
  static cudaError_t err[64];
  const int slot = device & 63;
  std::call_once(once[slot], [&] { err[slot] = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); });
  if (err[slot] != cudaSuccess) {
    set_error("cudaFuncSetAttribute(MaxDynamicSharedMemorySize = %d) -> %s", bytes, cudaGetErrorString(err[slot]));
    return GP_E_CUDA;
  }
  return GP_OK;
}

}  // namespace gp

// SKI / KISS-GP backend state (ski.cu): grid geometry, compact interpolation data, grid work blocks, Toeplitz factors
struct gp_ski_state {
  int G[4] = {0, 0, 0, 0};
  float lo[4] = {0, 0, 0, 0}, step[4] = {0, 0, 0, 0};
  int64_t M = 0;
  int tile_edge[4] = {0, 0, 0, 0}, tile_num[4] = {0, 0, 0, 0}, ntiles = 0;   // spatial buckets of the points (ski.cu)
  gp::DevBuf first, wts, gridA, gridB, gridC, gridD, T, dT, flag;
  gp::DevBuf perm, tile_off, tile_cnt, first_s, wts_s;                        // points sorted by tile + the permutation back
  gp::DevBuf tcol, dtcol, band;   // generating columns t_i, l dt_i/dl (sum_i G_i floats each) and their band ends (8 ints)
};

// Hadamard multitask state (tasks.cu): the operator is s K o B[t, t'].  Rows are sorted by task (stable), the columns of task b
// form one segment of the packed column layout (on the tensor-core path every segment starts at a 64-column tile), and one K.V
// is one launch of the plain fused kernel per column task into its own partial slots, combined with B row by row.
struct gp_task_state {
  int T = 0;
  std::vector<int> t1, t2;                 // host copies of the task ids (user order)
  std::vector<int64_t> off1, off2;         // [T + 1] start of every task in the sorted row / column order
  std::vector<int> perm1, perm2;           // sorted position -> user index
  // column layout of the packed inputs (backend dependent, tasks_pack): segment b = positions [seg[b], seg[b] + cnt_b)
  std::vector<int64_t> seg;                // [T + 1]
  int64_t ncol_layout = 0;
  std::vector<int64_t> tps;                // per column task: tiles (tensor cores) / columns (SIMT) per split
  std::vector<int> nsplit, slot0;          // per column task: splits and first partial slot (slot0[T] = all slots)
  bool lay_ok = false, lay_tc = false;     // the column layout above is current for this backend
  std::vector<float> B;                    // host T x T task covariance, row-major
  bool b_set = false;
  gp::DevBuf ids;                          // perm1 [n1] | ts1 [n1] (sorted row tasks) | t1 [n1] | t2 [n2] (user order)
  gp::DevBuf lay;                          // map2 [ncol_layout] (layout position -> user column, -1 = padding) | slot_task | slot0
  gp::DevBuf Bd;                           // B on the device
  gp::DevBuf Zs1, Zs2, Vs, Ls, tpart, red;
  int* d_perm1 = nullptr;
  int* d_ts1 = nullptr;
  int* d_t1 = nullptr;
  int* d_t2 = nullptr;
  int* d_map2 = nullptr;
  int* d_slot_task = nullptr;
  int* d_slot0 = nullptr;
};

constexpr int KRON_MAX_TERMS = 4;   // latent processes of one Kronecker plan (gp_plan_set_kron_terms)

// Kronecker multitask state (kron.cu): the operator is (s K_data) (x) B over interleaved rows i T + a.  One K.V mixes the block by
// B into ceil(T t / 16) zero-padded [N2, 16] column chunks, runs the data plan's fused kernel once per chunk into its own partial
// slots, and scatters the chunks back to rows i T + a of partial slot 0.
struct gp_kron_state {
  gp_plan* data = nullptr;                 // caller-owned plain plan of K_data
  int T = 0;
  std::vector<float> B;                    // host T x T task covariance, row-major
  bool b_set = false;
  bool b_bad = false;                      // B has a non-finite entry: every product and gradient is NaN
  gp::DevBuf Bd;                           // B on the device
  gp::DevBuf W, Vt, part;                  // mixed chunks [nchunk][npad][16] | their packed V tiles | data's slots per chunk
  gp::DevBuf Lw, red, idx, rows;           // gradient / row-extraction scratch
  // observed rows / columns (gp_plan_set_kron_observed): the operator is P_r ((s K) (x) B) P_c^T.  Host index lists (empty: all
  // observed), on the device the maps and their inverses (-1 where an interleaved row is not observed) as int32 (N T < 2^31)
  bool masked = false;
  int64_t mask_n1 = 0, mask_n2 = 0;        // data plan sizes N1, N2 the mask was given for
  std::vector<int> obs_r, obs_c;
  gp::DevBuf rowmap, colmap, rowpos, colpos;
  gp::DevBuf Lx, Rx, full, gidx;           // gradient operands expanded to N T rows | full rows / diagonal before the gather |
                                           // the interleaved row of each requested row
  // several latent processes (gp_plan_set_kron_terms, LCM): sum_q (s_q K_q) (x) B_q with Q = nterm terms; data == term[0], B and Bd
  // hold the Q blocks back to back (gp_plan_set_kron_term_covars).  nterm = 1 is the single-term operator above
  int nterm = 1;
  gp_plan* term[KRON_MAX_TERMS] = {};
};

// Derivative-observation state (deriv.cu, deriv_table.cuh): the RBF or Matern-5/2 value / gradient operator over interleaved rows
// i (d+1) + a on a plain data plan of the same kind.  Per dimension c < d: w[c] = 1 / (sqrt(C) l_c) turns a packed difference
// (z = (x - mean) sqrt(C) / l, C = log2 e for RBF, 10 for Matern-5/2, pack.cu) into u_c = D_c / l_c^2, il2[c] = 1 / l_c^2; both
// are 0 for c >= d.
constexpr int DERIV_DMAX = 16;   // d + 1 rows per point stay within the engine's 32-task limit; the kernels are built for DP <= 16
constexpr int DV_TI = 128;       // derivative kernels: points per CTA, one per thread
constexpr int DV_TJ = 64;        // staged points of the other side per step
struct DerivHyp {
  float w[DERIV_DMAX];
  float il2[DERIV_DMAX];
};
struct gp_deriv_state {
  gp_plan* data = nullptr;                 // caller-owned plain plan of covariance `kind`
  int kind = GP_RBF;                       // GP_RBF (gp_plan_set_deriv) or GP_MATERN52 (gp_plan_set_deriv_kind)
  DerivHyp hyp;                            // from data's lengthscales at the last refresh (kernel parameter)
  bool hyp_set = false;
  int nsplit = 1;                          // column splits of the derivative kernels (deriv_geometry)
  int64_t cps = 0;                         // points of the other side per split
  gp::DevBuf part, gout, hypd;             // split partials [nsplit][N1 (d+1)][16] | gradient CTA partials | hyp on the device
};

// Compact-support backend (compact.cu, GP_BACKEND_COMPACT): piecewise polynomial kernels over points in Morton order.  Row tiles
// of 128 and column tiles of 64 sorted points; per row tile the CSR list of the column tiles within reach (box gap < 1 in x / l).
constexpr int PP_DMAX = 16;      // input dimensions: bounds the template cases and the exponent j + q <= 15
constexpr int PP_TI = 128;       // sorted rows per row tile (one per thread)
constexpr int PP_TJ = 64;        // sorted columns per column tile
constexpr int PP_MAX_SLOTS = 32; // partial slots one row tile's list is split across
struct gp_compact_state {
  int q = 2;
  bool order_stale = true;         // set by gp_plan_set_data: the Morton order and the raw tile boxes are redone at the next packing
  int64_t ntile_i = 0, ntile_j = 0;
  int64_t pairs = 0;               // evaluated tile pairs of the current schedule
  int chunk = 1;                   // column tiles per partial slot of one row tile
  gp::DevBuf perm1, perm2;         // sorted position -> caller's row (int32) of the row / column side (perm2 aliases perm1 square)
  gp::DevBuf box1, box2;           // raw fp32 tile boxes [ntile][2][d] (lo | hi) of each side
  gp::DevBuf Zs1, Zs2;             // packed rows (x - mean) / l in sorted order [n][DP]
  gp::DevBuf rowptr, cols, cnt;    // CSR schedule: int64 [ntile_i + 1], int32 column tiles, int32 per-row-tile counts
  gp::DevBuf sortbuf, lohi, lsd;   // sort keys / values / CUB scratch; per-dimension lo / hi of the raw inputs; l_c in fp64
};

struct gp_comm {
  void* nccl_comm = nullptr;
  int rank = 0, world = 1;
};

struct gp_plan {
  int device = 0;
  cudaStream_t stream = nullptr;
  int n_sm = 132;
  int backend_req = GP_BACKEND_AUTO;
  int backend = GP_BACKEND_SIMT;
  int64_t launches = 0;
  // data
  const float* X1 = nullptr;
  const float* X2 = nullptr;
  int64_t n1 = 0, n2 = 0, ld1 = 0, ld2 = 0;
  int d = 0;
  bool same = false;
  int64_t row_begin = 0, row_count = 0;  // local rows of X1 (row sharding)
  bool data_set = false, hypers_set = false;
  // hypers
  int kind = GP_RBF;
  std::vector<float> ls;
  float outputscale = 1.f, noise = 0.f;
  const float* noise_diag = nullptr;  // optional per-row diagonal D [n2] (FixedNoiseGaussianLikelihood); replaces the scalar noise
  // derived geometry
  int DP = 0;      // padded feature width of the SIMT arrays
  int KP = 0;      // padded augmented width (3d+4 -> multiple of 8) of the tensor-core tiles
  int nsplit = 1;  // column splits of the K.V work (load balance over the SMs)
  int nparts = 1;  // partial-sum slots written by the K.V kernel (nsplit)
  int64_t ntile_i = 0, ntile_j = 0, tiles_per_split = 0;
  int64_t rows_pad = 0;  // local rows padded to 256: pitch of `partial`, rows of XA
  // device buffers
  int* xbad = nullptr;  // device flag: non-finite value in the packed inputs (lives behind mean[])
  gp::DevBuf mean, scale, Z1, Z2, XA, XB, V16, Vtiles, partial, out16;
  gp::DevBuf cgU, cgR, cgZ, cgP, cgV, cgPfull, red, sums, qtr, state, tmat_tmp, misc, misc2, misc3;
  gp::DevBuf pcdiag, pcperm, pcpos, pcstate, pcpart, gram, cholC;
  gp::DevBuf msw;   // multi-shift MINRES: Lanczos / direction blocks, partials, scalar state (minres.cu)
  gp_comm* comm = nullptr;
  gp_ski_state* ski = nullptr;   // non-null: backend == GP_BACKEND_SKI
  // kernel sums (GP_BACKEND_SUM): the terms (caller-owned plans over the same rows); while the parent launches a term's K.V
  // kernel the term writes into the parent's partial slots and reads the parent's packed V tiles
  std::vector<gp_plan*> terms;
  bool sum_tc = false;            // every term runs the tensor-core kernel (the direction block is packed once for all of them)
  bool sum_any_tc = false;        // at least one term reads the packed V tiles
  float* partial_ext = nullptr;   // set on a TERM for the duration of one launch by its parent
  float* vtiles_ext = nullptr;
  gp::DevBuf part_scale;          // [nslots] scale of each partial slot: the owning term's outputscale, 1 for the low-rank slot
  std::vector<float> part_scale_host;
  // low-rank correction (lowrank.cu): the operator is  s K - U U^T ; U [n2, lr_r] (leading dimension lr_ld) is caller-owned
  const float* lr_U = nullptr;
  int64_t lr_ld = 0;
  int64_t lr_n = 0;               // rows of U: the operator size when the correction was set (re-checked at every use)
  int lr_r = 0;
  gp::DevBuf lrw;                 // U^T V partials [G][16 r] | c = U^T V [r][16] fp64
  gp_task_state* tasks = nullptr; // non-null: Hadamard multitask operator s K o B[t, t'] (gp_plan_set_tasks)
  gp_kron_state* kron = nullptr;  // non-null: Kronecker multitask operator (s K_data) (x) B (gp_plan_set_kron)
  gp_deriv_state* deriv = nullptr;   // non-null: derivative-observation operator over a plain RBF plan (gp_plan_set_deriv)
  // kernel products (GP_BACKEND_PRODUCT, product.cu): the factors (caller-owned plain plans over the same rows); the plan's
  // outputscale is the product of theirs, its xbad flag the OR of theirs
  std::vector<gp_plan*> factors;
  bool prod_tc = false;           // two tensor-core factors with KP_a + KP_b <= 128: product_tc_kernel, else product_simt_kernel
  uint64_t pack_gen = 0;          // bumped by every re-pack of a plain plan
  uint64_t fac_gen[4] = {0, 0, 0, 0};   // the factors' pack_gen at the last product_pack
  // additive GPs (additive.cu): sum_{m=1}^{add_M} e_m(c_1 .. c_D), c_i = add_s[i] k(x_i, x'_i) over the D = d columns of a plain
  // SIMT plan with D ARD lengthscales; add_M = 0 is a plain plan.  The plan's outputscale is not applied (kernel_scale)
  int add_M = 0;
  std::vector<float> add_s;       // the D component scales
  double add_diag = 0.0;          // sum_{m=1}^{M} e_m(s_1 .. s_D): the constant diagonal of a square operator
  // spectral mixture kernels (spectral.cu): S prod_d sum_q w_q exp(-2 pi^2 v_qd^2 tau_d^2) cos(2 pi mu_qd tau_d) on a plain SIMT
  // plan whose Z1 / Z2 hold the packed rows [x | reduced phases] of DP = pad4(d + Q d) floats; sm_Q = 0 is a plain plan
  int sm_Q = 0;
  std::vector<float> sm_w, sm_mu, sm_v;   // weights [Q], means and scales [Q][d]
  double sm_diag = 0.0;           // S (sum_q w_q)^d: the constant diagonal of a square operator
  // periodic kernels (periodic.cu): S exp(-2 sum_d sin^2(pi tau_d / p_d) / l_d) as the RBF kernel of unit lengthscale over the
  // embedding u_d(x) = (cos, sin)(2 pi x_d / p_d) / sqrt(l_d); from the packing on the plan is a plain RBF plan of 2d packed
  // columns (packed_dims).  per_n = 0 is a plain plan, else 1 (one shared period) or d
  int per_n = 0;
  std::vector<float> per_p;       // the per_n periods
  // rational quadratic kernels (kind GP_RQ, gp_plan_set_hypers_rq): (1 + r^2 / (2 alpha))^-alpha over z = (x - mean) / l
  float rq_alpha = 0.f;
  // polynomial kernels (kind GP_POLY, gp_plan_set_hypers_poly): S (x.x' + c)^p over the raw inputs (no centring, no lengthscale)
  int poly_power = 0;
  float poly_offset = 0.f;
  gp_compact_state* compact = nullptr;   // non-null: piecewise polynomial kernel on GP_BACKEND_COMPACT (gp_plan_set_hypers_pp)
  int kron_cols = 16;             // columns of V16 a Kronecker or derivative product computes (KronColsScope); the rest must be zero or unused
  void* pinned = nullptr;  // small pinned host scratch: PINNED_BYTES, one PIN_* slot per user
};

// A solver loop that applies a Kronecker operator to blocks of t < 16 live columns narrows the mix to those columns for its
// lifetime: ceil(T t / 16) data-kernel launches per product instead of T.  Other plans ignore it.
struct KronColsScope {
  gp_plan* p;
  int old;
  KronColsScope(gp_plan* plan, int t) : p(plan), old(plan->kron_cols) { p->kron_cols = t < 1 ? 1 : (t > 16 ? 16 : t); }
  ~KronColsScope() { p->kron_cols = old; }
};

namespace gp {

// ---- plan settings (plan_settings.h), api.cu ---------------------------------------------
uint32_t plan_settings(const gp_plan* p);              // the PlanSetting bits p carries
int refuse_settings(const gp_plan* p, CallId call);    // GP_E_STATE naming the first setting of p that `call` refuses, else GP_OK

// ---- launches implemented across the .cu files -------------------------------------------
int pack_inputs(gp_plan* p);                                            // pack.cu
int to_v16(gp_plan* p, const float* V, int64_t ldv, int t, int64_t n, float* V16);
int pack_v_tiles(gp_plan* p, const float* V16);                         // pack.cu (tensor-core B operand of GEMM2)
int kmv_partials(gp_plan* p, const float* V16, const int* done_flag);   // dispatch simt / tensor cores
int kmv_tc_launch_kind(gp_plan* p, int kind, const int* done_flag);     // kind may be GP_DERIV + kind, or RQ_DL / RQ_DA on an RQ plan
int product_tc_launch(gp_plan* p, const int* done_flag);                // kmv_tc.cu: the two tensor-core factors of a product plan
int kmv_simt_launch(gp_plan* p, const float* V16, const int* done_flag);
int kmv_tc_launch(gp_plan* p, const int* done_flag);
int kmv_finish_user(gp_plan* p, const float* V16, float* OUT, int64_t ldo, int t, int add_noise);
int choose_geometry(gp_plan* p);
void choose_splits(gp_plan* p, bool tc);                                // column splits of the K.V work from ntile_i / ntile_j / n_sm
int ski_pack(gp_plan* p);                                               // ski.cu
int ski_kmv_partials(gp_plan* p, const float* V16, const int* done_flag);
int ski_bilinear(gp_plan* p, const float* L16, const float* R16, double* total);   // total[0] += <A, K_uu B>, total[1 + i] += <A, (l_i dK_uu/dl_i) B>
int sum_pack(gp_plan* p);                                               // sum.cu: geometry / buffers of a kernel-sum plan
int slot_scales_prepare(gp_plan* p);                                    // refresh the per-slot scales (sum / low-rank plans only)
int sum_kmv_launch(gp_plan* p, const float* V16, const int* done_flag); // one launch per term into the parent's partial slots
int product_pack(gp_plan* p);                                           // product.cu: validation / geometry / scale of a kernel product
int product_refresh(gp_plan* p);                                        // re-pack when a factor was re-packed since (host compare)
int product_kmv_launch(gp_plan* p, const float* V16, const int* done_flag);   // one launch: prod_f k_f V into the plan's partial slots
int product_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);   // the factors' rows multiplied in order
int product_kdiag_cross(gp_plan* p, float* OUT);                        // diagonal of a cross product: the factors' diagonals multiplied
int product_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os);
int lowrank_partials(gp_plan* p, const float* V16, const int* done_flag);   // lowrank.cu: -U U^T V into the last slot (no-op without U)
int lowrank_kdiag(gp_plan* p, float* OUT);                              // OUT[i] -= sum_j U_ij^2
int lowrank_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);   // OUT[r] -= U[idx_r] U^T
int sum_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);       // rows of a kernel sum (terms added in order)
// one launch of the fused kernels over an explicit column block (Hadamard plans): columns [0, ntile_j) tiles of XB / Vt (tensor
// cores) or [0, n2) rows of Z2 / V16 (SIMT), partial slots from `partial`, diag_row_begin = row_begin of the exact-diagonal test
int kmv_tc_launch_cols(gp_plan* p, int kind, const float* XA, const float* XB, const float* Vt, float* partial, int64_t ntile_j,
                       int64_t tiles_per_split, int nsplit, int64_t diag_row_begin, const int* done_flag);
int kmv_simt_launch_cols(gp_plan* p, int kind, const float* Z1, const float* Z2, const float* V16, float* partial, int64_t n2,
                         int64_t cols_per_split, int nsplit, int64_t diag_row_begin, const int* done_flag);
int sum_partials_double(gp_plan* p, const double* in, int64_t nblk, int stride, int nout, double* out);   // out[o] = sum_b in[b][o], NaN when xbad
bool sum_has_poly(const gp_plan* p);                                    // kmv_simt.cu: a kernel sum with a polynomial term
int sum_kdiag_terms(gp_plan* p, float* OUT);                            // kmv_simt.cu: its per-row diagonal, term by term
int64_t bilinear_blocks(const gp_plan* p, int64_t n2);                      // CTAs of one SIMT derivative launch over n2 columns
void bilinear_split(const gp_plan* p, int64_t n2, dim3* grid, int64_t* cps);  // its grid and columns per split (kmv_simt.cu)
int bilinear_launch_cols(gp_plan* p, bool ard, const float* Z1, const float* Z2, const float* L16, const float* R16, int64_t n2,
                         int64_t diag_row_begin, double* gout, int gstride, int64_t* nblk_out);
int pack_v_tiles_rows(gp_plan* p, const float* V16, int64_t nrows, int64_t ntiles, float* Vt);
int pack_tc_rows(gp_plan* p, const float* Z, int64_t nvalid, int64_t npad, bool is_a, float* out);
int tasks_pack(gp_plan* p);                                                  // tasks.cu
int tasks_kmv_partials(gp_plan* p, const float* V16, int kind, const int* done_flag);   // K o B V into partial slot 0
int tasks_kdiag_scale(gp_plan* p, float* OUT);                               // OUT[i] *= B[t1_i, t2_i]
int tasks_krows_scale(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);
int tasks_bilinear(gp_plan* p, const float* L16, const float* R16, bool ard, std::vector<double>& total);
int kron_pack(gp_plan* p);                                                   // kron.cu
int kron_kmv_partials(gp_plan* p, const float* V16, const int* done_flag);   // (s K) (x) B V into partial slot 0 (unscaled)
int kron_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);
int kron_kdiag(gp_plan* p, float* OUT);
int kron_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os);
int kron_refresh(gp_plan* p);                                                // re-check the data plan, take its scale / kind / flag
int kron_set_task_covar(gp_plan* p, const float* B, int T);                  // gp_plan_set_task_covar on a Kronecker plan
int kron_task_covar_grad_checked(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB);
int deriv_pack(gp_plan* p);                                                  // deriv.cu
int deriv_kmv_partials(gp_plan* p, const float* V16, const int* done_flag);  // K_grad V into partial slot 0 (unscaled)
int deriv_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);
int deriv_kdiag(gp_plan* p, float* OUT);
int deriv_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os);
int deriv_refresh(gp_plan* p);                                               // re-check the data plan, take its scale / lengthscales / flag
double deriv_trace(const gp_plan* p);                                        // s N (1 + c sum_c 1 / l_c^2) in fp64, c = 1 or 5/3
int mbcg_run(gp_plan* p, const float* RHS, int64_t ldr, int t, int n_tridiag, float tol, int max_iter,   // cg.cu
             int max_tridiag_iter, const float* W, int k, float* SOLVES, int64_t lds, float* TMAT, int* iters_out,
             int* tridiag_size, float* resid_out);
int nccl_allreduce_double(gp_comm* c, double* buf, size_t count, cudaStream_t st);                     // comm.cu
int nccl_allgather_float(gp_comm* c, float* buf, size_t count_per_rank, cudaStream_t st);
inline float* partial_ptr(gp_plan* p) { return p->partial_ext ? p->partial_ext : p->partial.as<float>(); }
inline float* vtiles_ptr(gp_plan* p) { return p->vtiles_ext ? p->vtiles_ext : p->Vtiles.as<float>(); }
// partial slots the finish kernels sum: the backend's nparts, plus the low-rank slot
inline int nslots(const gp_plan* p) { return p->nparts + (p->lr_U ? 1 : 0); }
// per-slot scales of the finish kernels: nullptr = one outputscale for all slots
inline const float* part_scale_ptr(gp_plan* p) {
  return (p->backend == GP_BACKEND_SUM || p->lr_U) ? p->part_scale.as<float>() : nullptr;
}
// the scale the finish kernels apply to the backend's slots: the outputscale, or 1 on an additive plan (whose components carry
// their own scales)
inline float kernel_scale(const gp_plan* p) { return p->add_M ? 1.f : p->outputscale; }
// additive.cu
int additive_pack(gp_plan* p);                                          // checks the plan against its components, forms add_diag
int additive_kmv_launch(gp_plan* p, const float* V16, const int* done_flag);
int additive_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);
int additive_kdiag(gp_plan* p, float* OUT);
int additive_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os);
// spectral.cu
int spectral_pack(gp_plan* p);                                          // packs [x | reduced phases] into Z1 / Z2, forms sm_diag
int spectral_kmv_launch(gp_plan* p, const float* V16, const int* done_flag);
int spectral_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);
int spectral_kdiag(gp_plan* p, float* OUT);
int spectral_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os);
// periodic.cu
int periodic_pack(gp_plan* p);                                          // embeds the inputs into Z1 / Z2 (and the tensor-core tiles)
int periodic_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os);
// compact.cu
int compact_pack(gp_plan* p);                                           // Morton order (when stale), sorted rows, tile lists, slots
int compact_kmv_partials(gp_plan* p, const float* V16, const int* done_flag);
int compact_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os);
int refuse_compact(const gp_plan* p, const char* call);                 // GP_E_STATE when p runs on GP_BACKEND_COMPACT
void compact_release(gp_plan* p);                                       // back to a plain plan (frees the backend state)
// columns of the packed rows the plain kernels see: the d inputs, or the 2d embedding columns of a periodic plan
inline int packed_dims(const gp_plan* p) { return p->per_n ? 2 * p->d : p->d; }
inline bool plan_is_tc(const gp_plan* p) {
  return p->backend == GP_BACKEND_TCGEN05 || (p->backend == GP_BACKEND_SUM && p->sum_tc) || (p->backend == GP_BACKEND_PRODUCT && p->prod_tc);
}

__host__ __device__ inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Per-plan parameters of the covariance, passed by value to every kernel that evaluates it; only GP_RQ and GP_POLY read them (the
// other kinds' code does not change with it).
struct CovParam {
  float alpha;    // RQ: alpha > 0
  float ialpha;   // RQ: 1 / alpha, rounded once from fp64
  float offset;   // POLY: c >= 0 (packed into the GEMM1 operands on the tensor-core path, added to the dot product on the CUDA cores)
  int power;      // POLY: 1 <= p <= 8
  int pp_e;       // PPOLY: exponent j + q <= 15
  float pp_c1, pp_c2, pp_c3;   // PPOLY: poly_q(r) = 1 + c1 r + c2 r^2 + c3 r^3, rounded once from fp64
};
CovParam pp_param(int q, int d);   // compact.cu: the piecewise polynomial's exponent and coefficients for d input columns
inline CovParam cov_param(const gp_plan* p) {
  if (p->kind == GP_PPOLY) return pp_param(p->compact ? p->compact->q : 0, p->d);
  if (p->kind == GP_POLY) return CovParam{0.f, 0.f, p->poly_offset, p->poly_power};
  return p->kind == GP_RQ ? CovParam{p->rq_alpha, (float)(1.0 / (double)p->rq_alpha), 0.f, 0} : CovParam{0.f, 0.f, 0.f, 0};
}

// ---- device helpers -----------------------------------------------------------------------
#if defined(__CUDACC__)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// round-to-nearest (ties away) to tf32: the tensor core truncates fp32 containers to their top 19 bits,
// so operands are pre-rounded and the 2-term split x = hi + lo is exact to ~2^-24 |x|.  A NaN keeps its bits: the rounding add
// would carry the payload of CUDA's canonical NaN 0x7fffffff (what fmaf returns for a NaN operand) into the sign bit, giving -0.
__device__ __forceinline__ float tf32_hi(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x7fffffffu) > 0x7f800000u ? x : __uint_as_float((u + 0x1000u) & 0xFFFFE000u);
}

// covariance from a = -0.5 |z_i - z_j|^2 in the pre-scaled units of pack.cu:
//   RBF     z = (x - mean) sqrt(log2 e) / l      k = 2^a                (rbf_covariance.py:19)
//   Matern  z = (x - mean) sqrt(4 nu) / l        rho^2 = -a = 2 nu r^2  (matern_covariance.py:21-47)
//   RQ      z = (x - mean) / l               t = -a / alpha = r^2 / (2 alpha),  k = (1 + t)^-alpha   (rq_kernel.py)
// internal "derivative kinds": the same tile loop evaluates g = l dk/dl (scalar lengthscale) instead of k, so that
// the bilinear derivative  sum_ij (L_i . R_j) g_ij = sum_i L_i . (G R)_i  is one more fused K.V launch
// (lazy_evaluated_kernel_tensor.py:69-105, functions/rbf_covariance.py:20-29, functions/matern_covariance.py:27-56)
// GP_DERIV + kind covers the four RBF / Matern kinds only: its codes 4..7 are the template arguments of the existing derivative
// instantiations (kmv_tc_kernel<4..7>).  The public GP_RQ = 4 is the same number, so it never reaches a template or a GP_DERIV +
// kind switch: every dispatcher first maps a plan of kind GP_RQ to the RQ codes below (rq_code), which no other kind uses.
constexpr int GP_DERIV = 4;   // GP_DERIV + kind, kind in GP_RBF .. GP_MATERN52
constexpr int RQ_K = 16;      // RQ: k
constexpr int RQ_DL = 17;     // RQ: l dk/dl (scalar lengthscale)
constexpr int RQ_DA = 18;     // RQ: dk/dalpha
__host__ __device__ constexpr bool is_rq_code(int code) { return code >= RQ_K && code <= RQ_DA; }
// Polynomial kernels (DESIGN 4.21): the kernel argument is not a distance but a = x_i . x_j + c over the raw inputs, and
// k = a^p, dk/dc = p a^(p-1) (FMA pipe only, no MUFU).  The public GP_POLY = 5 is the number of GP_DERIV + GP_MATERN12, so, as for
// RQ, only these codes of their own (two digits) reach a template.
constexpr int POLY_K = 24;    // POLY: k = a^p
constexpr int POLY_DC = 25;   // POLY: dk/dc = p a^(p-1)
__host__ __device__ constexpr bool is_poly_code(int code) { return code == POLY_K || code == POLY_DC; }
// Piecewise polynomial kernels (DESIGN 4.24): k = (1 - r)_+^e poly_q(r) with r = sqrt(-2 a) in the packed units (C = 1).  The public
// GP_PPOLY = 6 is the number of GP_DERIV + GP_MATERN32, so only this code of its own reaches a template.
constexpr int PP_K = 32;
// the code a dispatcher evaluates for `kind` on plan p: on an RQ plan GP_RQ (the plan's own kind) is RQ_K, on a polynomial plan
// GP_POLY is POLY_K
inline int rq_code(const gp_plan* p, int kind) {
  if (p->kind == GP_PPOLY && kind == GP_PPOLY) return PP_K;
  if (p->kind == GP_POLY && kind == GP_POLY) return POLY_K;
  return (p->kind == GP_RQ && kind == GP_RQ) ? RQ_K : kind;
}
// a^q for 0 <= q <= 8 by squaring: a^2, a^4, a^8 and the product of the ones q selects.  Every tree of multiplies that forms a^q
// carries at most (q - 1) roundings of 2^-24 relative (each product adds one to the sum of its factors'), as q - 1 multiplies in
// a row would; a negative a keeps the sign of a^q for odd q (torch.pow with an integral exponent)
__host__ __device__ __forceinline__ float poly_pow(float a, int q) {
  const float a2 = a * a, a4 = a2 * a2;
  float r = (q & 1) ? a : 1.f;
  if (q & 2) r *= a2;
  if (q & 4) r *= a4;
  if (q & 8) r = a4 * a4;   // q = 8 exactly (q <= 8)
  return r;
}

// m^e for 0 <= e <= 15 by squaring (m^2, m^4, m^8 and the product of the ones e selects)
__host__ __device__ __forceinline__ float pp_pow(float m, int e) {
  const float m2 = m * m, m4 = m2 * m2, m8 = m4 * m4;
  float r = (e & 1) ? m : 1.f;
  if (e & 2) r *= m2;
  if (e & 4) r *= m4;
  if (e & 8) r *= m8;
  return r;
}
// (1 - r)_+^e poly_q(r): exactly 0 for r >= 1, exactly 1 at r = 0
__host__ __device__ __forceinline__ float pp_k(float r, CovParam cp) {
  const float m = fmaxf(1.f - r, 0.f);
  return pp_pow(m, cp.pp_e) * fmaf(fmaf(fmaf(cp.pp_c3, r, cp.pp_c2), r, cp.pp_c1), r, 1.f);
}
// -dk/dr = m^(e-1) (e poly - m poly'), 0 for r >= 1 (m = 0, also where e = 1 leaves a kink at r = 1)
__host__ __device__ __forceinline__ float pp_mdk(float r, CovParam cp) {
  const float m = fmaxf(1.f - r, 0.f);
  const float P = fmaf(fmaf(fmaf(cp.pp_c3, r, cp.pp_c2), r, cp.pp_c1), r, 1.f);
  const float dP = fmaf(fmaf(3.f * cp.pp_c3, r, 2.f * cp.pp_c2), r, cp.pp_c1);
  return m > 0.f ? pp_pow(m, cp.pp_e - 1) * ((float)cp.pp_e * P - m * dP) : 0.f;
}

#if defined(__CUDACC__)
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
#endif
// RQ (DESIGN 4.20).  t = max(-a, 0) / alpha >= 0.  log2(1 + t) with an absolute error O(2^-24 t): the degree-6 Taylor polynomial of
// log1p on the FMA pipe below 1/16 (truncation t^7 / 7 < 2^-26 t), MUFU lg2 above, selected without a branch; the rounding of
// 1 + t and lg2's absolute error would otherwise be multiplied by alpha.  k = 2^(-alpha log2(1 + t)): two MUFU operations per entry.
__device__ __forceinline__ float rq_t(float a, CovParam cp) { return fmaxf(-a, 0.f) * cp.ialpha; }
#if defined(__CUDACC__)
__device__ __forceinline__ float rq_lg2_1p(float t) {
  float p = fmaf(t, -0.16666667f, 0.2f);
  p = fmaf(t, p, -0.25f);
  p = fmaf(t, p, 0.33333334f);
  p = fmaf(t, p, -0.5f);
  p = fmaf(t, p, 1.f);
  const float small = LOG2E * (t * p);
  const float big = lg2_approx(1.f + t);
  return t < 0.0625f ? small : big;
}
__device__ __forceinline__ float rq_k(float t, CovParam cp) { return ex2_approx(-cp.alpha * rq_lg2_1p(t)); }
// phi(t) = log1p(t) - t / (1 + t) = sum_{n>=2} (-1)^n (n-1)/n t^n  (dk/dalpha = -k phi) without cancellation: the series to n = 9
// below 1/8 (truncation 1.8 t^8 relative), the difference of the accurate log1pf and t / (1 + t) above (cancels at most a factor 18)
__device__ __forceinline__ float rq_phi(float t) {
  float s = fmaf(t, -0.88888889f, 0.875f);
  s = fmaf(t, s, -0.85714286f);
  s = fmaf(t, s, 0.83333333f);
  s = fmaf(t, s, -0.8f);
  s = fmaf(t, s, 0.75f);
  s = fmaf(t, s, -0.66666667f);
  s = fmaf(t, s, 0.5f);
  const float ser = (t * t) * s;
  const float dif = log1pf(t) - __fdividef(t, 1.f + t);
  return t < 0.125f ? ser : dif;
}
#endif

template <int KIND>
__device__ __forceinline__ float dcov_from_arg(float a, float* kout, CovParam cp);

template <int KIND>
__device__ __forceinline__ float cov_from_arg(float a, CovParam cp) {
  if (KIND == PP_K) {   // a = -r^2 / 2 from direct differences: r = 0 on the diagonal, k = 1
    return pp_k(sqrtf(fmaxf(-2.f * a, 0.f)), cp);
  } else if (KIND == POLY_K) {   // a = x_i . x_j + c (no clamp: a may be negative)
    return poly_pow(a, cp.power);
  } else if (KIND == POLY_DC) {
    return (float)cp.power * poly_pow(a, cp.power - 1);
  } else if (KIND == RQ_K) {
    return rq_k(rq_t(a, cp), cp);
  } else if (KIND == RQ_DL) {
    float k;
    return dcov_from_arg<RQ_K>(a, &k, cp);
  } else if (KIND == RQ_DA) {   // dk/dalpha = -k phi(t)
    const float t = rq_t(a, cp);
    return -rq_k(t, cp) * rq_phi(t);
  } else if (KIND >= GP_DERIV) {
    float k;
    return dcov_from_arg<KIND - GP_DERIV>(a, &k, cp);
  } else if (KIND == GP_RBF) {
    return ex2_approx(fminf(a, 0.f));
  } else {
    float rho = sqrt_approx(fmaxf(-a, 0.f));
    float e = ex2_approx(-LOG2E * rho);
    if (KIND == GP_MATERN12) return e;
    if (KIND == GP_MATERN32) return fmaf(rho, e, e);
    return fmaf(fmaf(rho, 0.33333334f, 1.f), rho, 1.f) * e;  // 1 + rho + rho^2/3
  }
}
// derivative factor: dk/d(log-ish) pieces for the bilinear gradient.  Returns g with
// dk/dl = g / l (scalar lengthscale):  RBF: sq*k ; M12: rho e ; M32: rho^2 e ; M52: (1+rho) rho^2/3 e ; RQ: r^2 k / (1 + t)
template <int KIND>
__device__ __forceinline__ float dcov_from_arg(float a, float* kout, CovParam cp) {
  if (KIND == POLY_K) {   // k and dk/dc = p a^(p-1): k = a a^(p-1)
    const float km1 = poly_pow(a, cp.power - 1);
    *kout = a * km1;
    return (float)cp.power * km1;
  } else if (KIND == RQ_K) {
    const float t = rq_t(a, cp);
    const float k = rq_k(t, cp);
    *kout = k;
    return (-2.f * fminf(a, 0.f)) * __fdividef(k, 1.f + t);   // r^2 = -2 a in the packed units (C = 1)
  } else if (KIND == GP_RBF) {
    float am = fminf(a, 0.f);
    float k = ex2_approx(am);
    *kout = k;
    return (-2.f / LOG2E) * am * k;  // |dx/l|^2 = -2 a / log2e
  } else {
    float m = fmaxf(-a, 0.f);
    float rho = sqrt_approx(m);
    float e = ex2_approx(-LOG2E * rho);
    if (KIND == GP_MATERN12) { *kout = e; return rho * e; }
    if (KIND == GP_MATERN32) { *kout = fmaf(rho, e, e); return m * e; }
    *kout = fmaf(fmaf(rho, 0.33333334f, 1.f), rho, 1.f) * e;
    return (rho + 1.f) * m * 0.33333334f * e;
  }
}
// Product form of the same covariances, for kernel products (product.cu).  In the packed units every kind is poly(rho) 2^e:
//   RBF     poly = 1, e = a;     Matern   rho = sqrt(-a), e = -log2e rho, poly = 1 + c1 rho + c2 rho^2
// with (c1, c2) = (0, 0) nu = 1/2, (1, 0) nu = 3/2, (1, 1/3) nu = 5/2, so  prod_f k_f = (prod_f poly_f) ex2(sum_f e_f): one ex2
// per pair whatever the number of factors, plus one sqrt per Matern factor.  l dk/dl has the same shape, gpoly(rho) 2^e with
//   RBF  gpoly = -2 a / log2e;   Matern  gpoly = rho (poly - poly') = rho ((1 - c1) + (c1 - 2 c2) rho + c2 rho^2)
// (dcov_from_arg's rho, rho^2, (1 + rho) rho^2 / 3).  CLAMP = false leaves an RBF argument unclamped, as cov_tc does.
struct CovPoly {
  float c1, c2;
};
__host__ __device__ inline CovPoly cov_poly_of(int kind) {
  return kind == GP_MATERN32 ? CovPoly{1.f, 0.f} : kind == GP_MATERN52 ? CovPoly{1.f, 0.33333334f} : CovPoly{0.f, 0.f};
}
template <bool CLAMP>
__device__ __forceinline__ void cov_poly_exp(bool rbf, CovPoly c, float a, float* poly, float* e) {
  if (rbf) {
    *poly = 1.f;
    *e = CLAMP ? fminf(a, 0.f) : a;
  } else {
    const float rho = sqrt_approx(fmaxf(-a, 0.f));
    *poly = fmaf(fmaf(c.c2, rho, c.c1), rho, 1.f);
    *e = -LOG2E * rho;
  }
}
// the same with the derivative polynomial gpoly (l dk/dl = gpoly 2^e for a scalar lengthscale)
__device__ __forceinline__ void dcov_poly_exp(bool rbf, CovPoly c, float a, float* poly, float* gpoly, float* e) {
  if (rbf) {
    const float am = fminf(a, 0.f);
    *poly = 1.f;
    *gpoly = (-2.f / LOG2E) * am;
    *e = am;
  } else {
    const float rho = sqrt_approx(fmaxf(-a, 0.f));
    *poly = fmaf(fmaf(c.c2, rho, c.c1), rho, 1.f);
    *gpoly = rho * fmaf(fmaf(c.c2, rho, c.c1 - 2.f * c.c2), rho, 1.f - c.c1);
    *e = -LOG2E * rho;
  }
}
// Additive GPs (additive.cu): components c_i = s_i k_i(z_i - z'_i) over one packed column each, combined by the positive
// recurrence e_m <- e_m + c_i e_{m-1} (m = M .. 1) into K = sum_{m=1}^{M} e_m(c_1 .. c_D).  No alternating signs: nothing cancels.
constexpr int ADD_DMAX = 32;   // components
constexpr int ADD_MMAX = 8;    // interaction degree
struct AddHyp {
  float s[ADD_DMAX];   // component scales (0 beyond D)
  int D, M;
  int rbf;             // kind RBF (else Matern with polynomial cp)
  CovPoly cp;
};
// e[0 .. MT] <- the recurrence with one more component c (degrees above M untouched; MT = M folds the test away)
template <int MT, class T>
__device__ __forceinline__ void esym_push(T (&e)[MT + 1], T c, int M) {
#pragma unroll
  for (int m = MT; m >= 1; --m)
    if (m <= M) e[m] = fma(c, e[m - 1], e[m]);
}
template <int MT, class T>
__device__ __forceinline__ T esym_total(const T (&e)[MT + 1], int M) {
  T k = e[1];
#pragma unroll
  for (int m = 2; m <= MT; ++m)
    if (m <= M) k += e[m];
  return k;
}
// k_i of one component from its packed difference df (RBF: poly = 1 folds away)
template <bool RBF>
__device__ __forceinline__ float add_comp(CovPoly cp, float df) {
  float pl, ex;
  cov_poly_exp<true>(RBF, cp, -0.5f * (df * df), &pl, &ex);
  return pl * ex2_approx(ex);
}
// one entry K(a, b) from two packed rows (rows, diagonal, pivoted Cholesky)
template <bool RBF>
__device__ __forceinline__ float add_pair(const AddHyp& h, const float* za, const float* zb) {
  float e[ADD_MMAX + 1];
  e[0] = 1.f;
#pragma unroll
  for (int m = 1; m <= ADD_MMAX; ++m) e[m] = 0.f;
  for (int c = 0; c < h.D; ++c) esym_push<ADD_MMAX>(e, h.s[c] * add_comp<RBF>(h.cp, za[c] - zb[c]), h.M);
  return esym_total<ADD_MMAX>(e, h.M);
}
__device__ __forceinline__ float add_pair_rt(const AddHyp& h, const float* za, const float* zb) {
  return h.rbf ? add_pair<true>(h, za, zb) : add_pair<false>(h, za, zb);
}
AddHyp additive_hyp(const gp_plan* p);   // additive.cu: the kernel argument of an additive plan
// Spectral mixture kernels (spectral.cu): the weights and the exponent coefficients beta_qc = -2 pi^2 v_qc^2 log2 e are uniform
// across threads and travel in the kernel argument; a packed row is [x_0 .. x_{d-1} | p_qc at d + q d + c] (reduced phases).
constexpr int SM_QMAX = 16;    // components
constexpr int SM_DMAX = 8;     // input dimensions
constexpr int SM_QDMAX = 32;   // Q d
constexpr int SM_WMAX = 40;    // packed row width: pad4(d + Q d) <= 40
struct SmHyp {
  float w[SM_QMAX];
  float beta[SM_QDMAX];
  int Q, d;
  float S;             // outputscale: rows, diagonals and pivoted-Cholesky entries (the K.V finish kernels apply it there)
};
// one entry S prod_c sum_q w_q 2^{beta_qc tau_c^2} cos(2 pi (p_qc - p'_qc)) from two packed rows (rows, diagonal, pivoted Cholesky)
__device__ __forceinline__ float sm_pair(const SmHyp& h, const float* za, const float* zb) {
  float k = h.S;
  for (int c = 0; c < h.d; ++c) {
    const float t = za[c] - zb[c];
    const float t2 = t * t;
    float s = 0.f;
    for (int q = 0; q < h.Q; ++q) {
      const int o = q * h.d + c;
      s = fmaf(h.w[q], ex2_approx(h.beta[o] * t2) * __cosf(6.2831853071795865f * (za[h.d + o] - zb[h.d + o])), s);
    }
    k *= s;
  }
  return k;
}
SmHyp spectral_hyp(const gp_plan* p);   // spectral.cu: the kernel argument of a spectral plan
// the argument a = x_i . x_j + c of a polynomial pair from two packed (raw, zero-padded) rows, fp32 FMAs in column order
__device__ __forceinline__ float poly_arg(const float* za, const float* zb, int n, float offset) {
  float s = 0.f;
  for (int c = 0; c < n; ++c) s = fmaf(za[c], zb[c], s);
  return s + offset;
}
// input-derivative factor q = dk/da of the same covariance (xgrad.cu): dk/dz_i = -q (z_i - z_j) in the packed units.
//   RBF: ln2 2^a ; M12: e / (2 rho) ; M32: e / 2 ; M52: (1 + rho) e / 6 ; RQ: k / (1 + t)      (e = exp(-rho), rho^2 = -a)
// q is the h of the raw-unit form  dk/dx_i = -h (x_i - x_j) / l^2  times l^2 / C (C = log2 e, 2, 6, 10 as in pack.cu).  A pair at
// distance 0 contributes 0 (its direction is 0; Matern-1/2's q is unbounded there): the caller masks a == 0.
//   POLY: not the difference form.  q = dk/da = p a^(p-1) with a = x_i . x_j + c and dk/dx_i = q x_j, so every pair contributes,
//   the diagonal of a square plan too (2 q_ii x_i from both arguments, which are the same point); xgrad.cu takes that branch.
template <int KIND>
__device__ __forceinline__ float hcov_from_arg(float a, CovParam cp) {
  if (KIND == POLY_K) {
    return (float)cp.power * poly_pow(a, cp.power - 1);
  } else if (KIND == RQ_K) {
    const float t = rq_t(a, cp);
    return __fdividef(rq_k(t, cp), 1.f + t);
  } else if (KIND == GP_RBF) {
    return 0.69314718f * ex2_approx(fminf(a, 0.f));
  } else {
    float rho = sqrt_approx(fmaxf(-a, 0.f));
    float e = ex2_approx(-LOG2E * rho);
    if (KIND == GP_MATERN12) return 0.5f * e / rho;
    if (KIND == GP_MATERN32) return 0.5f * e;
    return (rho + 1.f) * e * 0.16666667f;
  }
}
#endif

}  // namespace gp
