// lowrank.cu -- a low-rank correction on any square plan: the operator becomes  s K - U U^T  (+ its noise / per-row diagonal).
//
// The correction is one more partial slot, so no solver changes: every product runs the backend's K.V launches into slots
// [0, nparts) and then
//   utv    per-CTA fp32 partials of U^T V [G][16 r] (64-row chunks of U staged in shared memory, as the preconditioned msMINRES
//          passes stage theirs)
//   sum    c = U^T V [r][16] by the fixed-order fp64 reduction of the row passes (cg_sum_launch): deterministic, so repeated
//          products are bit-identical
//   apply  slot nparts = -U c
// and the finish kernels sum nslots(p) = nparts + 1 slots with the per-slot scales [s ... s, 1] (slot_scales_prepare).  All three
// launches honour the solver's done flag like the K.V launches.  The posterior covariance of LOVE, K** - K*x R R^T Kx*, is the
// caller this exists for (r = the Lanczos rank, <= 128).
#include "rowpass.cuh"

namespace gp {

constexpr int LR_RMAX = 128;

// odd pitch of a staged U row: the 8 rows a warp reads in lowrank_apply fall in 8 banks
__host__ __device__ inline int lr_pitch(int r) { return r | 1; }
inline size_t lr_utv_smem(int r) { return sizeof(float) * ((size_t)RP_ROWS * lr_pitch(r) + RP_ROWS * TP); }
inline size_t lr_apply_smem(int r) { return sizeof(float) * ((size_t)RP_ROWS * lr_pitch(r) + (size_t)r * TP); }

// rows [r0, r0 + nr) of U (leading dimension ldu) -> us [nr][pitch]
__device__ __forceinline__ int lr_stage_u(const float* __restrict__ U, int64_t ldu, int r, int64_t r0, int64_t n,
                                          float* __restrict__ us) {
  const int nr = (int)min((int64_t)RP_ROWS, n - r0);
  const int rp = lr_pitch(r);
  for (int e = threadIdx.x; e < nr * r; e += RP_THREADS) {
    const int i = e / r, a = e - i * r;
    us[i * rp + a] = U[(r0 + i) * ldu + a];
  }
  return nr;
}

// part[cta][a * 16 + c] = sum over the CTA's rows i of U[i][a] V[i][c]   (thread: c = tid & 15, a = (tid >> 4) + 16 j)
__global__ void __launch_bounds__(RP_THREADS)
lowrank_utv_kernel(const float* __restrict__ U, int64_t ldu, int r, const float* __restrict__ V16, int64_t n,
                   float* __restrict__ part, const int* __restrict__ done) {
  if (done && *done) return;
  extern __shared__ __align__(16) float lsh[];
  float* us = lsh;                           // [64][pitch]
  float* vs = lsh + RP_ROWS * lr_pitch(r);   // [64][16]
  const int tid = threadIdx.x, c = tid & 15, a0 = tid >> 4, rp = lr_pitch(r);
  float acc[LR_RMAX / 16] = {};
  for (int64_t r0 = (int64_t)blockIdx.x * RP_ROWS; r0 < n; r0 += (int64_t)gridDim.x * RP_ROWS) {
    const int nr = lr_stage_u(U, ldu, r, r0, n, us);
    for (int e = tid; e < nr * TP; e += RP_THREADS) vs[e] = V16[r0 * TP + e];
    __syncthreads();
    for (int i = 0; i < nr; ++i) {
      const float v = vs[i * TP + c];
#pragma unroll
      for (int j = 0; j < LR_RMAX / 16; ++j)
        if (a0 + 16 * j < r) acc[j] = fmaf(us[i * rp + a0 + 16 * j], v, acc[j]);
    }
    __syncthreads();
  }
  float* out = part + (size_t)blockIdx.x * TP * r;
#pragma unroll
  for (int j = 0; j < LR_RMAX / 16; ++j)
    if (a0 + 16 * j < r) out[(a0 + 16 * j) * TP + c] = acc[j];
}

// slot[i][c] = -sum_a U[i][a] cvec[a][c]   (row-pass layout: cg = tid & 3 a float4 column group, rl = tid >> 2 a row lane)
__global__ void __launch_bounds__(RP_THREADS)
lowrank_apply_kernel(const float* __restrict__ U, int64_t ldu, int r, const double* __restrict__ cvec, int64_t n,
                     float* __restrict__ slot, const int* __restrict__ done) {
  if (done && *done) return;
  extern __shared__ __align__(16) float lsh[];
  float* us = lsh;                           // [64][pitch]
  float* cs = lsh + RP_ROWS * lr_pitch(r);   // [r][16]
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2, rp = lr_pitch(r);
  for (int e = tid; e < r * TP; e += RP_THREADS) cs[e] = (float)cvec[e];
  for (int64_t r0 = (int64_t)blockIdx.x * RP_ROWS; r0 < n; r0 += (int64_t)gridDim.x * RP_ROWS) {
    __syncthreads();   // the previous chunk is consumed (first pass: cs is written)
    lr_stage_u(U, ldu, r, r0, n, us);
    __syncthreads();
    const int64_t i = r0 + rl;
    if (i < n) {
      const float* u = us + rl * rp;
      float4 s = make_float4(0, 0, 0, 0);
      for (int a = 0; a < r; ++a) {
        const float ua = u[a];
        const float4 c4 = reinterpret_cast<const float4*>(cs)[a * 4 + cg];
        s.x = fmaf(ua, c4.x, s.x); s.y = fmaf(ua, c4.y, s.y); s.z = fmaf(ua, c4.z, s.z); s.w = fmaf(ua, c4.w, s.w);
      }
      reinterpret_cast<float4*>(slot)[i * 4 + cg] = make_float4(-s.x, -s.y, -s.z, -s.w);
    }
  }
}

// OUT[i] -= sum_a U[i][a]^2, accumulated in index order
__global__ void lowrank_kdiag_kernel(const float* __restrict__ U, int64_t ldu, int r, int64_t n, float* __restrict__ OUT) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* u = U + i * ldu;
  float s = 0.f;
  for (int a = 0; a < r; ++a) s = fmaf(u[a], u[a], s);
  OUT[i] -= s;
}

// OUT[row][j] -= U[idx[row]] . U[j]   (grid: column blocks x rows; an out-of-range index keeps the NaN row of the base call)
__global__ void lowrank_krows_kernel(const float* __restrict__ U, int64_t ldu, int r, const int64_t* __restrict__ idx, int64_t n,
                                     float* __restrict__ OUT, int64_t ldo) {
  __shared__ float ui[LR_RMAX];
  const int64_t row = blockIdx.y;
  const int64_t i = idx[row];
  if (i < 0 || i >= n) return;   // CTA-uniform
  for (int a = threadIdx.x; a < r; a += blockDim.x) ui[a] = U[i * ldu + a];
  __syncthreads();
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const float* u = U + j * ldu;
  float s = 0.f;
  for (int a = 0; a < r; ++a) s = fmaf(ui[a], u[a], s);
  OUT[row * ldo + j] -= s;
}

// gp_plan_set_data / gp_plan_set_comm may change the operator after U was set: U then no longer matches it
static int lowrank_still_valid(const gp_plan* p) {
  GP_REQUIRE(p->same && p->n2 == p->lr_n && p->row_begin == 0 && p->row_count == p->n1 && !(p->comm && p->comm->world > 1), GP_E_STATE,
             "the low-rank correction was set for a square, unsharded operator of %lld rows; the plan's data or communicator changed "
             "since (%lld rows, rows [%lld,+%lld)): call gp_plan_set_lowrank again", (long long)p->lr_n, (long long)p->n2,
             (long long)p->row_begin, (long long)p->row_count);
  return GP_OK;
}

int lowrank_partials(gp_plan* p, const float* V16, const int* done_flag) {
  if (!p->lr_U) return GP_OK;
  GP_CHECK(lowrank_still_valid(p));
  GP_CHECK(slot_scales_prepare(p));
  GP_REQUIRE(p->partial.cap >= sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP, GP_E_STATE, "low-rank slot not allocated");
  cudaStream_t st = p->stream;
  const int64_t n = p->n2;
  const int r = p->lr_r;
  const int G = (int)std::min<int64_t>(cdiv(n, RP_ROWS), 2 * (int64_t)p->n_sm);
  const size_t L = (size_t)TP * r;
  GP_CHECK(p->lrw.ensure(sizeof(float) * G * L + sizeof(double) * L));
  float* part = p->lrw.as<float>();
  double* cvec = reinterpret_cast<double*>(part + (size_t)G * L);   // G * L * 4 bytes: a multiple of 64
  float* slot = p->partial.as<float>() + (size_t)p->nparts * p->rows_pad * TP;
  lowrank_utv_kernel<<<G, RP_THREADS, lr_utv_smem(r), st>>>(p->lr_U, p->lr_ld, r, V16, n, part, done_flag);
  cg_sum_launch(part, G, (int)L, cvec, done_flag, st);
  lowrank_apply_kernel<<<G, RP_THREADS, lr_apply_smem(r), st>>>(p->lr_U, p->lr_ld, r, cvec, n, slot, done_flag);
  p->launches += 3;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int lowrank_kdiag(gp_plan* p, float* OUT) {
  GP_CHECK(lowrank_still_valid(p));
  lowrank_kdiag_kernel<<<(unsigned)cdiv(p->n2, 256), 256, 0, p->stream>>>(p->lr_U, p->lr_ld, p->lr_r, p->n2, OUT);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int lowrank_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_CHECK(lowrank_still_valid(p));
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "rows of a low-rank plan: at most 65535 rows per call (m=%lld)", (long long)m);
  lowrank_krows_kernel<<<dim3((unsigned)cdiv(p->n2, 256), (unsigned)m), 256, 0, p->stream>>>(p->lr_U, p->lr_ld, p->lr_r, idx, p->n2,
                                                                                              OUT, ldo);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_lowrank(gp_plan* p, const float* U, int64_t ldu, int r) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  if (U == nullptr || r == 0) {
    p->lr_U = nullptr;
    p->lr_ld = 0;
    p->lr_n = 0;
    p->lr_r = 0;
    return GP_OK;
  }
  GP_REQUIRE(p->data_set, GP_E_STATE, "low-rank correction: call gp_plan_set_data first");
  GP_CHECK(refuse_settings(p, CALL_SET_LOWRANK));
  GP_REQUIRE(r >= 1 && r <= LR_RMAX, GP_E_SHAPE, "low-rank correction of rank %d: 1 <= r <= %d", r, LR_RMAX);
  GP_REQUIRE(ldu >= r, GP_E_SHAPE, "low-rank correction: ldu=%lld < r=%d", (long long)ldu, r);
  GP_REQUIRE(p->same, GP_E_SHAPE, "a low-rank correction needs a square operator (X2 == X1)");
  GP_REQUIRE(!(p->comm && p->comm->world > 1) && p->row_begin == 0 && p->row_count == p->n1, GP_E_SHAPE,
             "a low-rank correction is not supported on row-sharded plans");
  GP_CUDA(cudaSetDevice(p->device));
  p->lr_U = U;
  p->lr_ld = ldu;
  p->lr_n = p->n2;
  p->lr_r = r;
  if (p->hypers_set) {   // otherwise the packing (gp_plan_set_hypers) sizes the slots
    GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
    GP_CHECK(slot_scales_prepare(p));
  }
  return GP_OK;
}
