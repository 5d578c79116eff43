// rowpass.cuh -- the [n][16] row-pass layout shared by the mBCG (cg.cu) and multi-shift MINRES (minres.cu) solvers.
//
// Every vector block is [n][16] fp32.  A row-pass CTA has RP_THREADS threads: cg = tid & 3 picks a float4 column group,
// rl = tid >> 2 a row lane, so one pass covers RP_ROWS rows.  Column-wise dots are two-stage: per-CTA fp32 partials
// (block_reduce_cols), then a fixed-order fp64 sum over the CTAs (cg_sum_launch): deterministic.
#pragma once
#include "gp_common.cuh"

namespace gp {

constexpr int RP_THREADS = 256;
constexpr int RP_ROWS = 64;   // rows per pass of a CTA (4 float4 column groups x 64 row lanes)

// fixed-order fp64 sums of G partial rows of length L; launches are no-ops once *done is set (done may be null)
void cg_sum_launch(const float* in, int G, int L, double* out, const int* done, cudaStream_t st);
// per-CTA partials of the column sums of squares of RHS [n][t] (leading dimension ldr) into part [G][16]
void cg_rhs_sq_launch(const float* RHS, int64_t ldr, int t, int64_t n, float* part, int G, cudaStream_t st);

#if defined(__CUDACC__)
__device__ __forceinline__ void block_reduce_cols(float4 acc, float* red /*[RP_ROWS][TP]*/, float* out /*[TP] global*/) {
  const int tid = threadIdx.x, cg = tid & 3, rl = tid >> 2;
  reinterpret_cast<float4*>(red)[rl * 4 + cg] = acc;
  __syncthreads();
  for (int s = RP_ROWS / 2; s > 0; s >>= 1) {
    if (rl < s) {
      float4 a = reinterpret_cast<float4*>(red)[rl * 4 + cg];
      float4 b = reinterpret_cast<float4*>(red)[(rl + s) * 4 + cg];
      reinterpret_cast<float4*>(red)[rl * 4 + cg] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
    __syncthreads();
  }
  if (tid < TP) out[tid] = red[tid];
}

// K_hat X of row r, column group cg: os sum_s partial_s + d_r x, from the nsplit partial slots of the K.V kernel (pitch
// rows_pad) and d_r = dvec[r] (per-row noise) or noise.  A kernel sum scales slot s by the outputscale pscale[s] of the term
// that owns it instead of os.  poison is NaN when the packed inputs held a non-finite value (K.V is NaN in the reference), else 0.
__device__ __forceinline__ float4 khat_row(const float* __restrict__ kpart, int nsplit, int64_t rows_pad, float os,
                                           const float* __restrict__ pscale, float poison, const float* __restrict__ X,
                                           const float* __restrict__ dvec, float noise, int64_t r, int cg) {
  float4 s = make_float4(poison, poison, poison, poison);
  float osr = os;
  if (pscale) {
    for (int sp = 0; sp < nsplit; ++sp) {
      const float4 a = reinterpret_cast<const float4*>(kpart)[((int64_t)sp * rows_pad + r) * 4 + cg];
      const float w = pscale[sp];
      s.x = fmaf(w, a.x, s.x); s.y = fmaf(w, a.y, s.y); s.z = fmaf(w, a.z, s.z); s.w = fmaf(w, a.w, s.w);
    }
    osr = 1.f;
  } else {
    for (int sp = 0; sp < nsplit; ++sp) {
      const float4 a = reinterpret_cast<const float4*>(kpart)[((int64_t)sp * rows_pad + r) * 4 + cg];
      s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
    }
  }
  const float4 x = reinterpret_cast<const float4*>(X)[r * 4 + cg];
  const float d = dvec ? dvec[r] : noise;
  return make_float4(fmaf(d, x.x, osr * s.x), fmaf(d, x.y, osr * s.y), fmaf(d, x.z, osr * s.z), fmaf(d, x.w, osr * s.w));
}
#endif

// Host side of a solver loop that never synchronises inside: after iteration kk is enqueued, the device done flag is copied
// into a two-entry pinned ring and an event is recorded; the host then waits only for iteration kk - 1, so the GPU always
// has one iteration queued.  Polling starts at iteration first_poll (earlier iterations cannot stop).
class SolverLoop {
 public:
  SolverLoop(gp_plan* p, const char* name, const int* d_done, int first_poll)
      : st_(p->stream), name_(name), d_done_(d_done), h_done_(reinterpret_cast<int*>(static_cast<char*>(p->pinned) + PIN_DONE_RING)),
        first_(first_poll) {}
  SolverLoop(const SolverLoop&) = delete;
  SolverLoop& operator=(const SolverLoop&) = delete;
  ~SolverLoop() {
    for (cudaEvent_t e : ev_)
      if (e) cudaEventDestroy(e);
  }
  int create_events() {
    for (cudaEvent_t& e : ev_) GP_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    return GP_OK;
  }
  // call once iteration kk has been enqueued: true when iteration kk - 1 set the done flag
  bool finished(int kk) {
    if (kk < first_) return false;
    cudaMemcpyAsync(&h_done_[kk & 1], d_done_, sizeof(int), cudaMemcpyDeviceToHost, st_);
    cudaEventRecord(ev_[kk & 1], st_);
    if (kk == first_) return false;
    cudaEventSynchronize(ev_[(kk - 1) & 1]);
    return h_done_[(kk - 1) & 1] != 0;
  }
  // after the loop: a launch error fails the run unless the loop already failed
  int launch_status(int status) const {
    const cudaError_t le = cudaGetLastError();
    if (status == GP_OK && le != cudaSuccess) {
      set_error("%s launch failed: %s", name_, cudaGetErrorString(le));
      return GP_E_CUDA;
    }
    return status;
  }
  // waits for the stream; an execution error fails the run
  int sync() const {
    const cudaError_t se = cudaStreamSynchronize(st_);
    if (se != cudaSuccess) {
      set_error("%s execution failed: %s", name_, cudaGetErrorString(se));
      return GP_E_CUDA;
    }
    return GP_OK;
  }

 private:
  cudaStream_t st_;
  const char* name_;
  const int* d_done_;
  int* h_done_;
  int first_;
  cudaEvent_t ev_[2] = {nullptr, nullptr};
};

}  // namespace gp
