// kron.cu -- Kronecker multitask operator  (s K_data) (x) B  (MultitaskKernel, kernels/multitask_kernel.py:13-61: the reference
// builds KroneckerProductLinearOperator(covar_x, covar_i) over interleaved rows i T + a; examples/03_Multitask_Exact_GPs/
// Multitask_GP_Regression.ipynb).
//
// Products.  With V [N2 T, t] viewed as V_j[b, c] = V[j T + b, c],
//     ((K (x) B) V)[i T + a, c] = sum_j K[i, j] W[j, a t + c],   W[j, a t + c] = sum_b B[a, b] V[j T + b, c],
// so one product is one B-mix pass into ceil(T t / 16) zero-padded [N2, 16] column chunks of W (the data plan's V16 layout),
// one launch of the data plan's UNCHANGED fused kernel (kmv_tc.cu / kmv_simt.cu) per chunk into that chunk's partial slots, and
// one scatter pass that sums each chunk's slots in a fixed order into rows i T + a of the parent's partial slot 0.  The parent's
// finish kernels (outputscale, noise or noise diagonal, done flag) and every solver then run as on a plain plan of N T rows.  The
// kernel is evaluated on N1 x N2 pairs per chunk instead of the (N1 T) x (N2 T) pairs of the same operator in Hadamard form.
//
// Gradients.  sum L . ((d(sK) (x) B) R) is the data plan's bilinear derivative with L viewed as [N1, T t] and R mixed by B, run
// chunk by chunk.  dB[a][b] = s sum_i L[i T + a] . (K R_b)[i] with R_b[j] = R[j T + b] is the data kernel over the unmixed chunks,
// reduced in fp64 in a fixed tree.  Nothing here uses atomics: repeated calls on one plan give identical bits.
#include <math.h>

#include <algorithm>
#include <cmath>

#include "gp_common.cuh"

namespace gp {

constexpr int KRON_RED_ROWS = 2048;   // points per block of the dB reduction

// W[q][j][cc] = sum_b B[a][b] V16[j T + b][c] for the column col = 16 q + cc = a t + c (B == nullptr: V16[j T + a][c], the
// unmixed chunks); zero for col >= T t and for the padding rows j >= n
__global__ void kron_mix_kernel(const float* __restrict__ V16, int64_t n, int64_t npad, int T, int t, int nchunk,
                                const float* __restrict__ B, float* __restrict__ W, const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)nchunk * npad * TP) return;
  const int cc = (int)(idx % TP);
  const int64_t j = (idx / TP) % npad;
  const int q = (int)(idx / ((int64_t)TP * npad));
  const int col = q * TP + cc;
  float s = 0.f;
  if (j < n && col < T * t) {
    const int a = col / t, c = col % t;
    const float* v = V16 + j * T * TP + c;
    if (B) {
      const float* br = B + a * T;
      for (int b = 0; b < T; ++b) s = fmaf(br[b], v[b * TP], s);
    } else {
      s = v[a * TP];
    }
  }
  W[idx] = s;
}

// out[(i T + a)][c] = sum_sp part[q][sp][i][cc] for col = a t + c = 16 q + cc (c < t), 0 for c >= t; NaN for non-finite inputs or
// a non-finite B (the fused kernels' clamps and operand splits need not carry a NaN of the mixed block through)
__global__ void kron_scatter_kernel(const float* __restrict__ part, int nsplit, int64_t rows_pad, int64_t n1, int T, int t,
                                    float* __restrict__ out, const int* __restrict__ xbad, int bbad, const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n1 * T * TP) return;
  const int c = (int)(idx % TP);
  const int64_t r = idx / TP;
  const int64_t i = r / T;
  const int a = (int)(r % T);
  float s = 0.f;
  if (c < t) {
    const int col = a * t + c;
    const float* base = part + ((int64_t)(col / TP) * nsplit * rows_pad + i) * TP + col % TP;
    for (int sp = 0; sp < nsplit; ++sp) s += base[(int64_t)sp * rows_pad * TP];
  }
  if (bbad || *xbad) s = __int_as_float(0x7fc00000);
  out[idx] = s;
}

// dB reduction: block (z, a T + b) writes red[(z T + a) T + b] = sum over points i of chunk z and c < t of
// L16[i T + a][c] * P[i][b t + c], P = the data kernel's product of the unmixed chunks (slots summed in a fixed order)
__global__ void __launch_bounds__(256)
kron_dB_kernel(const float* __restrict__ part, int nsplit, int64_t rows_pad, const float* __restrict__ L16, int64_t n1, int T, int t,
               double* __restrict__ red, const int* __restrict__ xbad) {
  __shared__ double sh[256];
  const int z = blockIdx.x, ab = blockIdx.y, tid = threadIdx.x;
  const int a = ab / T, b = ab % T;
  const int64_t i0 = (int64_t)z * KRON_RED_ROWS, i1 = min(n1, i0 + KRON_RED_ROWS);
  double acc = 0.0;
  for (int64_t e = i0 * t + tid; e < i1 * t; e += 256) {
    const int64_t i = e / t;
    const int c = (int)(e % t);
    const int col = b * t + c;
    const float* base = part + ((int64_t)(col / TP) * nsplit * rows_pad + i) * TP + col % TP;
    float pv = 0.f;
    for (int sp = 0; sp < nsplit; ++sp) pv += base[(int64_t)sp * rows_pad * TP];
    acc += (double)L16[(i * T + a) * TP + c] * (double)pv;
  }
  sh[tid] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) sh[tid] += sh[tid + s];
    __syncthreads();
  }
  if (tid == 0) red[(int64_t)z * T * T + ab] = *xbad ? __longlong_as_double(0x7ff8000000000000LL) : sh[0];
}

// point index of every requested row (-1 outside [0, n1 T): the data plan returns a NaN row for it)
__global__ void kron_point_idx_kernel(const int64_t* __restrict__ idx, int64_t m, int T, int64_t n, int64_t* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const int64_t v = idx[r];
  out[r] = (v >= 0 && v < n) ? v / T : -1;
}

// OUT[r][j T + b] = rows[r][j] B[a][b], a = idx[r] mod T: row i T + a of (s K) (x) B from row i of s K
__global__ void kron_expand_rows_kernel(const float* __restrict__ rows, int64_t n2, const int64_t* __restrict__ idx, int64_t n,
                                        const float* __restrict__ B, int T, float* __restrict__ OUT, int64_t ldo) {
  const int64_t r = blockIdx.y;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n2 * T) return;
  const int64_t v = idx[r];
  const int a = (v >= 0 && v < n) ? (int)(v % T) : 0;
  OUT[r * ldo + e] = rows[r * n2 + e / T] * B[a * T + (int)(e % T)];
}

// OUT[i T + a] = d[i] B[a][a]
__global__ void kron_expand_diag_kernel(const float* __restrict__ d, int64_t n1, const float* __restrict__ B, int T, float* __restrict__ OUT) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n1 * T) return;
  const int a = (int)(e % T);
  OUT[e] = d[e / T] * B[a * T + a];
}

static int kron_check_data(const gp_plan* p, const gp_plan* q) {
  GP_REQUIRE(q->data_set && q->hypers_set, GP_E_STATE, "Kronecker plan: the data plan needs set_data + set_hypers");
  GP_REQUIRE(q->backend == GP_BACKEND_TCGEN05 || q->backend == GP_BACKEND_SIMT, GP_E_SHAPE,
             "Kronecker plan: the data plan must be a plain kernel plan (not SKI, not a kernel sum, not Kronecker)");
  GP_REQUIRE(q->tasks == nullptr, GP_E_STATE, "Kronecker plan: a data plan with task indices is not available");
  GP_REQUIRE(q->lr_U == nullptr, GP_E_STATE, "Kronecker plan: a data plan with a low-rank correction is not available");
  GP_REQUIRE(q->row_begin == 0 && q->row_count == q->n1 && !(q->comm && q->comm->world > 1), GP_E_SHAPE,
             "Kronecker plan: a row-sharded data plan is not available");
  GP_REQUIRE(q->device == p->device && q->stream == p->stream, GP_E_STATE, "Kronecker plan: the data plan must live on the same device and stream");
  GP_REQUIRE(q->n1 * p->kron->T < ((int64_t)1 << 31) && q->n2 * p->kron->T < ((int64_t)1 << 31), GP_E_SHAPE,
             "Kronecker plan: N T must stay below 2^31");
  return GP_OK;
}

// operator geometry from the data plan: N1 T x N2 T rows, one partial slot
static void kron_geometry(gp_plan* p) {
  const gp_plan* q = p->kron->data;
  const int T = p->kron->T;
  p->backend = GP_BACKEND_KRON;
  p->n1 = q->n1 * T;
  p->n2 = q->n2 * T;
  p->same = q->same;
  p->d = q->d;
  p->row_begin = 0;
  p->row_count = p->n1;
  p->rows_pad = cdiv(p->row_count, 2 * TILE_I) * 2 * TILE_I;
  p->ntile_i = p->rows_pad / TILE_I;
  p->ntile_j = cdiv(p->n2, TILE_J);
  p->DP = q->DP;
  p->KP = q->KP;
  p->nsplit = 1;
  p->nparts = 1;
}

int kron_refresh(gp_plan* p) {
  gp_kron_state* ks = p->kron;
  const gp_plan* q = ks->data;
  GP_CHECK(kron_check_data(p, q));
  GP_REFUSE_RQ(q, "a Kronecker operator (as the data plan)");
  GP_REFUSE_POLY(q, "a Kronecker operator (as the data plan)");
  GP_REQUIRE(p->n1 == q->n1 * ks->T && p->n2 == q->n2 * ks->T && p->same == q->same, GP_E_STATE,
             "Kronecker plan: the data plan changed its size; call gp_plan_set_kron again");
  p->kind = q->kind;
  p->outputscale = q->outputscale;   // the finish kernels scale the unscaled product by the data plan's s
  p->xbad = q->xbad;
  return GP_OK;
}

int kron_pack(gp_plan* p) {
  GP_CHECK(kron_check_data(p, p->kron->data));
  kron_geometry(p);
  GP_CHECK(kron_refresh(p));
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  return GP_OK;
}

// W-chunk pitch of the data plan: whole 64-row tiles on the tensor-core path (one pack call covers every chunk)
static int64_t kron_npad(const gp_plan* q) { return q->backend == GP_BACKEND_TCGEN05 ? q->ntile_j * TILE_J : q->n2; }

// V16 [N2 T][16] with t live columns, mixed by B (or not: B == nullptr) -> nchunk data-kernel products in ks->part
static int kron_chunks(gp_plan* p, const float* V16, int t, const float* B, int kind, const int* done_flag, int* nchunk_out) {
  gp_kron_state* ks = p->kron;
  gp_plan* q = ks->data;
  const bool tc = q->backend == GP_BACKEND_TCGEN05;
  const int T = ks->T;
  const int nchunk = (int)cdiv((int64_t)T * t, TP);
  const int64_t npad = kron_npad(q);
  const size_t slot_floats = (size_t)q->rows_pad * TP;
  GP_CHECK(ks->W.ensure(sizeof(float) * (size_t)nchunk * npad * TP));
  GP_CHECK(ks->part.ensure(sizeof(float) * (size_t)nchunk * q->nsplit * slot_floats));
  const int64_t tot = (int64_t)nchunk * npad * TP;
  kron_mix_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, p->stream>>>(V16, q->n2, npad, T, t, nchunk, B, ks->W.as<float>(), done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  if (tc) {
    GP_CHECK(ks->Vt.ensure(sizeof(float) * (size_t)nchunk * q->ntile_j * V_TILE_FLOATS));
    GP_CHECK(pack_v_tiles_rows(p, ks->W.as<float>(), (int64_t)nchunk * npad, (int64_t)nchunk * q->ntile_j, ks->Vt.as<float>()));
  }
  for (int c = 0; c < nchunk; ++c) {
    float* part = ks->part.as<float>() + (size_t)c * q->nsplit * slot_floats;
    if (tc) {
      GP_CHECK(kmv_tc_launch_cols(q, kind, q->XA.as<float>(), q->XB.as<float>(), ks->Vt.as<float>() + (size_t)c * q->ntile_j * V_TILE_FLOATS,
                                  part, q->ntile_j, q->tiles_per_split, q->nsplit, q->row_begin, done_flag));
    } else {
      const float* Z1 = q->same ? q->Z2.as<float>() : q->Z1.as<float>();
      GP_CHECK(kmv_simt_launch_cols(q, kind, Z1, q->Z2.as<float>(), ks->W.as<float>() + (size_t)c * npad * TP, part, q->n2,
                                    q->tiles_per_split * SIMT_TJ, q->nsplit, q->row_begin, done_flag));
    }
    p->launches++;
  }
  *nchunk_out = nchunk;
  return GP_OK;
}

int kron_kmv_partials(gp_plan* p, const float* V16, const int* done_flag) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CHECK(kron_refresh(p));
  const gp_plan* q = ks->data;
  const int t = p->kron_cols;
  int nchunk = 0;
  GP_CHECK(kron_chunks(p, V16, t, ks->Bd.as<float>(), q->kind, done_flag, &nchunk));
  kron_scatter_kernel<<<(unsigned)cdiv(p->n1 * TP, 256), 256, 0, p->stream>>>(ks->part.as<float>(), q->nsplit, q->rows_pad, q->n1, ks->T, t,
                                                                             p->partial.as<float>(), q->xbad, ks->b_bad ? 1 : 0, done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int kron_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "rows of a Kronecker plan: at most 65535 rows per call (m=%lld)", (long long)m);
  GP_CHECK(kron_refresh(p));
  gp_plan* q = ks->data;
  GP_CHECK(ks->idx.ensure(sizeof(int64_t) * m));
  GP_CHECK(ks->rows.ensure(sizeof(float) * (size_t)m * q->n2));
  kron_point_idx_kernel<<<(unsigned)cdiv(m, 256), 256, 0, p->stream>>>(idx, m, ks->T, p->n1, ks->idx.as<int64_t>());
  p->launches++;
  GP_CHECK(gp_krows(q, ks->idx.as<int64_t>(), m, ks->rows.as<float>(), q->n2));
  kron_expand_rows_kernel<<<dim3((unsigned)cdiv(p->n2, 256), (unsigned)m), 256, 0, p->stream>>>(ks->rows.as<float>(), q->n2, idx, p->n1,
                                                                                             ks->Bd.as<float>(), ks->T, OUT, ldo);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int kron_kdiag(gp_plan* p, float* OUT) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CHECK(kron_refresh(p));
  gp_plan* q = ks->data;
  GP_CHECK(ks->rows.ensure(sizeof(float) * q->n1));
  GP_CHECK(gp_kdiag(q, ks->rows.as<float>()));
  kron_expand_diag_kernel<<<(unsigned)cdiv(p->n1, 256), 256, 0, p->stream>>>(ks->rows.as<float>(), q->n1, ks->Bd.as<float>(), ks->T, OUT);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// lengthscale(s) and outputscale: the data plan's bilinear derivative over chunk pairs (L unmixed, R mixed by B), summed in order
int kron_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CHECK(kron_refresh(p));
  gp_plan* q = ks->data;
  const int T = ks->T;
  const int nls = (int)q->ls.size();
  std::vector<double> gl(nls, 0.0), tot(nls, 0.0);
  double go = 0.0, tot_os = 0.0;
  GP_CHECK(p->misc2.ensure(sizeof(float) * p->n1 * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * p->n2 * TP));
  for (int c0 = 0; c0 < s; c0 += TP) {
    const int tc = std::min(TP, s - c0);
    GP_CHECK(to_v16(p, L + c0, ldl, tc, p->n1, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, R + c0, ldr, tc, p->n2, p->misc3.as<float>()));
    const int nchunk = (int)cdiv((int64_t)T * tc, TP);
    GP_CHECK(ks->Lw.ensure(sizeof(float) * (size_t)nchunk * q->n1 * TP));
    GP_CHECK(ks->W.ensure(sizeof(float) * (size_t)nchunk * q->n2 * TP));
    kron_mix_kernel<<<(unsigned)cdiv((int64_t)nchunk * q->n1 * TP, 256), 256, 0, p->stream>>>(p->misc2.as<float>(), q->n1, q->n1, T, tc, nchunk,
                                                                                             nullptr, ks->Lw.as<float>(), nullptr);
    kron_mix_kernel<<<(unsigned)cdiv((int64_t)nchunk * q->n2 * TP, 256), 256, 0, p->stream>>>(p->misc3.as<float>(), q->n2, q->n2, T, tc, nchunk,
                                                                                             ks->Bd.as<float>(), ks->W.as<float>(), nullptr);
    p->launches += 2;
    GP_CUDA(cudaGetLastError());
    for (int c = 0; c < nchunk; ++c) {
      GP_CHECK(gp_bilinear_grad(q, ks->Lw.as<float>() + (size_t)c * q->n1 * TP, TP, ks->W.as<float>() + (size_t)c * q->n2 * TP, TP, TP,
                                gl.data(), &go));
      for (int e = 0; e < nls; ++e) tot[e] += gl[e];
      tot_os += go;
    }
  }
  for (int e = 0; e < nls; ++e) grad_ls[e] = ks->b_bad ? NAN : tot[e];
  *grad_os = ks->b_bad ? NAN : tot_os;
  return GP_OK;
}

static int kron_task_covar_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(t >= 1 && L && R && dB, GP_E_SHAPE, "gp_task_covar_grad: bad arguments");
  GP_REQUIRE((ldl >= t || p->n1 == 1) && (ldr >= t || p->n2 == 1), GP_E_SHAPE,
             "gp_task_covar_grad: leading dimensions must be >= t (ldl=%lld, ldr=%lld, t=%d)", (long long)ldl, (long long)ldr, t);
  GP_CHECK(kron_refresh(p));
  gp_plan* q = ks->data;
  const int T = ks->T;
  const int nz = (int)cdiv(q->n1, KRON_RED_ROWS);
  GP_CHECK(p->misc2.ensure(sizeof(float) * p->n1 * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * p->n2 * TP));
  GP_CHECK(ks->red.ensure(sizeof(double) * (size_t)nz * T * T));
  std::vector<double> acc((size_t)T * T, 0.0), h((size_t)nz * T * T);
  for (int c0 = 0; c0 < t; c0 += TP) {
    const int tc = std::min(TP, t - c0);
    GP_CHECK(to_v16(p, L + c0, ldl, tc, p->n1, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, R + c0, ldr, tc, p->n2, p->misc3.as<float>()));
    int nchunk = 0;
    GP_CHECK(kron_chunks(p, p->misc3.as<float>(), tc, nullptr, q->kind, nullptr, &nchunk));
    kron_dB_kernel<<<dim3((unsigned)nz, (unsigned)(T * T)), 256, 0, p->stream>>>(ks->part.as<float>(), q->nsplit, q->rows_pad,
                                                                                p->misc2.as<float>(), q->n1, T, tc, ks->red.as<double>(), q->xbad);
    p->launches++;
    GP_CUDA(cudaGetLastError());
    GP_CUDA(cudaMemcpyAsync(h.data(), ks->red.as<double>(), sizeof(double) * h.size(), cudaMemcpyDeviceToHost, p->stream));
    GP_CUDA(cudaStreamSynchronize(p->stream));
    for (int z = 0; z < nz; ++z)
      for (int e = 0; e < T * T; ++e) acc[(size_t)e] += h[(size_t)z * T * T + e];
  }
  for (int e = 0; e < T * T; ++e) dB[e] = (double)q->outputscale * acc[(size_t)e];
  return GP_OK;
}

static void kron_release(gp_plan* p) {
  gp_kron_state* ks = p->kron;
  gp::DevBuf* bufs[] = {&ks->Bd, &ks->W, &ks->Vt, &ks->part, &ks->Lw, &ks->red, &ks->idx, &ks->rows};
  for (auto* b : bufs) b->release();
  delete ks;
  p->kron = nullptr;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_kron(gp_plan* p, gp_plan* data, int T) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_CUDA(cudaSetDevice(p->device));
  if (data == nullptr) {
    if (p->kron) {
      GP_CUDA(cudaStreamSynchronize(p->stream));
      kron_release(p);
      p->backend_req = GP_BACKEND_AUTO;
      p->backend = GP_BACKEND_SIMT;
      p->data_set = false;   // the rows belonged to the data plan: gp_plan_set_data again
    }
    return GP_OK;
  }
  GP_REQUIRE(T >= 1 && T <= 32, GP_E_SHAPE, "number of tasks T=%d not in [1, 32]", T);
  GP_REQUIRE(data != p, GP_E_STATE, "a Kronecker plan cannot be its own data plan");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "a SKI plan cannot become a Kronecker plan");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel-sum plan cannot become a Kronecker plan");
  GP_REFUSE_TASKS(p, "gp_plan_set_kron");
  GP_REFUSE_LOWRANK(p, "gp_plan_set_kron");
  GP_REFUSE_DERIV(p, "gp_plan_set_kron");
  GP_REFUSE_PRODUCT(p, "gp_plan_set_kron");
  if (data) GP_REFUSE_PRODUCT(data, "gp_plan_set_kron (as the data plan)");
  GP_REFUSE_ADDITIVE(p, "gp_plan_set_kron");
  GP_REFUSE_SPECTRAL(p, "gp_plan_set_kron");
  if (data) GP_REFUSE_ADDITIVE(data, "gp_plan_set_kron (as the data plan)");
  if (data) GP_REFUSE_SPECTRAL(data, "gp_plan_set_kron (as the data plan)");
  GP_REFUSE_PERIODIC(p, "gp_plan_set_kron");
  if (data) GP_REFUSE_PERIODIC(data, "gp_plan_set_kron (as the data plan)");
  GP_REFUSE_RQ(p, "gp_plan_set_kron");
  if (data) GP_REFUSE_RQ(data, "gp_plan_set_kron (as the data plan)");
  GP_REFUSE_POLY(p, "gp_plan_set_kron");
  if (data) GP_REFUSE_POLY(data, "gp_plan_set_kron (as the data plan)");
  GP_REQUIRE(!(p->comm && p->comm->world > 1), GP_E_SHAPE, "a Kronecker plan is not available on a row-sharded plan");
  gp_kron_state* ks = p->kron ? p->kron : new gp_kron_state();
  const bool keep_b = p->kron && ks->T == T && ks->b_set;
  gp_plan* old = ks->data;
  const int oldT = ks->T;
  ks->data = data;
  ks->T = T;
  p->kron = ks;
  const int st = kron_check_data(p, data);
  if (st != GP_OK) {
    if (old) { ks->data = old; ks->T = oldT; }
    else kron_release(p);
    return st;
  }
  if (!keep_b) ks->b_set = false;
  p->backend_req = GP_BACKEND_KRON;
  kron_geometry(p);
  p->data_set = true;
  return p->hypers_set ? kron_pack(p) : GP_OK;   // without the noise yet: packed by gp_plan_set_hypers
}

// gp_plan_set_task_covar / gp_task_covar_grad on a Kronecker plan (tasks.cu forwards them here)
int gp::kron_set_task_covar(gp_plan* p, const float* B, int T) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(B != nullptr && T == ks->T, GP_E_SHAPE, "task covariance must be %d x %d (got T=%d)", ks->T, ks->T, T);
  GP_CUDA(cudaSetDevice(p->device));
  ks->B.assign(B, B + (size_t)T * T);
  ks->b_bad = false;
  for (float v : ks->B) ks->b_bad = ks->b_bad || !std::isfinite(v);
  GP_CHECK(ks->Bd.ensure(sizeof(float) * T * T));
  GP_CUDA(cudaMemcpyAsync(ks->Bd.p, ks->B.data(), sizeof(float) * T * T, cudaMemcpyHostToDevice, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));   // the next call may replace ks->B
  ks->b_set = true;
  return GP_OK;
}

int gp::kron_task_covar_grad_checked(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB) {
  GP_REQUIRE(p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(p->kron->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CUDA(cudaSetDevice(p->device));
  return kron_task_covar_grad(p, L, ldl, R, ldr, t, dB);
}
