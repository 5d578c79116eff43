// api.cu -- C-ABI entry points of libgpbbmm.so (see include/gp_bbmm.h for the reference interface each replaces).
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include <algorithm>

#include "gp_common.cuh"

namespace gp {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

uint32_t plan_settings(const gp_plan* p) {
  return (p->lr_U ? PS_LOWRANK : 0u) | (p->tasks ? PS_TASKS : 0u) | (p->kron ? PS_KRON : 0u) | (p->deriv ? PS_DERIV : 0u) |
         (p->backend_req == GP_BACKEND_PRODUCT ? PS_PRODUCT : 0u) | (p->add_M ? PS_ADDITIVE : 0u) | (p->sm_Q ? PS_SPECTRAL : 0u) |
         (p->per_n ? PS_PERIODIC : 0u) | (p->kind == GP_RQ ? PS_RQ : 0u) | (p->kind == GP_POLY ? PS_POLY : 0u);
}

int refuse_settings(const gp_plan* p, CallId call) {
  const CallRow& c = CALL_ROWS[call];
  const uint32_t hit = plan_settings(p) & c.refuses;
  if (hit == 0) return GP_OK;
  const SettingName& s = SETTING_NAMES[__builtin_ctz(hit)];   // the first refused setting in check order
  if (c.as)
    set_error("%s: %s as a %s is not available (%s)", c.name, s.noun, c.as, s.setter);
  else
    set_error("%s is not available on %s (%s)", c.name, s.noun, s.setter);
  return GP_E_STATE;
}

__global__ void concat_rhs_kernel(const float* __restrict__ probes, int tp, const float* __restrict__ y, int64_t n,
                                  float* __restrict__ rhs, float* __restrict__ pn_part) {
  // rhs[r][0..tp) = probes (normalised later), rhs[r][tp] = y
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * (tp + 1)) return;
  int64_t r = idx / (tp + 1);
  int c = (int)(idx % (tp + 1));
  rhs[idx] = (c < tp) ? probes[r * tp + c] : y[r];
}

// inv_quad partial: sum_r solves[r][tp] * y[r]
__global__ void invquad_kernel(const float* __restrict__ solves, int ld, int col, const float* __restrict__ y, int64_t n,
                               double* __restrict__ part) {
  __shared__ double sh[256];
  double acc = 0.0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
    acc += (double)solves[r * ld + col] * (double)y[r];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}

__global__ void extract_col_kernel(const float* __restrict__ solves, int ld, int col, int64_t n, float* __restrict__ out) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) out[r] = solves[r * ld + col];
}

}  // namespace gp

using namespace gp;

extern "C" const char* gp_version(void) { return "gpbbmm 0.1 (sm_90a; wgmma 3xTF32 fused K.V, device mBCG, pivoted-Cholesky precond, SLQ)"; }
extern "C" const char* gp_last_error(void) { return g_err; }
extern "C" const char* gp_status_string(int s) {
  switch (s) {
    case GP_OK: return "ok";
    case GP_E_SHAPE: return "shape / unsupported configuration";
    case GP_E_CUDA: return "CUDA error";
    case GP_E_NAN_MVM: return "NaNs encountered when trying to perform matrix-vector multiplication";
    case GP_W_NOT_CONVERGED: return "CG did not converge";
    case GP_W_PIVCHOL_NAN: return "NaNs encountered in preconditioner computation";
    case GP_E_NCCL: return "NCCL error";
    case GP_E_STATE: return "call order violated";
    case GP_W_EIG_NOT_CONVERGED: return "tridiagonal eigen-solver did not converge";
  }
  return "unknown";
}

extern "C" int gp_plan_create(gp_plan** out, int device, void* stream) {
  GP_REQUIRE(out != nullptr, GP_E_SHAPE, "null out pointer");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error("libgpbbmm needs a CUDA device (sm_90a); there is no CPU fallback: %s", cudaGetErrorString(e));
    return GP_E_CUDA;
  }
  GP_REQUIRE(device >= 0 && device < ndev, GP_E_SHAPE, "device %d out of range", device);
  GP_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  GP_CUDA(cudaGetDeviceProperties(&prop, device));
  GP_REQUIRE(prop.major == 9 && prop.minor == 0, GP_E_CUDA, "libgpbbmm is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
  gp_plan* p = new gp_plan();
  p->device = device;
  p->stream = reinterpret_cast<cudaStream_t>(stream);
  p->n_sm = prop.multiProcessorCount;
  GP_CUDA(cudaMallocHost(&p->pinned, PINNED_BYTES));
  memset(p->pinned, 0, PINNED_BYTES);
  *out = p;
  return GP_OK;
}

extern "C" int gp_plan_destroy(gp_plan* p) {
  if (!p) return GP_OK;
  cudaSetDevice(p->device);
  cudaStreamSynchronize(p->stream);
  gp::DevBuf* bufs[] = {&p->mean, &p->scale, &p->Z1, &p->Z2, &p->XA, &p->XB, &p->V16, &p->Vtiles, &p->partial, &p->out16,
                        &p->cgU, &p->cgR, &p->cgZ, &p->cgP, &p->cgV, &p->cgPfull, &p->red, &p->sums, &p->qtr, &p->state,
                        &p->tmat_tmp, &p->misc, &p->misc2, &p->misc3, &p->pcdiag, &p->pcperm, &p->pcpos, &p->pcstate,
                        &p->pcpart, &p->gram, &p->cholC, &p->part_scale, &p->msw, &p->lrw};
  for (auto* b : bufs) b->release();
  if (p->ski) {
    gp::DevBuf* sb[] = {&p->ski->first, &p->ski->wts, &p->ski->gridA, &p->ski->gridB, &p->ski->gridC, &p->ski->gridD, &p->ski->T, &p->ski->dT, &p->ski->flag,
                        &p->ski->perm, &p->ski->tile_off, &p->ski->tile_cnt, &p->ski->first_s, &p->ski->wts_s,
                        &p->ski->tcol, &p->ski->dtcol, &p->ski->band};
    for (auto* b : sb) b->release();
    delete p->ski;
  }
  if (p->tasks) {
    p->data_set = false;   // release only, no re-pack
    gp_plan_set_tasks(p, nullptr, nullptr, 0);
  }
  if (p->kron) gp_plan_set_kron(p, nullptr, 0);   // the data plan stays the caller's
  if (p->deriv) gp_plan_set_deriv(p, nullptr);
  if (p->pinned) cudaFreeHost(p->pinned);
  delete p;
  return GP_OK;
}

extern "C" int gp_plan_set_backend(gp_plan* p, int backend) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(backend >= GP_BACKEND_AUTO && backend <= GP_BACKEND_SIMT, GP_E_SHAPE, "bad backend %d", backend);
  GP_REQUIRE(p->backend != GP_BACKEND_SKI, GP_E_STATE, "the SKI backend is selected by gp_plan_set_ski");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel sum runs the backends of its terms");
  GP_REQUIRE(p->kron == nullptr, GP_E_STATE, "a Kronecker plan runs the backend of its data plan");
  GP_CHECK(refuse_settings(p, CALL_SET_BACKEND));
  p->backend_req = backend;
  if (p->data_set && p->hypers_set) return pack_inputs(p);
  return GP_OK;
}

extern "C" int gp_plan_set_data(gp_plan* p, const float* X1, int64_t n1, int64_t ld1, const float* X2, int64_t n2,
                                int64_t ld2, int d, int64_t row_begin, int64_t row_count) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(p->kron == nullptr, GP_E_STATE, "a Kronecker plan takes its rows from its data plan (gp_plan_set_kron)");
  GP_REQUIRE(p->deriv == nullptr, GP_E_STATE, "a derivative plan takes its rows from its data plan (gp_plan_set_deriv)");
  GP_REQUIRE(X1 != nullptr && n1 >= 1 && d >= 1 && ld1 >= d, GP_E_SHAPE, "bad X1 shape n1=%lld d=%d ld1=%lld", (long long)n1, d, (long long)ld1);
  GP_CUDA(cudaSetDevice(p->device));
  // task indices belong to the rows they were set for: new data drops them (gp_plan_set_tasks again)
  if (p->tasks) {
    p->data_set = false;   // no re-pack of the old layout on the way out
    GP_CHECK(gp_plan_set_tasks(p, nullptr, nullptr, 0));
  }
  p->X1 = X1; p->n1 = n1; p->ld1 = ld1; p->d = d;
  p->same = (X2 == nullptr) || (X2 == X1 && n2 == n1 && ld2 == ld1);
  if (p->same) { p->X2 = X1; p->n2 = n1; p->ld2 = ld1; }
  else {
    GP_REQUIRE(n2 >= 1 && ld2 >= d, GP_E_SHAPE, "bad X2 shape");
    p->X2 = X2; p->n2 = n2; p->ld2 = ld2;
  }
  if (row_count <= 0) { row_begin = 0; row_count = n1; }
  GP_REQUIRE(row_begin >= 0 && row_begin + row_count <= n1, GP_E_SHAPE, "row shard [%lld,+%lld) outside n1=%lld",
             (long long)row_begin, (long long)row_count, (long long)n1);
  GP_REQUIRE(p->same || (row_begin == 0 && row_count == n1), GP_E_SHAPE, "row sharding needs X2 == X1");
  p->row_begin = row_begin; p->row_count = row_count;
  p->data_set = true;
  if (p->hypers_set) {
    GP_REQUIRE(p->ls.size() == 1 || (int)p->ls.size() == d, GP_E_SHAPE, "lengthscale count does not match d");
    return pack_inputs(p);
  }
  return GP_OK;
}

extern "C" int gp_plan_set_hypers(gp_plan* p, int kind, const float* lengthscale, int n_ls, float outputscale, float noise) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(kind != GP_RQ, GP_E_SHAPE, "the rational quadratic kind takes alpha: call gp_plan_set_hypers_rq");
  GP_REQUIRE(kind != GP_POLY, GP_E_SHAPE, "the polynomial kind takes a power and an offset: call gp_plan_set_hypers_poly");
  GP_REQUIRE(kind >= GP_RBF && kind <= GP_MATERN52, GP_E_SHAPE, "nu expected to be 0.5, 1.5, or 2.5 (kind=%d)", kind);
  GP_REQUIRE(lengthscale && n_ls >= 1, GP_E_SHAPE, "lengthscale missing");
  GP_REQUIRE(!p->data_set || n_ls == 1 || n_ls == p->d, GP_E_SHAPE, "lengthscale count %d does not match d=%d", n_ls, p->d);
  for (int i = 0; i < n_ls; ++i)
    GP_REQUIRE(lengthscale[i] > 0.f && isfinite(lengthscale[i]), GP_E_SHAPE, "lengthscale[%d]=%g must be positive", i, lengthscale[i]);
  GP_REQUIRE(outputscale > 0.f && noise >= 0.f, GP_E_SHAPE, "outputscale must be > 0 and noise >= 0");
  GP_REQUIRE(p->per_n == 0 || kind == GP_RBF, GP_E_STATE, "gp_plan_set_hypers on a periodic plan (gp_plan_set_periodic) takes the kind GP_RBF (got %d)", kind);
  GP_CUDA(cudaSetDevice(p->device));
  p->kind = kind;
  p->ls.assign(lengthscale, lengthscale + n_ls);
  p->outputscale = outputscale;
  p->noise = noise;
  p->hypers_set = true;
  if (p->data_set) return pack_inputs(p);
  return GP_OK;
}

extern "C" int gp_plan_set_hypers_rq(gp_plan* p, const float* lengthscale, int n_ls, float alpha, float outputscale, float noise) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(lengthscale && n_ls >= 1, GP_E_SHAPE, "lengthscale missing");
  GP_REQUIRE(!p->data_set || n_ls == 1 || n_ls == p->d, GP_E_SHAPE, "lengthscale count %d does not match d=%d", n_ls, p->d);
  for (int i = 0; i < n_ls; ++i)
    GP_REQUIRE(lengthscale[i] > 0.f && isfinite(lengthscale[i]), GP_E_SHAPE, "lengthscale[%d]=%g must be positive", i, lengthscale[i]);
  GP_REQUIRE(alpha > 0.f && isfinite(alpha), GP_E_SHAPE, "alpha=%g must be positive and finite", alpha);
  GP_REQUIRE(outputscale > 0.f && noise >= 0.f, GP_E_SHAPE, "outputscale must be > 0 and noise >= 0");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "gp_plan_set_hypers_rq is not available on a SKI plan (gp_plan_set_ski)");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "gp_plan_set_hypers_rq is not available on a kernel-sum plan: give the kind to a term");
  GP_CHECK(refuse_settings(p, CALL_SET_HYPERS_RQ));
  GP_REQUIRE(!(p->comm && p->comm->world > 1), GP_E_STATE, "gp_plan_set_hypers_rq is not available on a row-sharded plan (gp_plan_set_comm)");
  GP_CUDA(cudaSetDevice(p->device));
  // all or nothing: a failed pack restores the previous hyper-parameters (and packing), so the number of gradient values a caller
  // sizes from the kind it asked for always matches what the engine writes
  const int old_kind = p->kind;
  const std::vector<float> old_ls = p->ls;
  const float old_alpha = p->rq_alpha, old_os = p->outputscale, old_noise = p->noise;
  const bool old_set = p->hypers_set;
  p->kind = GP_RQ;
  p->ls.assign(lengthscale, lengthscale + n_ls);
  p->rq_alpha = alpha;
  p->outputscale = outputscale;
  p->noise = noise;
  p->hypers_set = true;
  if (!p->data_set) return GP_OK;
  const int st = pack_inputs(p);
  if (st != GP_OK) {
    p->kind = old_kind;
    p->ls = old_ls;
    p->rq_alpha = old_alpha;
    p->outputscale = old_os;
    p->noise = old_noise;
    p->hypers_set = old_set;
    if (old_set) pack_inputs(p);   // the previous packing; the error reported is the first one
  }
  return st;
}

extern "C" int gp_plan_set_hypers_poly(gp_plan* p, int power, float offset, float outputscale, float noise) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(power >= 1 && power <= 8, GP_E_SHAPE, "power=%d must be an integer in [1, 8]", power);
  GP_REQUIRE(offset >= 0.f && isfinite(offset), GP_E_SHAPE, "offset=%g must be finite and >= 0", offset);
  GP_REQUIRE(outputscale > 0.f && noise >= 0.f, GP_E_SHAPE, "outputscale must be > 0 and noise >= 0");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "gp_plan_set_hypers_poly is not available on a SKI plan (gp_plan_set_ski)");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "gp_plan_set_hypers_poly is not available on a kernel-sum plan: give the kind to a term");
  GP_CHECK(refuse_settings(p, CALL_SET_HYPERS_POLY));
  GP_REQUIRE(!(p->comm && p->comm->world > 1), GP_E_STATE, "gp_plan_set_hypers_poly is not available on a row-sharded plan (gp_plan_set_comm)");
  GP_CUDA(cudaSetDevice(p->device));
  // all or nothing, as gp_plan_set_hypers_rq: a failed pack restores the previous hyper-parameters (and packing)
  const int old_kind = p->kind, old_power = p->poly_power;
  const std::vector<float> old_ls = p->ls;
  const float old_off = p->poly_offset, old_os = p->outputscale, old_noise = p->noise;
  const bool old_set = p->hypers_set;
  p->kind = GP_POLY;
  p->ls.assign(1, 1.f);   // no lengthscale: the inputs are packed raw (pack.cu)
  p->poly_power = power;
  p->poly_offset = offset;
  p->outputscale = outputscale;
  p->noise = noise;
  p->hypers_set = true;
  if (!p->data_set) return GP_OK;
  const int st = pack_inputs(p);
  if (st != GP_OK) {
    p->kind = old_kind;
    p->ls = old_ls;
    p->poly_power = old_power;
    p->poly_offset = old_off;
    p->outputscale = old_os;
    p->noise = old_noise;
    p->hypers_set = old_set;
    if (old_set) pack_inputs(p);   // the previous packing; the error reported is the first one
  }
  return st;
}

extern "C" int gp_plan_set_noise_diag(gp_plan* p, const float* diag, int64_t n) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(diag == nullptr || (p->data_set && p->same && n == p->n2), GP_E_SHAPE,
             "the noise diagonal needs one entry per row of a square operator (n=%lld)", (long long)n);
  p->noise_diag = diag;
  return GP_OK;
}

extern "C" int gp_kmv(gp_plan* p, const float* V, int64_t ldv, int t, float* OUT, int64_t ldo, int add_noise) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready (set_data + set_hypers)");
  GP_REQUIRE(t >= 1 && ldv >= t && ldo >= t, GP_E_SHAPE, "bad K.V shape t=%d ldv=%lld ldo=%lld", t, (long long)ldv, (long long)ldo);
  GP_CUDA(cudaSetDevice(p->device));
  GP_CHECK(p->V16.ensure(sizeof(float) * p->n2 * TP));
  for (int c0 = 0; c0 < t; c0 += TP) {
    int tc = std::min(TP, t - c0);
    KronColsScope kcols(p, tc);
    GP_CHECK(to_v16(p, V + c0, ldv, tc, p->n2, p->V16.as<float>()));
    GP_CHECK(kmv_partials(p, p->V16.as<float>(), nullptr));
    GP_CHECK(kmv_finish_user(p, p->V16.as<float>(), OUT + c0, ldo, tc, add_noise));
  }
  return GP_OK;
}

extern "C" int gp_plan_set_comm(gp_plan* p, gp_comm* comm) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(!(p->tasks && comm && comm->world > 1), GP_E_SHAPE, "task indices are not available on a row-sharded plan");
  GP_REQUIRE(!(p->kron && comm && comm->world > 1), GP_E_SHAPE, "a Kronecker plan is not available on a row-sharded plan");
  GP_REQUIRE(!(p->deriv && comm && comm->world > 1), GP_E_SHAPE, "a derivative plan is not available on a row-sharded plan");
  if (comm && comm->world > 1) GP_CHECK(refuse_settings(p, CALL_SET_COMM_SHARDED));
  p->comm = comm;
  return GP_OK;
}

extern "C" int64_t gp_kernel_launches(gp_plan* p) { return p ? p->launches : 0; }

extern "C" int gp_plan_info(gp_plan* p, int* backend, int* nsplit, int* kpad, int* n_sm) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  if (backend) *backend = p->backend;
  if (nsplit) *nsplit = p->nsplit;
  if (kpad) *kpad = p->KP;
  if (n_sm) *n_sm = p->n_sm;
  return GP_OK;
}

extern "C" int gp_time_kmv_kernel(gp_plan* p, const float* V, int64_t ldv, int t, int warmup, int reps, float* ms_per_launch) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(t >= 1 && t <= TP && reps >= 1 && ms_per_launch, GP_E_SHAPE, "bad timing arguments");
  GP_CUDA(cudaSetDevice(p->device));
  GP_CHECK(p->V16.ensure(sizeof(float) * p->n2 * TP));
  GP_CHECK(to_v16(p, V, ldv, t, p->n2, p->V16.as<float>()));
  KronColsScope kcols(p, t);
  if (p->backend == GP_BACKEND_PRODUCT) GP_CHECK(product_refresh(p));
  if (!p->tasks && !p->deriv && (p->backend == GP_BACKEND_TCGEN05 || (p->backend == GP_BACKEND_SUM && p->sum_any_tc) || (p->backend == GP_BACKEND_PRODUCT && p->prod_tc))) GP_CHECK(pack_v_tiles(p, p->V16.as<float>()));
  auto launch = [&]() -> int {
    // a multitask plan: the whole product (gather, V tiles, one launch per column task, combine)
    if (p->tasks) return tasks_kmv_partials(p, p->V16.as<float>(), p->kind, nullptr);
    // a Kronecker plan: the whole product (B mix, V tiles, one data-kernel launch per chunk, scatter)
    if (p->kron) return kron_kmv_partials(p, p->V16.as<float>(), nullptr);
    // a derivative plan: the derivative kernel over the live column chunks and the split sum
    if (p->deriv) return deriv_kmv_partials(p, p->V16.as<float>(), nullptr);
    if (p->backend == GP_BACKEND_SKI) return ski_kmv_partials(p, p->V16.as<float>(), nullptr);
    if (p->backend == GP_BACKEND_SUM) return sum_kmv_launch(p, p->V16.as<float>(), nullptr);
    if (p->backend == GP_BACKEND_PRODUCT) return product_kmv_launch(p, p->V16.as<float>(), nullptr);
    if (p->add_M) return additive_kmv_launch(p, p->V16.as<float>(), nullptr);
    if (p->sm_Q) return spectral_kmv_launch(p, p->V16.as<float>(), nullptr);
    return p->backend == GP_BACKEND_TCGEN05 ? kmv_tc_launch(p, nullptr) : kmv_simt_launch(p, p->V16.as<float>(), nullptr);
  };
  for (int i = 0; i < warmup; ++i) GP_CHECK(launch());
  cudaEvent_t e0, e1;
  GP_CUDA(cudaEventCreate(&e0));
  GP_CUDA(cudaEventCreate(&e1));
  GP_CUDA(cudaEventRecord(e0, p->stream));
  for (int i = 0; i < reps; ++i) GP_CHECK(launch());
  GP_CUDA(cudaEventRecord(e1, p->stream));
  GP_CUDA(cudaEventSynchronize(e1));
  float ms = 0.f;
  GP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *ms_per_launch = ms / reps;
  return GP_OK;
}

// MultivariateNormal.log_prob through inv_quad_logdet (distributions/multivariate_normal.py:248-251)
extern "C" int gp_mll(gp_plan* p, const float* y_minus_mean, const float* eps1, const float* eps2, const float* rademacher,
                      const gp_mll_opts* o, float* solve_out, gp_mll_result* res) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(p->same, GP_E_SHAPE, "MLL needs a square operator");
  GP_REQUIRE(o && res, GP_E_SHAPE, "opts/result missing");
  GP_REQUIRE(o->num_probes >= 1 && o->num_probes + 1 <= TP, GP_E_SHAPE, "num_probes must be in [1,%d]", TP - 1);
  GP_CUDA(cudaSetDevice(p->device));
  memset(res, 0, sizeof(*res));
  cudaStream_t st = p->stream;
  const int64_t n = p->row_count, N = p->n2;
  const int tp = o->num_probes, t = tp + 1;
  int flags = 0;
  // GP_MLL_TIMING=1: CUDA-event time of every phase, printed to stderr (profiling aid; adds event records only)
  const bool timing = getenv("GP_MLL_TIMING") != nullptr;
  cudaEvent_t tev[8];
  int ntev = 0;
  auto mark = [&]() {
    if (timing && ntev < 8) { cudaEventCreate(&tev[ntev]); cudaEventRecord(tev[ntev], st); ++ntev; }
  };
  mark();

  // --- preconditioner (AddedDiagLinearOperator._preconditioner) ---
  int k = 0;
  double logdet_p = 0.0;
  const float* W = nullptr;
  // SKI and low-rank-corrected plans run unpreconditioned (no pivoted Cholesky of a downdated operator, lowrank.cu)
  const bool want_precond = o->precond_rank > 0 && N >= o->min_precond_size && p->backend != GP_BACKEND_SKI && p->lr_U == nullptr;
  float* Lt = nullptr;
  if (want_precond) {
    int rank = (int)std::min<int64_t>(o->precond_rank, N);
    GP_REQUIRE(rank <= 128, GP_E_SHAPE, "precond_rank %d > 128", rank);
    GP_CHECK(p->misc.ensure(sizeof(float) * (size_t)rank * N + sizeof(int64_t) * rank + 64));
    Lt = p->misc.as<float>();
    int64_t* piv = reinterpret_cast<int64_t*>(Lt + (size_t)rank * N);
    int st_pc = gp_pivoted_cholesky(p, rank, o->precond_tol, Lt, piv, &k);
    if (st_pc == GP_W_PIVCHOL_NAN) { flags |= 1; k = 0; }
    else GP_CHECK(st_pc);
    if (k > 0) {
      GP_CHECK(p->misc2.ensure(sizeof(float) * (size_t)n * k));
      int st_pb = gp_precond_build(p, Lt, k, p->misc2.as<float>(), &logdet_p);
      if (st_pb == GP_W_PIVCHOL_NAN) { flags |= 1; k = 0; logdet_p = 0.0; }
      else GP_CHECK(st_pb);
      if (k > 0) W = p->misc2.as<float>();
    }
  }
  res->precond_rank = k;
  res->logdet_precond = logdet_p;
  mark();

  // --- probes and the [Z | y - mu] right-hand side ---
  GP_CHECK(p->misc3.ensure(sizeof(float) * (size_t)n * (tp + t + t) + sizeof(float) * (size_t)tp * o->max_tridiag_iter * o->max_tridiag_iter + 4096));
  float* probes = p->misc3.as<float>();                 // [n][tp]
  float* rhs = probes + (size_t)n * tp;                  // [n][t]
  float* solves = rhs + (size_t)n * t;                   // [n][t]
  float* tmat = solves + (size_t)n * t;                  // [tp][J][J]
  double* iq_part = reinterpret_cast<double*>(tmat + (size_t)tp * o->max_tridiag_iter * o->max_tridiag_iter + 16);
  iq_part = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(iq_part) + 7) & ~(uintptr_t)7);
  const float* pz = rademacher;
  if (k > 0) {
    GP_REQUIRE(eps1 && eps2, GP_E_SHAPE, "eps1/eps2 base samples are required with a preconditioner");
    GP_CHECK(gp_precond_probes(p, Lt, k, eps1, eps2, tp, probes));
    pz = probes;
  } else {
    GP_REQUIRE(rademacher != nullptr, GP_E_SHAPE, "rademacher probes are required without a preconditioner");
  }
  {
    int64_t tot = n * t;
    concat_rhs_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, st>>>(pz, tp, y_minus_mean, n, rhs, nullptr);
    p->launches++;
  }
  mark();
  // linear_cg normalises every column itself (probe_vector_norms only matter for the backward pass), so the
  // un-normalised probes give the same solves for the y column and the same tridiagonals.
  int iters = 0, J = 0;
  int st_cg = mbcg_run(p, rhs, t, t, tp, o->cg_tol, o->max_cg_iter, o->max_tridiag_iter, W, k, solves, t, tmat, &iters, &J, res->resid);
  if (st_cg == GP_W_NOT_CONVERGED) flags |= 2;
  else GP_CHECK(st_cg);
  res->cg_iters = iters;
  res->tridiag_size = J;
  mark();

  double logdet = 0.0;
  {
    int st_slq = gp_slq_logdet(p, tmat, tp, o->max_tridiag_iter, J, N, &logdet);
    if (st_slq == GP_W_EIG_NOT_CONVERGED) flags |= 4;
    else GP_CHECK(st_slq);
  }
  invquad_kernel<<<64, 256, 0, st>>>(solves, t, tp, y_minus_mean, n, iq_part);
  p->launches++;
  if (solve_out) {
    extract_col_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(solves, t, tp, n, solve_out);
    p->launches++;
  }
  double* h = reinterpret_cast<double*>(static_cast<char*>(p->pinned) + PIN_SCALARS);
  GP_CUDA(cudaMemcpyAsync(h, iq_part, sizeof(double) * 64, cudaMemcpyDeviceToHost, st));
  GP_CUDA(cudaStreamSynchronize(st));
  double iq = 0.0;
  for (int i = 0; i < 64; ++i) iq += h[i];
  if (timing) {
    mark();
    cudaEventSynchronize(tev[ntev - 1]);
    static const char* names[] = {"pivchol+precond_build", "probes+rhs", "mbcg", "slq+invquad"};
    fprintf(stderr, "[gp_mll timing]");
    for (int i = 0; i + 1 < ntev; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, tev[i], tev[i + 1]);
      fprintf(stderr, " %s %.3f ms;", names[i], ms);
    }
    fprintf(stderr, " cg_iters %d\n", iters);
    for (int i = 0; i < ntev; ++i) cudaEventDestroy(tev[i]);
  }
  if (p->comm && p->comm->world > 1) {
    // inv_quad is a sum over local rows: all-reduce it (one fp64)
    double* d_iq = iq_part;
    GP_CUDA(cudaMemcpyAsync(d_iq, &iq, sizeof(double), cudaMemcpyHostToDevice, st));
    GP_CHECK(nccl_allreduce_double(p->comm, d_iq, 1, st));
    GP_CUDA(cudaMemcpyAsync(h, d_iq, sizeof(double), cudaMemcpyDeviceToHost, st));
    GP_CUDA(cudaStreamSynchronize(st));
    iq = h[0];
  }
  res->inv_quad = iq;
  res->logdet = logdet + logdet_p;
  res->log_prob = -0.5 * (iq + res->logdet + (double)N * log(2.0 * M_PI));
  res->mll = res->log_prob / (double)N;
  res->status_flags = flags;
  return GP_OK;
}
