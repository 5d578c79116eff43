// sum.cu -- kernel sums  K = K_1 + ... + K_m  (AdditiveKernel, /root/reference/gpytorch/kernels/kernel.py:592-621: the reference
// evaluates every term densely and adds the matrices; here a product of the sum is one fused K.V launch per term, all writing
// disjoint column-split slots of ONE partial buffer that the usual finish kernels reduce with the owning term's outputscale).
//
// The parent plan (backend GP_BACKEND_SUM) owns no packed inputs: it holds the shared workspaces (partial slots, packed V
// tiles, CG state) and the noise; the terms are complete plans over the same rows that keep their own packed X (their
// lengthscales / active dimensions differ).  While the parent launches a term's kernel the term's output / V-tile pointers are
// redirected to the parent's buffers (gp_plan::partial_ext / vtiles_ext).
#include "gp_common.cuh"

namespace gp {

int sum_pack(gp_plan* p) {
  GP_REQUIRE(!p->terms.empty() && p->terms.size() <= 4, GP_E_SHAPE, "a kernel sum takes 1 to 4 terms");
  p->backend = GP_BACKEND_SUM;
  p->rows_pad = cdiv(p->row_count, 2 * TILE_I) * 2 * TILE_I;
  p->ntile_i = p->rows_pad / TILE_I;
  p->ntile_j = cdiv(p->n2, TILE_J);
  p->DP = 0;
  p->KP = 0;
  int np = 0;
  bool all_tc = true, any_tc = false;
  for (gp_plan* t : p->terms) {
    GP_REQUIRE(t && t != p && t->data_set && t->hypers_set, GP_E_STATE, "kernel sum: every term needs set_data + set_hypers");
    GP_REQUIRE(t->backend == GP_BACKEND_TCGEN05 || t->backend == GP_BACKEND_SIMT, GP_E_SHAPE,
               "kernel sum: a term must be a plain kernel plan (not SKI, not a sum)");
    GP_CHECK(refuse_settings(t, CALL_SUM_TERM_REFRESH));
    GP_CHECK(refuse_compact(t, "a kernel sum's term"));
    GP_REQUIRE(t->n1 == p->n1 && t->n2 == p->n2 && t->same == p->same && t->row_begin == p->row_begin && t->row_count == p->row_count,
               GP_E_SHAPE, "kernel sum: term shape %lld x %lld (rows [%lld,+%lld)) differs from the sum's %lld x %lld (rows [%lld,+%lld))",
               (long long)t->n1, (long long)t->n2, (long long)t->row_begin, (long long)t->row_count, (long long)p->n1, (long long)p->n2,
               (long long)p->row_begin, (long long)p->row_count);
    GP_REQUIRE(t->device == p->device && t->stream == p->stream, GP_E_STATE, "kernel sum: terms must live on the sum's device and stream");
    GP_REQUIRE(t->rows_pad == p->rows_pad, GP_E_STATE, "kernel sum: row padding mismatch");
    np += t->nsplit;
    all_tc = all_tc && t->backend == GP_BACKEND_TCGEN05;
    any_tc = any_tc || t->backend == GP_BACKEND_TCGEN05;
    p->KP = std::max(p->KP, t->KP);
  }
  p->sum_tc = all_tc;
  p->sum_any_tc = any_tc;
  p->nparts = np;
  p->nsplit = np;
  p->xbad = p->terms[0]->xbad;   // the terms see the same rows: one non-finite flag serves all
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  if (any_tc) GP_CHECK(p->Vtiles.ensure(sizeof(float) * p->ntile_j * (2 * TILE_J * TP + TILE_J * TP / 2)));
  p->part_scale_host.clear();
  return slot_scales_prepare(p);
}

// per-slot scales: a kernel sum scales each slot by the outputscale of the term that owns it, a low-rank plan scales the backend's
// slots by its outputscale and its own last slot by 1.  Refreshed whenever a term was re-packed or the hyper-parameters changed
// (cheap host compare per call); other plans keep one outputscale for all slots (part_scale_ptr = nullptr).
int slot_scales_prepare(gp_plan* p) {
  const bool sum = p->backend == GP_BACKEND_SUM;
  if (!sum && !p->lr_U) return GP_OK;
  std::vector<float> sc;
  if (sum) {
    for (gp_plan* t : p->terms)
      for (int s = 0; s < t->nsplit; ++s) sc.push_back(t->outputscale);
    GP_REQUIRE((int)sc.size() == p->nparts, GP_E_STATE, "kernel sum: a term changed its geometry (%d slots, expected %d); call gp_plan_set_sum again",
               (int)sc.size(), p->nparts);
  } else {
    sc.assign(p->nparts, kernel_scale(p));
  }
  if (p->lr_U) sc.push_back(1.f);
  if (sizeof(float) * sc.size() > p->part_scale.cap) {
    GP_CHECK(p->part_scale.ensure(sizeof(float) * std::max<size_t>(64, sc.size())));
    p->part_scale_host.clear();
  }
  if (sc != p->part_scale_host) {
    p->part_scale_host = sc;
    // pageable source: staged by the runtime before the call returns
    GP_CUDA(cudaMemcpyAsync(p->part_scale.p, p->part_scale_host.data(), sizeof(float) * sc.size(), cudaMemcpyHostToDevice, p->stream));
  }
  return GP_OK;
}

int sum_kmv_launch(gp_plan* p, const float* V16, const int* done_flag) {
  GP_CHECK(slot_scales_prepare(p));
  int off = 0;
  for (gp_plan* t : p->terms) {
    GP_REQUIRE(t->backend == GP_BACKEND_TCGEN05 || V16 != nullptr, GP_E_STATE, "kernel sum: fp32 rows of V needed for a CUDA-core term");
    t->partial_ext = p->partial.as<float>() + (size_t)off * p->rows_pad * TP;
    t->vtiles_ext = p->Vtiles.as<float>();
    const int st = (t->backend == GP_BACKEND_TCGEN05) ? kmv_tc_launch(t, done_flag) : kmv_simt_launch(t, V16, done_flag);
    t->partial_ext = nullptr;
    t->vtiles_ext = nullptr;
    if (st != GP_OK) return st;
    p->launches++;
    off += t->nsplit;
  }
  return GP_OK;
}

// rows of the sum: term 0 writes OUT, every later term writes scratch rows that are added in term order
__global__ void add_rows_kernel(const float* __restrict__ src, int64_t m, int64_t n, float* __restrict__ OUT, int64_t ldo) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) OUT[blockIdx.y * ldo + j] += src[blockIdx.y * n + j];
}

int sum_krows(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  GP_REQUIRE(m <= 65535, GP_E_SHAPE, "rows of a kernel sum: at most 65535 rows per call (m=%lld)", (long long)m);
  GP_CHECK(gp_krows(p->terms[0], idx, m, OUT, ldo));
  if (p->terms.size() > 1) GP_CHECK(p->misc.ensure(sizeof(float) * (size_t)m * p->n2));
  for (size_t t = 1; t < p->terms.size(); ++t) {
    GP_CHECK(gp_krows(p->terms[t], idx, m, p->misc.as<float>(), p->n2));
    add_rows_kernel<<<dim3((unsigned)cdiv(p->n2, 256), (unsigned)m), 256, 0, p->stream>>>(p->misc.as<float>(), m, p->n2, OUT, ldo);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_sum(gp_plan* p, gp_plan* const* terms, int n_terms) {
  GP_REQUIRE(p && p->data_set, GP_E_STATE, "kernel sum: call gp_plan_set_data on the sum first");
  GP_REQUIRE(terms != nullptr && n_terms >= 1 && n_terms <= 4, GP_E_SHAPE, "a kernel sum takes 1 to 4 terms (got %d)", n_terms);
  GP_REQUIRE(p->ski == nullptr, GP_E_STATE, "a SKI plan cannot become a kernel sum");
  GP_CHECK(refuse_settings(p, CALL_SET_SUM));
  GP_CHECK(refuse_compact(p, "gp_plan_set_sum"));
  for (int t = 0; t < n_terms; ++t) {
    if (terms[t]) GP_CHECK(refuse_settings(terms[t], CALL_SUM_TERM));
    if (terms[t]) GP_CHECK(refuse_compact(terms[t], "gp_plan_set_sum (a term)"));
  }
  GP_CUDA(cudaSetDevice(p->device));
  p->terms.assign(terms, terms + n_terms);
  p->backend_req = GP_BACKEND_SUM;
  p->backend = GP_BACKEND_SUM;
  return p->hypers_set ? sum_pack(p) : GP_OK;   // without hyper-parameters (the noise) yet: packed by gp_plan_set_hypers
}
