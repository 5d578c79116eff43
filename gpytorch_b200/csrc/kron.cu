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
//
// Several terms (gp_plan_set_kron_terms; LCMKernel, kernels/lcm_kernel.py): sum_q (s_q K_q) (x) B_q.  Each term runs the pipeline
// above up to its own partial slots (its B_q mix, its data plan's launches); lcm_scatter_kernel sums s_q times each term's slots in
// term order.  Rows, the diagonal and the gradients run the single-term passes per term with that term's B_q.
#include <math.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "gp_common.cuh"

namespace gp {

constexpr int KRON_RED_ROWS = 2048;   // points per block of the dB reduction

// W[q][j][cc] = sum_b B[a][b] V16[j T + b][c] for the column col = 16 q + cc = a t + c (B == nullptr: V16[j T + a][c], the
// unmixed chunks); zero for col >= T t and for the padding rows j >= n.  MASKED: V16 holds the observed rows only, and row j T + b
// is V16[colpos[j T + b]], or 0 where colpos is -1 (a missing column of P_r ((s K) (x) B) P_c^T)
template <bool MASKED>
__global__ void kron_mix_kernel(const float* __restrict__ V16, int64_t n, int64_t npad, int T, int t, int nchunk,
                                const float* __restrict__ B, float* __restrict__ W, const int* __restrict__ done_flag,
                                const int* __restrict__ colpos) {
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
    if constexpr (MASKED) {
      const int* cp = colpos + j * T;
      if (B) {
        const float* br = B + a * T;
        for (int b = 0; b < T; ++b) {
          const int r = cp[b];
          s = fmaf(br[b], r >= 0 ? V16[(int64_t)r * TP + c] : 0.f, s);
        }
      } else {
        const int r = cp[a];
        s = r >= 0 ? V16[(int64_t)r * TP + c] : 0.f;
      }
    } else {
      const float* v = V16 + j * T * TP + c;
      if (B) {
        const float* br = B + a * T;
        for (int b = 0; b < T; ++b) s = fmaf(br[b], v[b * TP], s);
      } else {
        s = v[a * TP];
      }
    }
  }
  W[idx] = s;
}

// out[(i T + a)][c] = sum_sp part[q][sp][i][cc] for col = a t + c = 16 q + cc (c < t), 0 for c >= t; NaN for non-finite inputs or
// a non-finite B (the fused kernels' clamps and operand splits need not carry a NaN of the mixed block through).  MASKED: out has
// the nrows observed rows, and observed row r is interleaved row rowmap[r] = i T + a
template <bool MASKED>
__global__ void kron_scatter_kernel(const float* __restrict__ part, int nsplit, int64_t rows_pad, int64_t n1, int T, int t,
                                    float* __restrict__ out, const int* __restrict__ xbad, int bbad, const int* __restrict__ done_flag,
                                    const int* __restrict__ rowmap, int64_t nrows) {
  if (done_flag && *done_flag) return;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (MASKED ? nrows : n1 * T) * TP) return;
  const int c = (int)(idx % TP);
  const int64_t r = MASKED ? (int64_t)rowmap[idx / TP] : idx / TP;
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

// ---- several terms (gp_plan_set_kron_terms): sum_q (s_q K_q) (x) B_q ----
struct LcmTerms {
  const float* part[KRON_MAX_TERMS];   // each term's partial slots [nchunk][nsplit][rows_pad][16]
  int nsplit[KRON_MAX_TERMS];
  int64_t rows_pad[KRON_MAX_TERMS];
  float s[KRON_MAX_TERMS];             // the term data plan's outputscale
  const int* xbad[KRON_MAX_TERMS];
  int Q;
};

// out[(i T + a)][c] = sum_q s_q sum_sp part_q[q'][sp][i][cc] for col = a t + c = 16 q' + cc (c < t), 0 for c >= t; terms outer,
// splits inner.  NaN when any term has non-finite inputs, or a B_q a non-finite entry (bbad)
__global__ void lcm_scatter_kernel(const LcmTerms lt, int64_t n1, int T, int t, float* __restrict__ out, int bbad,
                                   const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n1 * T * TP) return;
  const int c = (int)(idx % TP);
  const int64_t r = idx / TP;
  const int64_t i = r / T;
  const int a = (int)(r % T);
  float s = 0.f;
  bool bad = bbad != 0;
  for (int q = 0; q < lt.Q; ++q) {
    bad = bad || *lt.xbad[q];
    if (c < t) {
      const int col = a * t + c;
      const int64_t rp = lt.rows_pad[q];
      const float* base = lt.part[q] + ((int64_t)(col / TP) * lt.nsplit[q] * rp + i) * TP + col % TP;
      float v = 0.f;
      for (int sp = 0; sp < lt.nsplit[q]; ++sp) v += base[(int64_t)sp * rp * TP];
      s = fmaf(lt.s[q], v, s);
    }
  }
  if (bad) s = __int_as_float(0x7fc00000);
  out[idx] = s;
}

// OUT[r][j T + b] = sum_q rows[q][r][j] B_q[a][b], a = idx[r] mod T: row i T + a of sum_q (s_q K_q) (x) B_q from row i of every s_q K_q
__global__ void lcm_expand_rows_kernel(const float* __restrict__ rows, int Q, int64_t m, int64_t n2, const int64_t* __restrict__ idx,
                                       int64_t n, const float* __restrict__ B, int T, float* __restrict__ OUT, int64_t ldo) {
  const int64_t r = blockIdx.y;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n2 * T) return;
  const int64_t v = idx[r];
  const int a = (v >= 0 && v < n) ? (int)(v % T) : 0;
  const int b = (int)(e % T);
  float s = 0.f;
  for (int q = 0; q < Q; ++q) s = fmaf(rows[((int64_t)q * m + r) * n2 + e / T], B[((int64_t)q * T + a) * T + b], s);
  OUT[r * ldo + e] = s;
}

// OUT[i T + a] = sum_q d[q][i] B_q[a][a]
__global__ void lcm_expand_diag_kernel(const float* __restrict__ d, int Q, int64_t n1, const float* __restrict__ B, int T,
                                       float* __restrict__ OUT) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n1 * T) return;
  const int a = (int)(e % T);
  float s = 0.f;
  for (int q = 0; q < Q; ++q) s = fmaf(d[(int64_t)q * n1 + e / T], B[((int64_t)q * T + a) * T + a], s);
  OUT[e] = s;
}

// masked plans: OUT[r][e] = SRC[r][map[e]] (observed columns of full rows, or observed entries of the full diagonal with m = 1)
__global__ void masked_kron_gather_kernel(const float* __restrict__ SRC, int64_t lds, const int* __restrict__ map, int64_t ncols,
                                   float* __restrict__ OUT, int64_t ldo) {
  const int64_t r = blockIdx.y;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ncols) return;
  OUT[r * ldo + e] = SRC[r * lds + map[e]];
}

// masked plans: the interleaved row rowmap[v] of each requested observed row v (-1 outside [0, nrows): a NaN row, as unmasked)
__global__ void masked_kron_idx_kernel(const int64_t* __restrict__ idx, int64_t m, const int* __restrict__ rowmap, int64_t nrows,
                                    int64_t* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const int64_t v = idx[r];
  out[r] = (v >= 0 && v < nrows) ? (int64_t)rowmap[v] : -1;
}

// masked plans: OUT [nfull][s] = the observed rows of SRC [.][ld] at their interleaved rows, zero on the missing rows (the gradients
// of P_r ((s K) (x) B) P_c^T are those of (s K) (x) B with L and R zero there)
__global__ void masked_kron_expand_kernel(const float* __restrict__ SRC, int64_t ld, int s, const int* __restrict__ pos, int64_t nfull,
                                       float* __restrict__ OUT) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nfull * s) return;
  const int r = pos[e / s];
  OUT[e] = r >= 0 ? SRC[(int64_t)r * ld + (int)(e % s)] : 0.f;
}

static int kron_check_data(const gp_plan* p, const gp_plan* q, int T) {
  GP_REQUIRE(q->data_set && q->hypers_set, GP_E_STATE, "Kronecker plan: the data plan needs set_data + set_hypers");
  GP_REQUIRE(q->backend == GP_BACKEND_TCGEN05 || q->backend == GP_BACKEND_SIMT, GP_E_SHAPE,
             "Kronecker plan: the data plan must be a plain kernel plan (not SKI, not a kernel sum, not Kronecker)");
  GP_CHECK(refuse_settings(q, CALL_KRON_DATA_REFRESH));
  GP_CHECK(refuse_compact(q, "a Kronecker operator's data plan"));
  GP_REQUIRE(q->row_begin == 0 && q->row_count == q->n1 && !(q->comm && q->comm->world > 1), GP_E_SHAPE,
             "Kronecker plan: a row-sharded data plan is not available");
  GP_REQUIRE(q->device == p->device && q->stream == p->stream, GP_E_STATE, "Kronecker plan: the data plan must live on the same device and stream");
  GP_REQUIRE(q->n1 * T < ((int64_t)1 << 31) && q->n2 * T < ((int64_t)1 << 31), GP_E_SHAPE,
             "Kronecker plan: N T must stay below 2^31");
  return GP_OK;
}

// operator geometry from the data plan: N1 T x N2 T rows, one partial slot
static void kron_geometry(gp_plan* p) {
  const gp_plan* q = p->kron->data;
  const int T = p->kron->T;
  p->backend = GP_BACKEND_KRON;
  p->n1 = p->kron->masked ? (int64_t)p->kron->obs_r.size() : q->n1 * T;
  p->n2 = p->kron->masked ? (int64_t)p->kron->obs_c.size() : q->n2 * T;
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
  GP_CHECK(kron_check_data(p, q, ks->T));
  const int64_t n1 = ks->masked ? (int64_t)ks->obs_r.size() : q->n1 * ks->T, n2 = ks->masked ? (int64_t)ks->obs_c.size() : q->n2 * ks->T;
  GP_REQUIRE(p->n1 == n1 && p->n2 == n2 && p->same == q->same && (!ks->masked || (q->n1 == ks->mask_n1 && q->n2 == ks->mask_n2)), GP_E_STATE,
             "Kronecker plan: the data plan changed its size; call gp_plan_set_kron again");
  p->kind = q->kind;
  p->outputscale = q->outputscale;   // the finish kernels scale the unscaled product by the data plan's s
  p->xbad = q->xbad;
  for (int t = 1; t < ks->nterm; ++t) {
    const gp_plan* qt = ks->term[t];
    GP_CHECK(kron_check_data(p, qt, ks->T));
    GP_REQUIRE(qt->n1 == q->n1 && qt->n2 == q->n2 && qt->same == q->same, GP_E_STATE,
               "Kronecker plan: a term's data plan changed its size; call gp_plan_set_kron_terms again");
  }
  if (ks->nterm > 1) p->outputscale = 1.f;   // every term's s_q is applied in the scatter (lcm_scatter_kernel)
  return GP_OK;
}

int kron_pack(gp_plan* p) {
  GP_CHECK(kron_check_data(p, p->kron->data, p->kron->T));
  kron_geometry(p);
  GP_CHECK(kron_refresh(p));
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  return GP_OK;
}

// W-chunk pitch of the data plan: whole 64-row tiles on the tensor-core path (one pack call covers every chunk)
static int64_t kron_npad(const gp_plan* q) { return q->backend == GP_BACKEND_TCGEN05 ? q->ntile_j * TILE_J : q->n2; }

// floats of the partial slots of data plan q's products over nchunk column chunks
static size_t kron_part_floats(const gp_plan* q, int nchunk) { return (size_t)nchunk * q->nsplit * q->rows_pad * TP; }

// V16 [N2 T][16] with t live columns, mixed by B (or not: B == nullptr) -> nchunk products of data plan q in ks->part from float
// part_off on (a Kronecker plan with several terms puts the terms' products back to back; ks->W and ks->Vt are re-used term after
// term in stream order).  MASKED: V16 holds the observed columns only (ks->colpos places them)
template <bool MASKED>
static int kron_chunks(gp_plan* p, gp_plan* q, const float* V16, int t, const float* B, const int* done_flag, size_t part_off,
                       int* nchunk_out) {
  gp_kron_state* ks = p->kron;
  const int kind = q->kind;
  const bool tc = q->backend == GP_BACKEND_TCGEN05;
  const int T = ks->T;
  const int nchunk = (int)cdiv((int64_t)T * t, TP);
  const int64_t npad = kron_npad(q);
  const size_t slot_floats = (size_t)q->rows_pad * TP;
  GP_CHECK(ks->W.ensure(sizeof(float) * (size_t)nchunk * npad * TP));
  GP_CHECK(ks->part.ensure(sizeof(float) * (part_off + kron_part_floats(q, nchunk))));
  const int64_t tot = (int64_t)nchunk * npad * TP;
  kron_mix_kernel<MASKED><<<(unsigned)cdiv(tot, 256), 256, 0, p->stream>>>(V16, q->n2, npad, T, t, nchunk, B, ks->W.as<float>(), done_flag,
                                                                            ks->colpos.as<int>());
  p->launches++;
  GP_CUDA(cudaGetLastError());
  if (tc) {
    GP_CHECK(ks->Vt.ensure(sizeof(float) * (size_t)nchunk * q->ntile_j * V_TILE_FLOATS));
    GP_CHECK(pack_v_tiles_rows(p, ks->W.as<float>(), (int64_t)nchunk * npad, (int64_t)nchunk * q->ntile_j, ks->Vt.as<float>()));
  }
  for (int c = 0; c < nchunk; ++c) {
    float* part = ks->part.as<float>() + part_off + (size_t)c * q->nsplit * slot_floats;
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

// several terms: every term's mixed chunks through its own data kernel, then one scatter of sum_q s_q (its slots) into slot 0
static int lcm_kmv_partials(gp_plan* p, const float* V16, const int* done_flag) {
  gp_kron_state* ks = p->kron;
  const int T = ks->T, t = p->kron_cols, Q = ks->nterm;
  const int nchunk = (int)cdiv((int64_t)T * t, TP);
  size_t off[KRON_MAX_TERMS], tot = 0, wmax = 0, vtmax = 0;
  for (int k = 0; k < Q; ++k) {   // one allocation of each buffer up front: no term's ensure frees a buffer in use
    const gp_plan* q = ks->term[k];
    off[k] = tot;
    tot += kron_part_floats(q, nchunk);
    wmax = std::max(wmax, (size_t)nchunk * kron_npad(q) * TP);
    if (q->backend == GP_BACKEND_TCGEN05) vtmax = std::max(vtmax, (size_t)nchunk * q->ntile_j * V_TILE_FLOATS);
  }
  GP_CHECK(ks->part.ensure(sizeof(float) * tot));
  GP_CHECK(ks->W.ensure(sizeof(float) * wmax));
  if (vtmax) GP_CHECK(ks->Vt.ensure(sizeof(float) * vtmax));
  LcmTerms lt;
  memset(&lt, 0, sizeof(lt));
  lt.Q = Q;
  for (int k = 0; k < Q; ++k) {
    gp_plan* q = ks->term[k];
    int nc = 0;
    GP_CHECK(kron_chunks<false>(p, q, V16, t, ks->Bd.as<float>() + (size_t)k * T * T, done_flag, off[k], &nc));
    lt.part[k] = ks->part.as<float>() + off[k];
    lt.nsplit[k] = q->nsplit;
    lt.rows_pad[k] = q->rows_pad;
    lt.s[k] = q->outputscale;
    lt.xbad[k] = q->xbad;
  }
  lcm_scatter_kernel<<<(unsigned)cdiv(p->n1 * TP, 256), 256, 0, p->stream>>>(lt, ks->data->n1, T, t, p->partial.as<float>(),
                                                                             ks->b_bad ? 1 : 0, done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int kron_kmv_partials(gp_plan* p, const float* V16, const int* done_flag) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CHECK(kron_refresh(p));
  if (ks->nterm > 1) return lcm_kmv_partials(p, V16, done_flag);
  gp_plan* q = ks->data;
  const int t = p->kron_cols;
  int nchunk = 0;
  const unsigned grid = (unsigned)cdiv(p->n1 * TP, 256);
  if (ks->masked) {
    GP_CHECK(kron_chunks<true>(p, q, V16, t, ks->Bd.as<float>(), done_flag, 0, &nchunk));
    kron_scatter_kernel<true><<<grid, 256, 0, p->stream>>>(ks->part.as<float>(), q->nsplit, q->rows_pad, q->n1, ks->T, t, p->partial.as<float>(),
                                                           q->xbad, ks->b_bad ? 1 : 0, done_flag, ks->rowmap.as<int>(), p->n1);
  } else {
    GP_CHECK(kron_chunks<false>(p, q, V16, t, ks->Bd.as<float>(), done_flag, 0, &nchunk));
    kron_scatter_kernel<false><<<grid, 256, 0, p->stream>>>(ks->part.as<float>(), q->nsplit, q->rows_pad, q->n1, ks->T, t, p->partial.as<float>(),
                                                            q->xbad, ks->b_bad ? 1 : 0, done_flag, nullptr, 0);
  }
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
  const int64_t n1f = q->n1 * ks->T, n2f = q->n2 * ks->T;
  GP_CHECK(ks->idx.ensure(sizeof(int64_t) * m));
  if (ks->nterm > 1) {   // every term's rows of s_q K_q back to back, then one expand-and-accumulate pass
    const int Q = ks->nterm;
    GP_CHECK(ks->rows.ensure(sizeof(float) * (size_t)Q * m * q->n2));
    kron_point_idx_kernel<<<(unsigned)cdiv(m, 256), 256, 0, p->stream>>>(idx, m, ks->T, n1f, ks->idx.as<int64_t>());
    p->launches++;
    for (int k = 0; k < Q; ++k)
      GP_CHECK(gp_krows(ks->term[k], ks->idx.as<int64_t>(), m, ks->rows.as<float>() + (size_t)k * m * q->n2, q->n2));
    lcm_expand_rows_kernel<<<dim3((unsigned)cdiv(n2f, 256), (unsigned)m), 256, 0, p->stream>>>(ks->rows.as<float>(), Q, m, q->n2, idx, n1f,
                                                                                            ks->Bd.as<float>(), ks->T, OUT, ldo);
    p->launches++;
    GP_CUDA(cudaGetLastError());
    return GP_OK;
  }
  GP_CHECK(ks->rows.ensure(sizeof(float) * (size_t)m * q->n2));
  if (ks->masked) {   // requested observed rows -> interleaved rows; full rows into scratch, then the observed columns
    GP_CHECK(ks->gidx.ensure(sizeof(int64_t) * m));
    GP_CHECK(ks->full.ensure(sizeof(float) * (size_t)m * n2f));
    masked_kron_idx_kernel<<<(unsigned)cdiv(m, 256), 256, 0, p->stream>>>(idx, m, ks->rowmap.as<int>(), p->n1, ks->gidx.as<int64_t>());
    p->launches++;
    idx = ks->gidx.as<int64_t>();
  }
  kron_point_idx_kernel<<<(unsigned)cdiv(m, 256), 256, 0, p->stream>>>(idx, m, ks->T, n1f, ks->idx.as<int64_t>());
  p->launches++;
  GP_CHECK(gp_krows(q, ks->idx.as<int64_t>(), m, ks->rows.as<float>(), q->n2));
  float* dst = ks->masked ? ks->full.as<float>() : OUT;
  kron_expand_rows_kernel<<<dim3((unsigned)cdiv(n2f, 256), (unsigned)m), 256, 0, p->stream>>>(ks->rows.as<float>(), q->n2, idx, n1f,
                                                                                          ks->Bd.as<float>(), ks->T, dst,
                                                                                          ks->masked ? n2f : ldo);
  p->launches++;
  if (ks->masked) {
    masked_kron_gather_kernel<<<dim3((unsigned)cdiv(p->n2, 256), (unsigned)m), 256, 0, p->stream>>>(dst, n2f, ks->colmap.as<int>(), p->n2, OUT, ldo);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int kron_kdiag(gp_plan* p, float* OUT) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CHECK(kron_refresh(p));
  gp_plan* q = ks->data;
  const int64_t n1f = q->n1 * ks->T;
  if (ks->nterm > 1) {   // sum_q s_q k_q(x_i, x_i) B_q[a, a]
    const int Q = ks->nterm;
    GP_CHECK(ks->rows.ensure(sizeof(float) * (size_t)Q * q->n1));
    for (int k = 0; k < Q; ++k) GP_CHECK(gp_kdiag(ks->term[k], ks->rows.as<float>() + (size_t)k * q->n1));
    lcm_expand_diag_kernel<<<(unsigned)cdiv(n1f, 256), 256, 0, p->stream>>>(ks->rows.as<float>(), Q, q->n1, ks->Bd.as<float>(), ks->T, OUT);
    p->launches++;
    GP_CUDA(cudaGetLastError());
    return GP_OK;
  }
  GP_CHECK(ks->rows.ensure(sizeof(float) * q->n1));
  GP_CHECK(gp_kdiag(q, ks->rows.as<float>()));
  if (ks->masked) GP_CHECK(ks->full.ensure(sizeof(float) * n1f));
  float* dst = ks->masked ? ks->full.as<float>() : OUT;
  kron_expand_diag_kernel<<<(unsigned)cdiv(n1f, 256), 256, 0, p->stream>>>(ks->rows.as<float>(), q->n1, ks->Bd.as<float>(), ks->T, dst);
  p->launches++;
  if (ks->masked) {   // s B[a, a] k_ii gathered by the row map
    masked_kron_gather_kernel<<<dim3((unsigned)cdiv(p->n1, 256), 1u), 256, 0, p->stream>>>(dst, 0, ks->rowmap.as<int>(), p->n1, OUT, 0);
    p->launches++;
  }
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// masked plans: L [n_rows][.] and R [n_cols][.] expanded with zeros to the N1 T and N2 T interleaved rows (ld = s), so that the
// unmasked gradient passes below run on them unchanged; unmasked plans pass L and R through
static int kron_expand_operands(gp_plan* p, const float** L, int64_t* ldl, const float** R, int64_t* ldr, int s) {
  gp_kron_state* ks = p->kron;
  if (!ks->masked) return GP_OK;
  const gp_plan* q = ks->data;
  const int64_t n1f = q->n1 * ks->T, n2f = q->n2 * ks->T;
  GP_CHECK(ks->Lx.ensure(sizeof(float) * (size_t)n1f * s));
  GP_CHECK(ks->Rx.ensure(sizeof(float) * (size_t)n2f * s));
  masked_kron_expand_kernel<<<(unsigned)cdiv(n1f * s, 256), 256, 0, p->stream>>>(*L, *ldl, s, ks->rowpos.as<int>(), n1f, ks->Lx.as<float>());
  masked_kron_expand_kernel<<<(unsigned)cdiv(n2f * s, 256), 256, 0, p->stream>>>(*R, *ldr, s, ks->colpos.as<int>(), n2f, ks->Rx.as<float>());
  p->launches += 2;
  GP_CUDA(cudaGetLastError());
  *L = ks->Lx.as<float>(); *R = ks->Rx.as<float>();
  *ldl = s; *ldr = s;
  return GP_OK;
}

// lengthscale(s) and outputscale of one term: data plan q's bilinear derivative over chunk pairs (L unmixed, R mixed by B, the
// term's T x T block on the device), summed in order.  L [N1 T][ldl], R [N2 T][ldr] over the interleaved rows
static int kron_bilinear_term(gp_plan* p, gp_plan* q, const float* B, const float* L, int64_t ldl, const float* R, int64_t ldr, int s,
                              double* grad_ls, double* grad_os) {
  gp_kron_state* ks = p->kron;
  const int T = ks->T;
  const int64_t n1f = q->n1 * T, n2f = q->n2 * T;
  const int nls = (int)q->ls.size();
  std::vector<double> gl(nls, 0.0), tot(nls, 0.0);
  double go = 0.0, tot_os = 0.0;
  GP_CHECK(p->misc2.ensure(sizeof(float) * n1f * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * n2f * TP));
  for (int c0 = 0; c0 < s; c0 += TP) {
    const int tc = std::min(TP, s - c0);
    GP_CHECK(to_v16(p, L + c0, ldl, tc, n1f, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, R + c0, ldr, tc, n2f, p->misc3.as<float>()));
    const int nchunk = (int)cdiv((int64_t)T * tc, TP);
    GP_CHECK(ks->Lw.ensure(sizeof(float) * (size_t)nchunk * q->n1 * TP));
    GP_CHECK(ks->W.ensure(sizeof(float) * (size_t)nchunk * q->n2 * TP));
    kron_mix_kernel<false><<<(unsigned)cdiv((int64_t)nchunk * q->n1 * TP, 256), 256, 0, p->stream>>>(p->misc2.as<float>(), q->n1, q->n1, T, tc,
                                                                                                    nchunk, nullptr, ks->Lw.as<float>(), nullptr,
                                                                                                    nullptr);
    kron_mix_kernel<false><<<(unsigned)cdiv((int64_t)nchunk * q->n2 * TP, 256), 256, 0, p->stream>>>(p->misc3.as<float>(), q->n2, q->n2, T, tc,
                                                                                                    nchunk, B, ks->W.as<float>(), nullptr, nullptr);
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

// dB of one term: dB[a][b] = s sum_i L[i T + a] . (K R_b)[i] over data plan q's products of the unmixed chunks, in fp64
static int kron_dB_term(gp_plan* p, gp_plan* q, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB) {
  gp_kron_state* ks = p->kron;
  const int T = ks->T;
  const int64_t n1f = q->n1 * T, n2f = q->n2 * T;
  const int nz = (int)cdiv(q->n1, KRON_RED_ROWS);
  GP_CHECK(p->misc2.ensure(sizeof(float) * n1f * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * n2f * TP));
  GP_CHECK(ks->red.ensure(sizeof(double) * (size_t)nz * T * T));
  std::vector<double> acc((size_t)T * T, 0.0), h((size_t)nz * T * T);
  for (int c0 = 0; c0 < t; c0 += TP) {
    const int tc = std::min(TP, t - c0);
    GP_CHECK(to_v16(p, L + c0, ldl, tc, n1f, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, R + c0, ldr, tc, n2f, p->misc3.as<float>()));
    int nchunk = 0;
    GP_CHECK(kron_chunks<false>(p, q, p->misc3.as<float>(), tc, nullptr, nullptr, 0, &nchunk));
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

// a call that takes one task covariance, on a plan with several terms
static int kron_refuse_terms(const gp_plan* p, const char* call, const char* instead) {
  GP_REQUIRE(p->kron->nterm == 1, GP_E_STATE, "%s is not available on a Kronecker plan with %d terms (gp_plan_set_kron_terms): call %s",
             call, p->kron->nterm, instead);
  return GP_OK;
}

// lengthscale(s) and outputscale: the data plan's bilinear derivative over chunk pairs (L unmixed, R mixed by B), summed in order
int kron_bilinear_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int s, double* grad_ls, double* grad_os) {
  gp_kron_state* ks = p->kron;
  GP_CHECK(kron_refuse_terms(p, "gp_bilinear_grad", "gp_kron_terms_grad"));
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CHECK(kron_refresh(p));
  GP_CHECK(kron_expand_operands(p, &L, &ldl, &R, &ldr, s));
  return kron_bilinear_term(p, ks->data, ks->Bd.as<float>(), L, ldl, R, ldr, s, grad_ls, grad_os);
}

static int kron_task_covar_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(t >= 1 && L && R && dB, GP_E_SHAPE, "gp_task_covar_grad: bad arguments");
  GP_REQUIRE((ldl >= t || p->n1 == 1) && (ldr >= t || p->n2 == 1), GP_E_SHAPE,
             "gp_task_covar_grad: leading dimensions must be >= t (ldl=%lld, ldr=%lld, t=%d)", (long long)ldl, (long long)ldr, t);
  GP_CHECK(kron_refresh(p));
  GP_CHECK(kron_expand_operands(p, &L, &ldl, &R, &ldr, t));
  return kron_dB_term(p, ks->data, L, ldl, R, ldr, t, dB);
}

static void kron_release(gp_plan* p) {
  gp_kron_state* ks = p->kron;
  gp::DevBuf* bufs[] = {&ks->Bd, &ks->W, &ks->Vt, &ks->part, &ks->Lw, &ks->red, &ks->idx, &ks->rows, &ks->rowmap, &ks->colmap,
                        &ks->rowpos, &ks->colpos, &ks->Lx, &ks->Rx, &ks->full, &ks->gidx};
  for (auto* b : bufs) b->release();
  delete ks;
  p->kron = nullptr;
}

}  // namespace gp

using namespace gp;

// gp_plan_set_kron (Q = 1) and gp_plan_set_kron_terms: every check before the plan changes, so a refused call leaves it as it was
static int kron_attach(gp_plan* p, gp_plan* const* data, int Q, int T) {
  GP_REQUIRE(T >= 1 && T <= 32, GP_E_SHAPE, "number of tasks T=%d not in [1, 32]", T);
  for (int k = 0; k < Q; ++k) GP_REQUIRE(data[k] != p, GP_E_STATE, "a Kronecker plan cannot be its own data plan");
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "a SKI plan cannot become a Kronecker plan");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "a kernel-sum plan cannot become a Kronecker plan");
  GP_CHECK(refuse_settings(p, CALL_SET_KRON));
  GP_CHECK(refuse_compact(p, "gp_plan_set_kron"));
  for (int k = 0; k < Q; ++k) GP_CHECK(refuse_settings(data[k], CALL_KRON_DATA));
  for (int k = 0; k < Q; ++k) GP_CHECK(refuse_compact(data[k], "gp_plan_set_kron (the data plan)"));
  GP_REQUIRE(!(p->comm && p->comm->world > 1), GP_E_SHAPE, "a Kronecker plan is not available on a row-sharded plan");
  for (int k = 0; k < Q; ++k) GP_CHECK(kron_check_data(p, data[k], T));
  for (int k = 1; k < Q; ++k)
    GP_REQUIRE(data[k]->n1 == data[0]->n1 && data[k]->n2 == data[0]->n2 && data[k]->same == data[0]->same, GP_E_SHAPE,
               "gp_plan_set_kron_terms: term %d has %lld x %lld points, term 0 %lld x %lld (the terms share their points' count)", k,
               (long long)data[k]->n1, (long long)data[k]->n2, (long long)data[0]->n1, (long long)data[0]->n2);
  gp_kron_state* ks = p->kron ? p->kron : new gp_kron_state();
  const bool keep_b = p->kron && ks->T == T && ks->b_set && ks->nterm == Q;
  const int oldT = ks->T;
  ks->data = data[0];
  ks->T = T;
  ks->nterm = Q;
  for (int k = 0; k < KRON_MAX_TERMS; ++k) ks->term[k] = k < Q ? data[k] : nullptr;
  p->kron = ks;
  if (!keep_b) ks->b_set = false;
  // the mask was for other sizes, or the plan now has several terms (which take no mask)
  if (ks->masked && !(Q == 1 && oldT == T && data[0]->n1 == ks->mask_n1 && data[0]->n2 == ks->mask_n2)) {
    ks->masked = false;
    ks->obs_r.clear();
    ks->obs_c.clear();
    p->noise_diag = nullptr;
  }
  p->backend_req = GP_BACKEND_KRON;
  kron_geometry(p);
  p->data_set = true;
  return p->hypers_set ? kron_pack(p) : GP_OK;   // without the noise yet: packed by gp_plan_set_hypers
}

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
  return kron_attach(p, &data, 1, T);
}

extern "C" int gp_plan_set_kron_terms(gp_plan* p, gp_plan* const* data, int Q, int T) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  if (data == nullptr) return gp_plan_set_kron(p, nullptr, 0);
  GP_REQUIRE(Q >= 1 && Q <= KRON_MAX_TERMS, GP_E_SHAPE, "number of terms Q=%d not in [1, %d]", Q, KRON_MAX_TERMS);
  for (int k = 0; k < Q; ++k) GP_REQUIRE(data[k] != nullptr, GP_E_SHAPE, "gp_plan_set_kron_terms: data plan of term %d missing", k);
  GP_CUDA(cudaSetDevice(p->device));
  return kron_attach(p, data, Q, T);
}

// host index list -> int32 vector; nullptr: every one of the nfull rows (empty vector)
static int kron_obs_list(const int64_t* idx, int64_t m, int64_t nfull, const char* what, std::vector<int>* out) {
  out->clear();
  if (idx == nullptr) return GP_OK;
  GP_REQUIRE(m >= 1 && m <= nfull, GP_E_SHAPE, "gp_plan_set_kron_observed: %lld observed %s not in [1, %lld]", (long long)m, what,
             (long long)nfull);
  for (int64_t r = 0; r < m; ++r) {
    GP_REQUIRE(idx[r] >= 0 && idx[r] < nfull && (r == 0 || idx[r] > idx[r - 1]), GP_E_SHAPE,
               "gp_plan_set_kron_observed: %s must be strictly increasing in [0, %lld) (entry %lld is %lld)", what, (long long)nfull,
               (long long)r, (long long)idx[r]);
  }
  if (m == nfull) return GP_OK;   // every row observed: the unmasked operator
  out->resize((size_t)m);
  for (int64_t r = 0; r < m; ++r) (*out)[(size_t)r] = (int)idx[r];
  return GP_OK;
}

// map [m] and its inverse [nfull] (-1 where missing) on the device; an empty list stands for the identity
static int kron_obs_upload(const std::vector<int>& obs, int64_t nfull, gp::DevBuf* map, gp::DevBuf* pos, cudaStream_t st) {
  std::vector<int> m(obs), inv((size_t)nfull, -1);
  if (m.empty()) {
    m.resize((size_t)nfull);
    for (int64_t r = 0; r < nfull; ++r) m[(size_t)r] = (int)r;
  }
  for (size_t r = 0; r < m.size(); ++r) inv[(size_t)m[r]] = (int)r;
  GP_CHECK(map->ensure(sizeof(int) * m.size()));
  GP_CHECK(pos->ensure(sizeof(int) * inv.size()));
  GP_CUDA(cudaMemcpyAsync(map->p, m.data(), sizeof(int) * m.size(), cudaMemcpyHostToDevice, st));
  GP_CUDA(cudaMemcpyAsync(pos->p, inv.data(), sizeof(int) * inv.size(), cudaMemcpyHostToDevice, st));
  GP_CUDA(cudaStreamSynchronize(st));   // the host vectors go out of scope
  return GP_OK;
}

extern "C" int gp_plan_set_kron_observed(gp_plan* p, const int64_t* rows, int64_t n_rows, const int64_t* cols, int64_t n_cols) {
  GP_REQUIRE(p != nullptr && p->kron != nullptr, GP_E_STATE, "gp_plan_set_kron_observed: not a Kronecker plan (gp_plan_set_kron)");
  GP_CHECK(kron_refuse_terms(p, "gp_plan_set_kron_observed", "gp_plan_set_kron with one data plan first"));
  GP_CUDA(cudaSetDevice(p->device));
  gp_kron_state* ks = p->kron;
  const gp_plan* q = ks->data;
  const int64_t n1f = q->n1 * ks->T, n2f = q->n2 * ks->T;
  std::vector<int> r, c;
  GP_CHECK(kron_obs_list(rows, n_rows, n1f, "rows", &r));
  GP_CHECK(kron_obs_list(cols, n_cols, n2f, "columns", &c));
  GP_REQUIRE(!q->same || r == c, GP_E_SHAPE, "gp_plan_set_kron_observed: a square plan takes equal row and column masks");
  GP_CUDA(cudaStreamSynchronize(p->stream));   // in-flight products may read the old maps
  const bool masked = !r.empty() || !c.empty();
  if (masked) {
    GP_CHECK(kron_obs_upload(r, n1f, &ks->rowmap, &ks->rowpos, p->stream));
    GP_CHECK(kron_obs_upload(c, n2f, &ks->colmap, &ks->colpos, p->stream));
    if (r.empty()) { r.resize((size_t)n1f); for (int64_t i = 0; i < n1f; ++i) r[(size_t)i] = (int)i; }
    if (c.empty()) { c.resize((size_t)n2f); for (int64_t i = 0; i < n2f; ++i) c[(size_t)i] = (int)i; }
  }
  const int64_t old_n1 = p->n1;
  ks->masked = masked;
  ks->obs_r.swap(r);
  ks->obs_c.swap(c);
  ks->mask_n1 = q->n1;
  ks->mask_n2 = q->n2;
  kron_geometry(p);
  if (p->n1 != old_n1) p->noise_diag = nullptr;   // it had one entry per row of the old operator
  return p->hypers_set ? kron_pack(p) : GP_OK;
}

// the Q task covariance blocks, row-major T x T each, to the host copy and the device
static int kron_set_blocks(gp_plan* p, const float* B, int Q, int T) {
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(B != nullptr && T == ks->T, GP_E_SHAPE, "task covariance must be %d x %d (got T=%d)", ks->T, ks->T, T);
  GP_CUDA(cudaSetDevice(p->device));
  const size_t nb = (size_t)Q * T * T;
  ks->B.assign(B, B + nb);
  ks->b_bad = false;
  for (float v : ks->B) ks->b_bad = ks->b_bad || !std::isfinite(v);
  GP_CHECK(ks->Bd.ensure(sizeof(float) * nb));
  GP_CUDA(cudaMemcpyAsync(ks->Bd.p, ks->B.data(), sizeof(float) * nb, cudaMemcpyHostToDevice, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));   // the next call may replace ks->B
  ks->b_set = true;
  return GP_OK;
}

extern "C" int gp_plan_set_kron_term_covars(gp_plan* p, const float* B, int Q, int T) {
  GP_REQUIRE(p != nullptr && p->kron != nullptr, GP_E_STATE, "gp_plan_set_kron_term_covars: not a Kronecker plan (gp_plan_set_kron_terms)");
  GP_REQUIRE(Q == p->kron->nterm, GP_E_SHAPE, "gp_plan_set_kron_term_covars: the plan has %d terms (got Q=%d)", p->kron->nterm, Q);
  return kron_set_blocks(p, B, Q, T);
}

extern "C" int gp_kron_terms_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* grad_ls,
                                  double* grad_os, double* dB) {
  GP_REQUIRE(p != nullptr && p->kron != nullptr, GP_E_STATE, "gp_kron_terms_grad: not a Kronecker plan (gp_plan_set_kron_terms)");
  GP_REQUIRE(p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(t >= 1 && L && R && grad_ls && grad_os && dB, GP_E_SHAPE, "gp_kron_terms_grad: bad arguments");
  GP_REQUIRE((ldl >= t || p->n1 == 1) && (ldr >= t || p->n2 == 1), GP_E_SHAPE,
             "gp_kron_terms_grad: leading dimensions must be >= t (ldl=%lld, ldr=%lld, t=%d)", (long long)ldl, (long long)ldr, t);
  gp_kron_state* ks = p->kron;
  GP_REQUIRE(ks->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_kron_term_covars)");
  GP_CUDA(cudaSetDevice(p->device));
  if (ks->nterm == 1) {   // the single-term passes, observed-row masks included
    GP_CHECK(kron_bilinear_grad(p, L, ldl, R, ldr, t, grad_ls, grad_os));
    return kron_task_covar_grad(p, L, ldl, R, ldr, t, dB);
  }
  GP_CHECK(kron_refresh(p));
  const int T = ks->T;
  int ls_off = 0;
  for (int k = 0; k < ks->nterm; ++k) {   // term order; each term's sums are fp64 in a fixed order
    gp_plan* q = ks->term[k];
    const float* Bk = ks->Bd.as<float>() + (size_t)k * T * T;
    GP_CHECK(kron_bilinear_term(p, q, Bk, L, ldl, R, ldr, t, grad_ls + ls_off, grad_os + k));
    GP_CHECK(kron_dB_term(p, q, L, ldl, R, ldr, t, dB + (size_t)k * T * T));
    ls_off += (int)q->ls.size();
  }
  return GP_OK;
}

// gp_plan_set_task_covar / gp_task_covar_grad on a Kronecker plan (tasks.cu forwards them here)
int gp::kron_set_task_covar(gp_plan* p, const float* B, int T) {
  GP_CHECK(kron_refuse_terms(p, "gp_plan_set_task_covar", "gp_plan_set_kron_term_covars"));
  return kron_set_blocks(p, B, 1, T);
}

int gp::kron_task_covar_grad_checked(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB) {
  GP_CHECK(kron_refuse_terms(p, "gp_task_covar_grad", "gp_kron_terms_grad"));
  GP_REQUIRE(p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(p->kron->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CUDA(cudaSetDevice(p->device));
  return kron_task_covar_grad(p, L, ldl, R, ldr, t, dB);
}
