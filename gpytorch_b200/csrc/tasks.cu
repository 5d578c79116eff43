// tasks.cu -- Hadamard multitask operator  s K(x, x') o B[t, t']  (IndexKernel, kernels/index_kernel.py:18-117, multiplied into
// the data kernel by linear_operator's MulLinearOperator; examples/03_Multitask_Exact_GPs/Hadamard_Multitask_GP_Regression.ipynb).
//
// Layout.  gp_plan_set_tasks sorts the rows (x1) and the columns (x2) by task, stably.  Packed rows keep the sorted order; the
// columns of task b form segment b of the packed column layout, which on the tensor-core path starts at a 64-column tile (the
// tail of a segment is zero padding: zero inputs and zero V rows, so it adds nothing).
//
// Products.  For a row i of task a
//     (K o B V)_i = sum_b B[a, b] P_b[i],   P_b = K[:, cols of b] V[cols of b],
// so one K.V is one launch of the UNCHANGED fused kernel (kmv_tc.cu / kmv_simt.cu) per column task over that task's segment, each
// into its own partial slots, and one combine pass that applies B row by row and scatters the rows back to user order into partial
// slot 0.  Every finish kernel and solver pass then runs as on a plain plan.  The segments cover about ntile_j + T - 1 column
// tiles per row tile, one copy of V is packed, and B never enters the fused kernels: their register budget is untouched.
//
// Gradients.  The derivative kinds (l dk/dl) run the same launches.  The task-covariance gradient
//     dB[a][b] = s sum_{i in a, j in b} (L_i . R_j) k_ij = s sum_{i in a} L_i . P_b[i]   (P_b of V = R)
// is the same set of launches without the combine, reduced by row task in a fixed order (rows of one task are contiguous).
// Nothing here uses atomics: repeated calls on one plan give identical bits.
#include <algorithm>

#include "gp_common.cuh"

namespace gp {

constexpr int TASK_RED_ROWS = 2048;                                                // sorted rows per block of the dB reduction

// dst[r] = src[map[r]] (width floats per row), zero where map[r] < 0
__global__ void task_gather_kernel(const float* __restrict__ src, int width, const int* __restrict__ map, int64_t nrows,
                                   float* __restrict__ dst) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nrows * width) return;
  const int64_t r = idx / width;
  const int c = (int)(idx % width);
  const int m = map[r];
  dst[idx] = (m >= 0) ? src[(int64_t)m * width + c] : 0.f;
}

// OUT[perm1[i]][c] = sum_slot B[t_i, task(slot)] tpart[slot][i][c]   (i in sorted row order, slots in a fixed order)
__global__ void task_combine_kernel(const float* __restrict__ tpart, int nslot, int64_t rows_pad, const int* __restrict__ slot_task,
                                    const int* __restrict__ ts1, const int* __restrict__ perm1, const float* __restrict__ B, int T,
                                    int64_t n1, float* __restrict__ out, const int* __restrict__ done_flag) {
  if (done_flag && *done_flag) return;
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n1 * TP) return;
  const int64_t i = idx / TP;
  const int c = (int)(idx % TP);
  const float* brow = B + (int64_t)ts1[i] * T;
  float s = 0.f;
  for (int sl = 0; sl < nslot; ++sl) s = fmaf(brow[slot_task[sl]], tpart[((int64_t)sl * rows_pad + i) * TP + c], s);
  out[(int64_t)perm1[i] * TP + c] = s;
}

// out[i][c] = B[t_i, b] L16[perm1[i]][c]   (sorted rows, B folded into the left factor of the SIMT derivative pass)
__global__ void task_scale_rows_kernel(const float* __restrict__ L16, const int* __restrict__ ts1, const int* __restrict__ perm1,
                                       const float* __restrict__ B, int T, int b, int64_t n1, float* __restrict__ out) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n1 * TP) return;
  const int64_t i = idx / TP;
  const int c = (int)(idx % TP);
  out[idx] = B[(int64_t)ts1[i] * T + b] * L16[(int64_t)perm1[i] * TP + c];
}

__global__ void task_scale_diag_kernel(float* __restrict__ out, const int* __restrict__ t1, const int* __restrict__ t2,
                                       const float* __restrict__ B, int T, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] *= B[(int64_t)t1[i] * T + t2[i]];
}

// rows of a valid index are scaled by B[t1[idx], t2[j]]; an out-of-range index already holds a NaN row
__global__ void task_scale_rows_out_kernel(float* __restrict__ out, int64_t ldo, const int64_t* __restrict__ idx, int64_t n1, int64_t n2,
                                           const int* __restrict__ t1, const int* __restrict__ t2, const float* __restrict__ B, int T) {
  const int64_t r = blockIdx.y;
  const int64_t i = idx[r];
  if (i < 0 || i >= n1) return;
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n2) out[r * ldo + j] *= B[(int64_t)t1[i] * T + t2[j]];
}

// dB reduction: block (chunk z of TASK_RED_ROWS sorted rows, column task b) writes out[(z T + b) T + a] = sum over its rows i of task a
// of L16[perm1[i]] . sum_{slots of b} tpart[slot][i]  (fp64, fixed tree; 0 for tasks absent from the chunk)
__global__ void __launch_bounds__(256)
task_dB_kernel(const float* __restrict__ tpart, int64_t rows_pad, const int* __restrict__ slot0, const int* __restrict__ ts1,
               const int* __restrict__ perm1, const float* __restrict__ L16, int T, int64_t n1, double* __restrict__ out,
               const int* __restrict__ xbad) {
  __shared__ double red[256];
  const int z = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int64_t r0 = (int64_t)z * TASK_RED_ROWS, r1 = min(n1, r0 + TASK_RED_ROWS);
  const int s0 = slot0[b], s1 = slot0[b + 1];
  const int a_lo = ts1[r0], a_hi = ts1[r1 - 1];   // sorted rows: the chunk holds tasks a_lo..a_hi only
  double* o = out + ((int64_t)z * T + b) * T;
  for (int a = tid; a < T; a += 256)
    if (a < a_lo || a > a_hi) o[a] = 0.0;
  for (int a = a_lo; a <= a_hi; ++a) {
    double acc = 0.0;
    for (int64_t i = r0 + tid; i < r1; i += 256) {
      if (ts1[i] != a) continue;
      const float* l = L16 + (int64_t)perm1[i] * TP;
      double v = 0.0;
      for (int c = 0; c < TP; ++c) {
        float pc = 0.f;
        for (int sl = s0; sl < s1; ++sl) pc += tpart[((int64_t)sl * rows_pad + i) * TP + c];
        v += (double)l[c] * (double)pc;
      }
      acc += v;
    }
    __syncthreads();
    red[tid] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
      if (tid < s) red[tid] += red[tid + s];
      __syncthreads();
    }
    if (tid == 0) o[a] = *xbad ? __longlong_as_double(0x7ff8000000000000LL) : red[0];
  }
}

// column splits of one segment: the rule of choose_geometry (pack.cu) over the segment's column tiles
static void segment_split(const gp_plan* p, bool tc, int64_t ntj, int64_t* tps, int* nsplit) {
  const int64_t nti = tc ? p->ntile_i : cdiv(p->row_count, SIMT_TI);
  int best = 1;
  double best_eff = -1.0;
  for (int s = 1; s <= 16; ++s) {
    if (s > ntj) break;
    int64_t per = cdiv(ntj, s);
    if (s > 1 && per < 8) break;
    int64_t units = nti * s;
    const int64_t slots = (int64_t)p->n_sm * (tc ? 2 : 1);
    int64_t waves = cdiv(units, slots);
    double eff = (double)(nti * ntj) / (double)(waves * slots * per);
    if (eff > best_eff + 0.02) { best_eff = eff; best = s; }
  }
  *tps = cdiv(ntj, best);
  *nsplit = (int)cdiv(ntj, *tps);
}

static int tasks_layout(gp_plan* p) {
  gp_task_state* ts = p->tasks;
  const bool tc = p->backend == GP_BACKEND_TCGEN05;
  const int T = ts->T;
  ts->seg.assign(T + 1, 0);
  ts->tps.assign(T, 0);
  ts->nsplit.assign(T, 0);
  ts->slot0.assign(T + 1, 0);
  for (int b = 0; b < T; ++b) {
    const int64_t cnt = ts->off2[b + 1] - ts->off2[b];
    ts->seg[b + 1] = ts->seg[b] + (tc ? cdiv(cnt, TILE_J) * TILE_J : cnt);
    if (cnt > 0) segment_split(p, tc, tc ? cdiv(cnt, TILE_J) : cdiv(cnt, SIMT_TJ), &ts->tps[b], &ts->nsplit[b]);
    ts->slot0[b + 1] = ts->slot0[b] + ts->nsplit[b];
  }
  ts->ncol_layout = ts->seg[T];
  const int nslot = ts->slot0[T];
  std::vector<int> h((size_t)ts->ncol_layout + nslot + T + 1, -1);
  for (int b = 0; b < T; ++b)
    for (int64_t k = 0; k < ts->off2[b + 1] - ts->off2[b]; ++k) h[(size_t)(ts->seg[b] + k)] = ts->perm2[(size_t)(ts->off2[b] + k)];
  int* st = h.data() + ts->ncol_layout;
  for (int b = 0; b < T; ++b)
    for (int s = ts->slot0[b]; s < ts->slot0[b + 1]; ++s) st[s] = b;
  for (int b = 0; b <= T; ++b) st[nslot + b] = ts->slot0[b];
  GP_CHECK(ts->lay.ensure(sizeof(int) * h.size()));
  ts->d_map2 = ts->lay.as<int>();
  ts->d_slot_task = ts->d_map2 + ts->ncol_layout;
  ts->d_slot0 = ts->d_slot_task + nslot;
  GP_CUDA(cudaMemcpyAsync(ts->d_map2, h.data(), sizeof(int) * h.size(), cudaMemcpyHostToDevice, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));   // h is a stack-lifetime vector
  ts->lay_ok = true;
  ts->lay_tc = tc;
  return GP_OK;
}

int tasks_pack(gp_plan* p) {
  gp_task_state* ts = p->tasks;
  const bool tc = p->backend == GP_BACKEND_TCGEN05;
  if (!ts->lay_ok || ts->lay_tc != tc) GP_CHECK(tasks_layout(p));
  cudaStream_t st = p->stream;
  const int DP = p->DP;
  const int64_t n1 = p->n1, ncol = ts->ncol_layout;
  const float* Zu1 = p->same ? p->Z2.as<float>() : p->Z1.as<float>();
  GP_CHECK(ts->Zs1.ensure(sizeof(float) * n1 * DP));
  GP_CHECK(ts->Zs2.ensure(sizeof(float) * ncol * DP));
  task_gather_kernel<<<(unsigned)cdiv(n1 * DP, 256), 256, 0, st>>>(Zu1, DP, ts->d_perm1, n1, ts->Zs1.as<float>());
  task_gather_kernel<<<(unsigned)cdiv(ncol * DP, 256), 256, 0, st>>>(p->Z2.as<float>(), DP, ts->d_map2, ncol, ts->Zs2.as<float>());
  p->launches += 2;
  if (tc) {
    GP_CHECK(p->XA.ensure(sizeof(float) * p->rows_pad * p->KP));
    GP_CHECK(p->XB.ensure(sizeof(float) * ncol * p->KP));
    GP_CHECK(pack_tc_rows(p, ts->Zs1.as<float>(), n1, p->rows_pad, true, p->XA.as<float>()));
    GP_CHECK(pack_tc_rows(p, ts->Zs2.as<float>(), ncol, ncol, false, p->XB.as<float>()));
    GP_CHECK(p->Vtiles.ensure(sizeof(float) * (ncol / TILE_J) * V_TILE_FLOATS));
  }
  GP_CHECK(ts->Vs.ensure(sizeof(float) * ncol * TP));
  GP_CHECK(ts->tpart.ensure(sizeof(float) * (size_t)std::max(1, ts->slot0[ts->T]) * p->rows_pad * TP));
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// per column task: P_b = K[:, b] V[b] into the task's partial slots (sorted rows)
static int tasks_segments(gp_plan* p, const float* V16, int kind, const int* done_flag) {
  gp_task_state* ts = p->tasks;
  const bool tc = p->backend == GP_BACKEND_TCGEN05;
  const int64_t ncol = ts->ncol_layout;
  float* Vs = ts->Vs.as<float>();
  task_gather_kernel<<<(unsigned)cdiv(ncol * TP, 256), 256, 0, p->stream>>>(V16, TP, ts->d_map2, ncol, Vs);
  p->launches++;
  if (tc) GP_CHECK(pack_v_tiles_rows(p, Vs, ncol, ncol / TILE_J, p->Vtiles.as<float>()));
  for (int b = 0; b < ts->T; ++b) {
    if (ts->nsplit[b] == 0) continue;
    const int64_t cnt = ts->off2[b + 1] - ts->off2[b];
    float* part = ts->tpart.as<float>() + (size_t)ts->slot0[b] * p->rows_pad * TP;
    if (tc) {
      GP_CHECK(kmv_tc_launch_cols(p, kind, p->XA.as<float>(), p->XB.as<float>() + ts->seg[b] * p->KP,
                                  p->Vtiles.as<float>() + (ts->seg[b] / TILE_J) * V_TILE_FLOATS, part, cdiv(cnt, TILE_J), ts->tps[b],
                                  ts->nsplit[b], -ts->off2[b], done_flag));
    } else {
      GP_CHECK(kmv_simt_launch_cols(p, kind, ts->Zs1.as<float>(), ts->Zs2.as<float>() + ts->seg[b] * p->DP, Vs + ts->seg[b] * TP, part,
                                    cnt, ts->tps[b] * SIMT_TJ, ts->nsplit[b], -ts->off2[b], done_flag));
    }
  }
  return GP_OK;
}

int tasks_kmv_partials(gp_plan* p, const float* V16, int kind, const int* done_flag) {
  gp_task_state* ts = p->tasks;
  GP_REQUIRE(ts->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  GP_CHECK(tasks_segments(p, V16, kind, done_flag));
  task_combine_kernel<<<(unsigned)cdiv(p->n1 * TP, 256), 256, 0, p->stream>>>(
      ts->tpart.as<float>(), ts->slot0[ts->T], p->rows_pad, ts->d_slot_task, ts->d_ts1, ts->d_perm1, ts->Bd.as<float>(), ts->T, p->n1,
      p->partial.as<float>(), done_flag);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int tasks_kdiag_scale(gp_plan* p, float* OUT) {
  gp_task_state* ts = p->tasks;
  GP_REQUIRE(ts->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  task_scale_diag_kernel<<<(unsigned)cdiv(p->row_count, 256), 256, 0, p->stream>>>(OUT, ts->d_t1, p->same ? ts->d_t1 : ts->d_t2,
                                                                                  ts->Bd.as<float>(), ts->T, p->row_count);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int tasks_krows_scale(gp_plan* p, const int64_t* idx, int64_t m, float* OUT, int64_t ldo) {
  gp_task_state* ts = p->tasks;
  GP_REQUIRE(ts->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  dim3 grid((unsigned)cdiv(p->n2, 256), (unsigned)m);
  task_scale_rows_out_kernel<<<grid, 256, 0, p->stream>>>(OUT, ldo, idx, p->row_count, p->n2, ts->d_t1, p->same ? ts->d_t1 : ts->d_t2,
                                                          ts->Bd.as<float>(), ts->T);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// SIMT derivative pass (ARD, or a SIMT plan): one bilinear launch per column task with B[t_i, b] folded into the sorted left rows
int tasks_bilinear(gp_plan* p, const float* L16, const float* R16, bool ard, std::vector<double>& total) {
  gp_task_state* ts = p->tasks;
  GP_REQUIRE(ts->b_set, GP_E_STATE, "task covariance not set (gp_plan_set_task_covar)");
  const int nout = 1 + (ard ? p->d : 1);
  const int64_t ncol = ts->ncol_layout, n1 = p->n1;
  GP_CHECK(ts->Ls.ensure(sizeof(float) * n1 * TP));   // one B-scaled left factor, rewritten per task (stream order)
  float* Rs = ts->Vs.as<float>();
  task_gather_kernel<<<(unsigned)cdiv(ncol * TP, 256), 256, 0, p->stream>>>(R16, TP, ts->d_map2, ncol, Rs);
  p->launches++;
  // block partials of every task's launch back to back, then one fixed-order fp64 sum on the host
  int64_t nblk_tot = 0;
  for (int b = 0; b < ts->T; ++b)
    if (ts->off2[b + 1] > ts->off2[b]) nblk_tot += bilinear_blocks(p, ts->off2[b + 1] - ts->off2[b]);
  GP_CHECK(p->misc.ensure(sizeof(double) * (nblk_tot * nout + 1)));
  double* gout = p->misc.as<double>();
  int64_t off = 0;
  for (int b = 0; b < ts->T; ++b) {
    const int64_t cnt = ts->off2[b + 1] - ts->off2[b];
    if (cnt == 0) continue;
    float* Lb = ts->Ls.as<float>();
    task_scale_rows_kernel<<<(unsigned)cdiv(n1 * TP, 256), 256, 0, p->stream>>>(L16, ts->d_ts1, ts->d_perm1, ts->Bd.as<float>(), ts->T, b,
                                                                                 n1, Lb);
    p->launches++;
    int64_t nb = 0;
    GP_CHECK(bilinear_launch_cols(p, ard, ts->Zs1.as<float>(), ts->Zs2.as<float>() + ts->seg[b] * p->DP, Lb, Rs + ts->seg[b] * TP, cnt,
                                  -ts->off2[b], gout + off * nout, nout, &nb));
    off += nb;
  }
  std::vector<double> h((size_t)nblk_tot * nout);
  int xb = 0;
  GP_CUDA(cudaMemcpyAsync(h.data(), p->misc.as<double>(), sizeof(double) * h.size(), cudaMemcpyDeviceToHost, p->stream));
  GP_CUDA(cudaMemcpyAsync(&xb, p->xbad, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));
  for (int o = 0; o < nout; ++o) {
    double s = 0.0;
    for (int64_t k = 0; k < nblk_tot; ++k) s += h[(size_t)k * nout + o];
    total[o] += xb ? NAN : s;
  }
  return GP_OK;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_plan_set_tasks(gp_plan* p, const int32_t* task1, const int32_t* task2, int T) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_CUDA(cudaSetDevice(p->device));
  if (task1 == nullptr) {
    if (p->tasks) {
      gp::DevBuf* bufs[] = {&p->tasks->ids, &p->tasks->lay, &p->tasks->Bd, &p->tasks->Zs1, &p->tasks->Zs2, &p->tasks->Vs, &p->tasks->Ls,
                            &p->tasks->tpart, &p->tasks->red};
      GP_CUDA(cudaStreamSynchronize(p->stream));
      for (auto* b : bufs) b->release();
      delete p->tasks;
      p->tasks = nullptr;
      if (p->data_set && p->hypers_set) return pack_inputs(p);
    }
    return GP_OK;
  }
  GP_CHECK(refuse_settings(p, CALL_SET_TASKS));
  GP_REQUIRE(p->data_set, GP_E_STATE, "gp_plan_set_tasks: call gp_plan_set_data first");
  GP_REQUIRE(T >= 1 && T <= 32, GP_E_SHAPE, "number of tasks T=%d not in [1, 32]", T);
  GP_REQUIRE(p->ski == nullptr && p->backend != GP_BACKEND_SKI, GP_E_STATE, "task indices are not available on a SKI plan");
  GP_REQUIRE(p->backend_req != GP_BACKEND_SUM, GP_E_STATE, "task indices are not available on a kernel-sum plan");
  GP_CHECK(refuse_settings(p, CALL_SET_TASKS_LOWRANK));
  GP_REQUIRE(p->row_begin == 0 && p->row_count == p->n1 && !(p->comm && p->comm->world > 1), GP_E_SHAPE,
             "task indices are not available on a row-sharded plan");
  GP_REQUIRE(p->same ? (task2 == nullptr || task2 == task1) : task2 != nullptr, GP_E_SHAPE,
             p->same ? "a square plan takes one task array (task2 = NULL)" : "a cross plan needs the task ids of both inputs");
  GP_REQUIRE(p->n1 < ((int64_t)1 << 31) && p->n2 < ((int64_t)1 << 31), GP_E_SHAPE, "too many rows for task indices");
  const int64_t n1 = p->n1, n2 = p->n2;
  std::vector<int> t1(n1), t2;
  GP_CUDA(cudaMemcpyAsync(t1.data(), task1, sizeof(int) * n1, cudaMemcpyDeviceToHost, p->stream));
  if (!p->same) {
    t2.resize(n2);
    GP_CUDA(cudaMemcpyAsync(t2.data(), task2, sizeof(int) * n2, cudaMemcpyDeviceToHost, p->stream));
  }
  GP_CUDA(cudaStreamSynchronize(p->stream));
  for (int64_t i = 0; i < n1; ++i)
    GP_REQUIRE(t1[i] >= 0 && t1[i] < T, GP_E_SHAPE, "task index %d of row %lld outside [0, %d)", t1[i], (long long)i, T);
  for (size_t j = 0; j < t2.size(); ++j)
    GP_REQUIRE(t2[j] >= 0 && t2[j] < T, GP_E_SHAPE, "task index %d of column %lld outside [0, %d)", t2[j], (long long)j, T);
  gp_task_state* ts = p->tasks ? p->tasks : new gp_task_state();
  const bool had_b = p->tasks && ts->T == T && ts->b_set;
  ts->T = T;
  ts->t1 = t1;
  ts->t2 = p->same ? t1 : t2;
  // stable counting sort by task
  auto sort_by_task = [T](const std::vector<int>& t, std::vector<int64_t>& off, std::vector<int>& perm) {
    off.assign(T + 1, 0);
    for (int v : t) off[v + 1]++;
    for (int b = 0; b < T; ++b) off[b + 1] += off[b];
    std::vector<int64_t> next(off.begin(), off.end() - 1);
    perm.assign(t.size(), 0);
    for (size_t i = 0; i < t.size(); ++i) perm[(size_t)next[t[i]]++] = (int)i;
  };
  sort_by_task(ts->t1, ts->off1, ts->perm1);
  sort_by_task(ts->t2, ts->off2, ts->perm2);
  std::vector<int> h((size_t)3 * n1 + n2);
  for (int64_t i = 0; i < n1; ++i) {
    h[(size_t)i] = ts->perm1[(size_t)i];
    h[(size_t)(n1 + i)] = ts->t1[(size_t)ts->perm1[(size_t)i]];
    h[(size_t)(2 * n1 + i)] = ts->t1[(size_t)i];
  }
  for (int64_t j = 0; j < n2; ++j) h[(size_t)(3 * n1 + j)] = ts->t2[(size_t)j];
  p->tasks = ts;
  ts->lay_ok = false;
  if (!had_b) ts->b_set = false;
  GP_CHECK(ts->ids.ensure(sizeof(int) * h.size()));
  ts->d_perm1 = ts->ids.as<int>();
  ts->d_ts1 = ts->d_perm1 + n1;
  ts->d_t1 = ts->d_ts1 + n1;
  ts->d_t2 = ts->d_t1 + n1;
  GP_CUDA(cudaMemcpyAsync(ts->d_perm1, h.data(), sizeof(int) * h.size(), cudaMemcpyHostToDevice, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));   // h is a stack-lifetime vector
  if (p->hypers_set) return pack_inputs(p);
  return GP_OK;
}

extern "C" int gp_plan_set_task_covar(gp_plan* p, const float* B, int T) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  if (p->kron) return kron_set_task_covar(p, B, T);   // the B of (s K) (x) B (kron.cu)
  GP_REQUIRE(p->tasks != nullptr, GP_E_STATE, "gp_plan_set_task_covar: no task indices (gp_plan_set_tasks)");
  GP_REQUIRE(B != nullptr && T == p->tasks->T, GP_E_SHAPE, "task covariance must be %d x %d (got T=%d)", p->tasks->T, p->tasks->T, T);
  GP_CUDA(cudaSetDevice(p->device));
  gp_task_state* ts = p->tasks;
  ts->B.assign(B, B + (size_t)T * T);
  GP_CHECK(ts->Bd.ensure(sizeof(float) * T * T));
  GP_CUDA(cudaMemcpyAsync(ts->Bd.p, ts->B.data(), sizeof(float) * T * T, cudaMemcpyHostToDevice, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));   // the next call may replace ts->B
  ts->b_set = true;
  return GP_OK;
}

extern "C" int gp_task_covar_grad(gp_plan* p, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  if (p->kron) return kron_task_covar_grad_checked(p, L, ldl, R, ldr, t, dB);   // dB of (s K) (x) B (kron.cu)
  GP_REQUIRE(p->tasks != nullptr, GP_E_STATE, "gp_task_covar_grad: no task indices (gp_plan_set_tasks)");
  GP_REQUIRE(t >= 1 && L && R && dB, GP_E_SHAPE, "gp_task_covar_grad: bad arguments");
  GP_REQUIRE((ldl >= t || p->n1 == 1) && (ldr >= t || p->n2 == 1), GP_E_SHAPE,
             "gp_task_covar_grad: leading dimensions must be >= t (ldl=%lld, ldr=%lld, t=%d)", (long long)ldl, (long long)ldr, t);
  GP_CUDA(cudaSetDevice(p->device));
  gp_task_state* ts = p->tasks;
  const int T = ts->T;
  const int64_t n1 = p->n1;
  const int nz = (int)cdiv(n1, TASK_RED_ROWS);
  GP_CHECK(p->misc2.ensure(sizeof(float) * n1 * TP));
  GP_CHECK(p->misc3.ensure(sizeof(float) * p->n2 * TP));
  GP_CHECK(ts->red.ensure(sizeof(double) * (size_t)nz * T * T));
  std::vector<double> acc((size_t)T * T, 0.0), h((size_t)nz * T * T);
  for (int c0 = 0; c0 < t; c0 += TP) {
    const int tc = std::min(TP, t - c0);
    GP_CHECK(to_v16(p, L + c0, ldl, tc, n1, p->misc2.as<float>()));
    GP_CHECK(to_v16(p, R + c0, ldr, tc, p->n2, p->misc3.as<float>()));
    GP_CHECK(tasks_segments(p, p->misc3.as<float>(), p->kind, nullptr));
    task_dB_kernel<<<dim3((unsigned)nz, (unsigned)T), 256, 0, p->stream>>>(ts->tpart.as<float>(), p->rows_pad, ts->d_slot0, ts->d_ts1,
                                                                           ts->d_perm1, p->misc2.as<float>(), T, n1, ts->red.as<double>(),
                                                                           p->xbad);
    p->launches++;
    GP_CUDA(cudaGetLastError());
    GP_CUDA(cudaMemcpyAsync(h.data(), ts->red.as<double>(), sizeof(double) * h.size(), cudaMemcpyDeviceToHost, p->stream));
    GP_CUDA(cudaStreamSynchronize(p->stream));
    for (int z = 0; z < nz; ++z)
      for (int b = 0; b < T; ++b)
        for (int a = 0; a < T; ++a) acc[(size_t)a * T + b] += h[((size_t)z * T + b) * T + a];
  }
  for (int e = 0; e < T * T; ++e) dB[e] = (double)p->outputscale * acc[(size_t)e];
  return GP_OK;
}
