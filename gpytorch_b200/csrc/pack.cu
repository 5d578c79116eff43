// pack.cu -- input re-packing for the fused K.V kernels.
//
// The reference scales inputs by 1/lengthscale and mean-centres them before forming distances
// (kernels/kernel.py:29-30, functions/matern_covariance.py:19-21).  We do the same once per
// hyper-parameter update and additionally fold the covariance constant into the scale so that the
// fused kernels evaluate  a_ij = -0.5 |z_i - z_j|^2  and k = f(a) with one ex2 (gp_common.cuh).
//
// HBM layouts produced here
//   Z2   [n2][DP]            fp32, zero padded features           (SIMT kernel, row extraction)
//   Z1   [n1_local][DP]      only when X2 != X1 (otherwise Z1 aliases Z2 + row_begin*DP)
//   XA   [ntile_i][KP/4][128][4]   wgmma K-major no-swizzle tiles of the A operand
//                                  [z_hi | z_lo | z_hi | n_hi n_lo 1 1 | 0..]   (3xTF32 split)
//   XB   [ntile_j][KP/4][ 64][4]   B operand  [z_hi | z_hi | z_lo | 1 1 n_hi n_lo | 0..], the columns of every 8-column
//                                  group stored in the order 0 4 1 5 2 6 3 7 (kmv_tc.cu: the GEMM1 accumulator is then the
//                                  tf32 A fragment of GEMM2)
//   so that  sum_k A_ik B_jk = z_i.z_j (to ~2^-22) + n_i + n_j,  n = -0.5 |z|^2  = a_ij.
//   Vt   per 64-row tile: [64/4][32][4] tf32 (rows 0-15 hi, 16-31 lo) + [64/8][16][8] bf16  (B operands of GEMM2)
#include <stdlib.h>

#include "gp_common.cuh"

namespace gp {

__global__ void col_mean_kernel(const float* __restrict__ X, int64_t n, int64_t ld, int d, float* __restrict__ mean) {
  int c = blockIdx.x;
  double acc = 0.0;
  for (int64_t r = threadIdx.x; r < n; r += blockDim.x) acc += (double)X[r * ld + c];
  __shared__ double sh[256];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) mean[c] = (float)(sh[0] / (double)n);
}

__global__ void pack_simt_kernel(const float* __restrict__ X, int64_t n, int64_t ld, int d, int DP,
                                 const float* __restrict__ mean, const float* __restrict__ scale,
                                 float* __restrict__ Z, int* __restrict__ xbad) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * DP) return;
  int64_t r = idx / DP;
  int c = (int)(idx % DP);
  float z = (c < d) ? (X[r * ld + c] - mean[c]) * scale[c] : 0.f;
  Z[idx] = z;
  // a NaN/Inf anywhere in the inputs makes every entry of K (hence of K.V) NaN in the reference (mean-centring in
  // kernels/kernel.py:35-37 spreads it); the covariance code clamps with fmin/fmax, which would swallow it, so record it
  if (!(fabsf(z) <= 3.402823466e38f)) *xbad = 1;
}

// one thread per (padded) row; writes KP floats as KP/4 float4 (coalesced across rows)
// off >= 0: a polynomial plan (DESIGN 4.21).  Its rows are the raw inputs and the spare columns carry the offset instead of the
// norms: A [z_hi | z_lo | z_hi | c_hi c_lo 1 1 | 0..], B [z_hi | z_hi | z_lo | 1 1 0 0 | 0..], so GEMM1 gives a = z_i.z_j + c
template <bool IS_A>
__global__ void pack_tc_kernel(const float* __restrict__ Z, int64_t row0, int64_t nrows_valid, int64_t nrows_pad,
                               int d, int DP, int KP, int tile_rows, float* __restrict__ out, float off) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // local padded row
  if (r >= nrows_pad) return;
  int64_t tile = r / tile_rows;
  int rr = (int)(r % tile_rows);
  if (!IS_A) rr = (rr & ~7) | ((rr & 4) ? 2 * (rr & 3) + 1 : 2 * (rr & 3));   // column c of a group -> position 2 (c % 4) + c / 4
  float4* dst = reinterpret_cast<float4*>(out + tile * (int64_t)tile_rows * KP);
  const bool valid = r < nrows_valid;
  const float* z = Z + (row0 + r) * DP;
  const bool poly = off >= 0.f;
  double nn = 0.0;
  if (valid && !poly)
    for (int c = 0; c < d; ++c) nn += (double)z[c] * (double)z[c];
  nn *= -0.5;
  if (poly && IS_A) nn = (double)off;   // B keeps n = 0: its columns (1, 1, 0, 0) pick c_hi + c_lo
  float n_hi = tf32_hi((float)nn);
  float n_lo = tf32_hi((float)(nn - (double)n_hi));
  for (int kc = 0; kc < KP / 4; ++kc) {
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      int kk = kc * 4 + q;
      float val = 0.f;
      if (valid) {
        if (kk < 3 * d) {
          int seg = kk / d, c = kk % d;
          float zz = z[c];
          float hi = tf32_hi(zz);
          float lo = tf32_hi(zz - hi);
          // A: hi lo hi ; B: hi hi lo
          bool want_lo = IS_A ? (seg == 1) : (seg == 2);
          val = want_lo ? lo : hi;
        } else {
          int e = kk - 3 * d;
          if (IS_A) val = (e == 0) ? n_hi : (e == 1) ? n_lo : (e < 4 ? 1.f : 0.f);
          else      val = (e < 2) ? 1.f : (e == 2) ? n_hi : (e == 3 ? n_lo : 0.f);
        }
      }
      v[q] = val;
    }
    dst[(int64_t)kc * tile_rows + rr] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

__global__ void to_v16_kernel(const float* __restrict__ V, int64_t ldv, int t, int64_t n, float* __restrict__ V16) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * TP) return;
  int64_t r = idx / TP;
  int c = (int)(idx % TP);
  V16[idx] = (c < t) ? V[r * ldv + c] : 0.f;
}

// thread per (4-row chunk, column): V16 [n2][16] -> Vt tiles.  Per 64-row tile (10240 B):
//   [0, 8192)      tf32 tile  [64/4][32 rows][4]: rows 0-15 = hi, rows 16-31 = lo of the 16 columns
//   [8192, 10240)  bf16 tile  [64/8][16 rows][8]: bf16(v), the B operand of the P_lo pass
__global__ void pack_v_tiles_kernel(const float* __restrict__ V16, int64_t n2, int64_t ntile_j, float* __restrict__ Vt) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nchunk = ntile_j * (TILE_J / 4);
  if (idx >= nchunk * TP) return;
  int c = (int)(idx % TP);
  int64_t chunk = idx / TP;
  int64_t tile = chunk / (TILE_J / 4);
  int kc = (int)(chunk % (TILE_J / 4));
  int64_t j0 = tile * TILE_J + kc * 4;
  float hi[4], lo[4], v[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    int64_t j = j0 + q;
    v[q] = (j < n2) ? V16[j * TP + c] : 0.f;
    hi[q] = tf32_hi(v[q]);
    lo[q] = tf32_hi(v[q] - hi[q]);
  }
  float* tbase = Vt + tile * (int64_t)V_TILE_FLOATS;
  float4* base = reinterpret_cast<float4*>(tbase);
  base[kc * (2 * TP) + c] = make_float4(hi[0], hi[1], hi[2], hi[3]);        // B rows 0..15  = V_hi columns
  base[kc * (2 * TP) + TP + c] = make_float4(lo[0], lo[1], lo[2], lo[3]);   // B rows 16..31 = V_lo columns
  // bf16 tile: element (row c, k = kc*4+q) at [(k/8)][c][k%8]
  uint32_t w0, w1;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w0) : "f"(v[1]), "f"(v[0]));
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w1) : "f"(v[3]), "f"(v[2]));
  uint2* wb = reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(tbase) + 2 * TILE_J * TP * 4);
  wb[((kc >> 1) * TP + c) * 2 + (kc & 1)] = make_uint2(w0, w1);
}

static int round_dp(int d) {
  const int opts[] = {4, 8, 12, 16, 24, 32, 48, 64, 96, 128};
  for (int o : opts)
    if (d <= o) return o;
  return -1;
}

int choose_geometry(gp_plan* p) {
  const int w = packed_dims(p);   // 2d embedding columns on a periodic plan
  p->DP = round_dp(w);
  GP_REQUIRE(p->DP > 0, GP_E_SHAPE, "input dimension d=%d > 128 is not supported", p->d);
  int kp = 3 * w + 4;
  p->KP = ((kp + 7) / 8) * 8;
  int want = p->backend_req;
  if (want == GP_BACKEND_AUTO) want = (p->KP <= KP_MAX) ? GP_BACKEND_TCGEN05 : GP_BACKEND_SIMT;
  if (p->add_M) want = GP_BACKEND_SIMT;   // additive plans run their own CUDA-core kernels on Z (additive.cu)
  if (p->sm_Q) want = GP_BACKEND_SIMT;    // so do spectral plans, on their own packed rows (spectral.cu)
  if (p->compact) want = GP_BACKEND_COMPACT;   // piecewise polynomial plans run their tile-pair lists (compact.cu)
  GP_REQUIRE(!(want == GP_BACKEND_TCGEN05 && p->KP > KP_MAX), GP_E_SHAPE,
             "tcgen05 (tensor-core) backend needs 3d+4 <= %d (d=%d)", KP_MAX, p->d);
  p->backend = want;
  p->rows_pad = cdiv(p->row_count, 2 * TILE_I) * 2 * TILE_I;
  p->ntile_i = p->rows_pad / TILE_I;
  p->ntile_j = cdiv(p->n2, TILE_J);
  choose_splits(p, p->backend == GP_BACKEND_TCGEN05);
  return GP_OK;
}

// column splits: pick the smallest nsplit whose unit count fills the SMs best
void choose_splits(gp_plan* p, bool tc) {
  int64_t nti = tc ? p->ntile_i : cdiv(p->row_count, SIMT_TI);
  int64_t ntj = tc ? p->ntile_j : cdiv(p->n2, SIMT_TJ);
  int best = 1;
  double best_eff = -1.0;
  for (int s = 1; s <= 16; ++s) {
    if (s > ntj) break;
    int64_t per = cdiv(ntj, s);
    if (s > 1 && per < 8) break;  // keep units long enough to amortise the prologue
    int64_t units = nti * s;
    // 2 slots per SM on the tensor-core path: the K.V kernel now runs one 384-thread CTA per SM, but the factor is kept so
    // that the work units -- and with them the split of every row sum into partials, hence the results bit for bit -- stay
    // what they were
    const int64_t slots = (int64_t)p->n_sm * (tc ? 2 : 1);
    int64_t waves = cdiv(units, slots);
    double eff = (double)(nti * ntj) / (double)(waves * slots * per);
    if (eff > best_eff + 0.02) { best_eff = eff; best = s; }
  }
  p->tiles_per_split = cdiv(ntj, best);
  p->nsplit = (int)cdiv(ntj, p->tiles_per_split);  // no empty splits
}

int pack_inputs(gp_plan* p) {
  GP_REQUIRE(p->data_set && p->hypers_set, GP_E_STATE, "set_data and set_hypers must both be called");
  if (p->backend == GP_BACKEND_SKI) return ski_pack(p);
  if (p->backend_req == GP_BACKEND_SUM) return sum_pack(p);
  if (p->backend_req == GP_BACKEND_KRON) return kron_pack(p);
  if (p->backend_req == GP_BACKEND_DERIV) return deriv_pack(p);
  if (p->backend_req == GP_BACKEND_PRODUCT) return product_pack(p);
  p->pack_gen++;   // a kernel product over this plan re-reads its scale, geometry and flag (product.cu)
  GP_CHECK(choose_geometry(p));
  if (p->sm_Q) return spectral_pack(p);
  if (p->per_n) return periodic_pack(p);
  cudaStream_t st = p->stream;
  const int d = p->d, DP = p->DP;
  GP_CHECK(p->mean.ensure(sizeof(float) * (d + 4)));
  p->xbad = reinterpret_cast<int*>(p->mean.as<float>() + d);
  GP_CUDA(cudaMemsetAsync(p->xbad, 0, sizeof(int), st));
  GP_CHECK(p->scale.ensure(sizeof(float) * d));
  // scale_c = sqrt(const) / l_c
  std::vector<float> sc(d);
  // RQ: C = 1 (alpha stays out of the packing, so the value and both derivatives read the same a = -r^2 / 2)
  double cst = (p->kind == GP_RBF) ? 1.4426950408889634
               : (p->kind == GP_MATERN12 ? 2.0 : (p->kind == GP_MATERN32 ? 6.0 : (p->kind == GP_RQ || p->kind == GP_PPOLY ? 1.0 : 10.0)));
  const bool poly = p->kind == GP_POLY;   // a dot-product kernel: the raw inputs, no centring and no scale (DESIGN 4.21)
  for (int c = 0; c < d; ++c) {
    double l = (p->ls.size() == 1) ? p->ls[0] : p->ls[c];
    sc[c] = poly ? 1.f : (float)(sqrt(cst) / l);
  }
  GP_CUDA(cudaMemcpyAsync(p->scale.p, sc.data(), sizeof(float) * d, cudaMemcpyHostToDevice, st));
  GP_CUDA(cudaStreamSynchronize(st));  // sc is a stack-lifetime vector
  if (poly) {
    GP_CUDA(cudaMemsetAsync(p->mean.p, 0, sizeof(float) * d, st));
  } else {
    col_mean_kernel<<<d, 256, 0, st>>>(p->X1, p->n1, p->ld1, d, p->mean.as<float>());
    p->launches++;
  }
  const float* X2 = p->same ? p->X1 : p->X2;
  int64_t ld2 = p->same ? p->ld1 : p->ld2;
  GP_CHECK(p->Z2.ensure(sizeof(float) * p->n2 * DP));
  {
    int64_t tot = p->n2 * DP;
    pack_simt_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, st>>>(X2, p->n2, ld2, d, DP, p->mean.as<float>(),
                                                              p->scale.as<float>(), p->Z2.as<float>(), p->xbad);
    p->launches++;
  }
  if (!p->same) {
    GP_CHECK(p->Z1.ensure(sizeof(float) * p->row_count * DP));
    int64_t tot = p->row_count * DP;
    pack_simt_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, st>>>(p->X1 + p->row_begin * p->ld1, p->row_count, p->ld1, d, DP,
                                                              p->mean.as<float>(), p->scale.as<float>(), p->Z1.as<float>(), p->xbad);
    p->launches++;
  }
  if (p->tasks) {
    GP_CHECK(tasks_pack(p));   // task-sorted packing and the per-task column segments (tasks.cu)
  } else if (p->backend == GP_BACKEND_TCGEN05) {
    const int KP = p->KP;
    int64_t padA = p->rows_pad, padB = p->ntile_j * TILE_J;
    GP_CHECK(p->XA.ensure(sizeof(float) * padA * KP));
    GP_CHECK(p->XB.ensure(sizeof(float) * padB * KP));
    const float* ZA = p->same ? p->Z2.as<float>() : p->Z1.as<float>();
    int64_t rowA0 = p->same ? p->row_begin : 0;
    const float off = poly ? p->poly_offset : -1.f;
    pack_tc_kernel<true><<<(unsigned)cdiv(padA, 128), 128, 0, st>>>(ZA, rowA0, p->row_count, padA, d, DP, KP, TILE_I, p->XA.as<float>(), off);
    pack_tc_kernel<false><<<(unsigned)cdiv(padB, 128), 128, 0, st>>>(p->Z2.as<float>(), 0, p->n2, padB, d, DP, KP, TILE_J, p->XB.as<float>(), off);
    p->launches += 2;
    GP_CHECK(p->Vtiles.ensure(sizeof(float) * p->ntile_j * (2 * TILE_J * TP + TILE_J * TP / 2)));
  }
  p->nparts = p->tasks ? 1 : p->nsplit;   // a Hadamard product is combined into one slot in user row order
  if (p->add_M) GP_CHECK(additive_pack(p));
  if (p->compact) GP_CHECK(compact_pack(p));   // sets nparts: the slots of the longest tile-pair list
  GP_CHECK(p->partial.ensure(sizeof(float) * (size_t)nslots(p) * p->rows_pad * TP));
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int to_v16(gp_plan* p, const float* V, int64_t ldv, int t, int64_t n, float* V16) {
  int64_t tot = n * TP;
  to_v16_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, p->stream>>>(V, ldv, t, n, V16);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

// tensor-core operand tiles of rows [0, npad) of Z (rows >= nvalid zero): the A side (XA layout) or the B side (XB layout)
int pack_tc_rows(gp_plan* p, const float* Z, int64_t nvalid, int64_t npad, bool is_a, float* out) {
  const int w = packed_dims(p);
  if (is_a) pack_tc_kernel<true><<<(unsigned)cdiv(npad, 128), 128, 0, p->stream>>>(Z, 0, nvalid, npad, w, p->DP, p->KP, TILE_I, out, -1.f);
  else pack_tc_kernel<false><<<(unsigned)cdiv(npad, 128), 128, 0, p->stream>>>(Z, 0, nvalid, npad, w, p->DP, p->KP, TILE_J, out, -1.f);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

int pack_v_tiles(gp_plan* p, const float* V16) {
  return pack_v_tiles_rows(p, V16, p->n2, p->ntile_j, p->Vtiles.as<float>());
}

int pack_v_tiles_rows(gp_plan* p, const float* V16, int64_t nrows, int64_t ntiles, float* Vt) {
  int64_t tot = ntiles * (TILE_J / 4) * TP;
  pack_v_tiles_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, p->stream>>>(V16, nrows, ntiles, Vt);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  return GP_OK;
}

}  // namespace gp
