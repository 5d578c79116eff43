// lanczos.cu -- Lanczos tridiagonalisation with full re-orthogonalisation of (K + noise I).
//
// Restates linear_operator.utils.lanczos.lanczos_tridiag (SURVEY.md Appendix A.6), the routine behind
// root_decomposition / root_inv_decomposition (LOVE caches, /root/reference/gpytorch/models/
// exact_prediction_strategies.py:268-272).  One start vector; the matrix product is the fused K.V kernel;
// the Gram-Schmidt passes are two skinny GEMVs against the stored basis Qt [J][n].
#include <math.h>

#include <algorithm>

#include "gp_common.cuh"

namespace gp {

// part[blk] = sum a.b over the block's slice (fp64)
__global__ void lz_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, double* __restrict__ part) {
  __shared__ double sh[256];
  double acc = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    acc += (double)a[i] * (double)b[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}
__global__ void lz_sum_kernel(const double* __restrict__ part, int g, double* __restrict__ out, int do_sqrt) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < g; ++i) s += part[i];
    *out = do_sqrt ? sqrt(s) : s;
  }
}
// r = r - (*coef) * q     (coef on device)
__global__ void lz_axpy_kernel(float* __restrict__ r, const float* __restrict__ q, const double* __restrict__ coef, int64_t n) {
  const float c = (float)(*coef);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    r[i] = fmaf(-c, q[i], r[i]);
}
// out = r / (*nrm)
__global__ void lz_scale_kernel(const float* __restrict__ r, const double* __restrict__ nrm, int64_t n, float* __restrict__ out) {
  const float inv = (float)(1.0 / *nrm);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = r[i] * inv;
}
// c[a] = Qt[a] . r   (one CTA per basis vector); also cmax = max_a c[a] via atomicMax on an int-encoded double? -> host
__global__ void lz_gemv_t_kernel(const float* __restrict__ Qt, int64_t n, const float* __restrict__ r, double* __restrict__ c) {
  __shared__ double sh[256];
  const float* q = Qt + (int64_t)blockIdx.x * n;
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) acc += (double)q[i] * (double)r[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) c[blockIdx.x] = sh[0];
}
// r[j] -= sum_a Qt[a][j] c[a]
__global__ void lz_gemv_n_kernel(const float* __restrict__ Qt, int m, int64_t n, const double* __restrict__ c, float* __restrict__ r) {
  extern __shared__ float cs[];
  for (int a = threadIdx.x; a < m; a += blockDim.x) cs[a] = (float)c[a];
  __syncthreads();
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int a = 0; a < m; ++a) s = fmaf(Qt[(int64_t)a * n + j], cs[a], s);
    r[j] -= s;
  }
}

__global__ void lz_sqrt_kernel(double* v) { *v = sqrt(*v); }

}  // namespace gp

using namespace gp;

extern "C" int gp_lanczos(gp_plan* p, const float* INIT, int max_iter, float tol, float* Qt, float* T, int* J_out) {
  GP_REQUIRE(p && p->data_set && p->hypers_set, GP_E_STATE, "plan not ready");
  GP_REQUIRE(p->same, GP_E_SHAPE, "Lanczos needs a square operator");
  GP_REQUIRE(max_iter >= 1, GP_E_SHAPE, "max_iter must be >= 1");
  KronColsScope kcols(p, 1);   // one Lanczos vector per product
  cudaStream_t st = p->stream;
  // row-sharded runs (one process per GPU): every vector (INIT, the basis rows of Qt, r) holds this rank's rows only; the
  // products all-gather the current basis vector, the dots / Gram-Schmidt coefficients are all-reduced (fp64)
  const bool sharded = p->comm && p->comm->world > 1;
  const int64_t N = p->n2;
  const int64_t n = p->row_count;
  GP_REQUIRE(!sharded || (n * p->comm->world == N && p->row_begin == (int64_t)p->comm->rank * n), GP_E_SHAPE,
             "row-sharded Lanczos needs equal contiguous shards");
  const int num_iter = (int)std::min<int64_t>(max_iter, N);
  const int G = 2 * p->n_sm;
  GP_CHECK(p->misc.ensure(sizeof(float) * (n + 2) + sizeof(double) * (G + num_iter + 16)));
  GP_CHECK(p->V16.ensure(sizeof(float) * N * TP));
  if (sharded) GP_CHECK(p->cgPfull.ensure(sizeof(float) * N));
  float* qfull = sharded ? p->cgPfull.as<float>() : nullptr;
  float* r = p->misc.as<float>();
  double* part = reinterpret_cast<double*>(r + ((n + 1) / 2) * 2);
  double* ds = part + G;            // device scalars: [0] alpha [1] beta / norm
  double* cvec = ds + 8;            // [num_iter]
  std::vector<float> Th((size_t)max_iter * max_iter, 0.f);
  double* h = reinterpret_cast<double*>(static_cast<char*>(p->pinned) + PIN_SCALARS);

  auto dot = [&](const float* a, const float* b, double* out, int do_sqrt) {
    lz_dot_kernel<<<G, 256, 0, st>>>(a, b, n, part);
    lz_sum_kernel<<<1, 32, 0, st>>>(part, G, out, sharded ? 0 : do_sqrt);
    p->launches += 2;
    if (sharded) {
      nccl_allreduce_double(p->comm, out, 1, st);
      if (do_sqrt) { lz_sqrt_kernel<<<1, 1, 0, st>>>(out); p->launches++; }
    }
  };
  auto matvec = [&](const float* q, float* out) -> int {
    const float* qv = q;
    if (sharded) {
      GP_CUDA(cudaMemcpyAsync(qfull + p->row_begin, q, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
      GP_CHECK(nccl_allgather_float(p->comm, qfull, (size_t)n, st));
      qv = qfull;
    }
    GP_CHECK(to_v16(p, qv, 1, 1, N, p->V16.as<float>()));
    GP_CHECK(kmv_partials(p, p->V16.as<float>(), nullptr));
    return kmv_finish_user(p, p->V16.as<float>(), out, 1, 1, 1);
  };
  auto fetch = [&](int cnt) -> int {
    GP_CUDA(cudaMemcpyAsync(h, ds, sizeof(double) * cnt, cudaMemcpyDeviceToHost, st));
    GP_CUDA(cudaStreamSynchronize(st));
    return GP_OK;
  };
  auto gemv_t = [&](int m) {
    lz_gemv_t_kernel<<<m, 256, 0, st>>>(Qt, n, r, cvec);
    if (sharded) nccl_allreduce_double(p->comm, cvec, (size_t)m, st);
  };
  auto reorth = [&](int m) {  // r -= Q[:m] (Q[:m]^T r)
    gemv_t(m);
    lz_gemv_n_kernel<<<G, 256, sizeof(float) * ((m + 3) & ~3), st>>>(Qt, m, n, cvec, r);
    p->launches += 2;
  };

  // q_0 = init / |init|
  dot(INIT, INIT, ds + 1, 1);
  lz_scale_kernel<<<G, 256, 0, st>>>(INIT, ds + 1, n, Qt);
  GP_CHECK(matvec(Qt, r));
  dot(Qt, r, ds + 0, 0);
  lz_axpy_kernel<<<G, 256, 0, st>>>(r, Qt, ds + 0, n);
  dot(r, r, ds + 1, 1);
  p->launches += 2;
  GP_CHECK(fetch(2));
  Th[0] = (float)h[0];
  int k = 0;
  if (num_iter > 1) {
    Th[1] = (float)h[1];
    Th[(size_t)max_iter] = (float)h[1];
    lz_scale_kernel<<<G, 256, 0, st>>>(r, ds + 1, n, Qt + n);
    p->launches++;
  }
  for (k = 1; k < num_iter; ++k) {
    float* qk = Qt + (int64_t)k * n;
    float* qp = Qt + (int64_t)(k - 1) * n;
    GP_CHECK(matvec(qk, r));
    // r -= beta_prev q_prev   (beta_prev = T[k][k-1], still in ds[1] from the previous step)
    lz_axpy_kernel<<<G, 256, 0, st>>>(r, qp, ds + 1, n);
    dot(qk, r, ds + 0, 0);
    p->launches++;
    if (k + 1 < num_iter) {
      lz_axpy_kernel<<<G, 256, 0, st>>>(r, qk, ds + 0, n);
      p->launches++;
      reorth(k + 1);
      dot(r, r, ds + 1, 1);
      lz_scale_kernel<<<G, 256, 0, st>>>(r, ds + 1, n, r);
      p->launches++;
      // inner products after normalisation
      gemv_t(k + 1);
      p->launches++;
      GP_CUDA(cudaMemcpyAsync(h, ds, sizeof(double) * 2, cudaMemcpyDeviceToHost, st));
      GP_CUDA(cudaMemcpyAsync(h + 8, cvec, sizeof(double) * (k + 1), cudaMemcpyDeviceToHost, st));
      GP_CUDA(cudaStreamSynchronize(st));
      const double alpha = h[0], beta = h[1];
      Th[(size_t)k * max_iter + k] = (float)alpha;
      Th[(size_t)k * max_iter + k + 1] = (float)beta;
      Th[(size_t)(k + 1) * max_iter + k] = (float)beta;
      bool could = false;
      for (int rep = 0; rep < 10; ++rep) {
        bool any = false;
        for (int a = 0; a <= k; ++a) any |= (h[8 + a] > (double)tol);
        if (!any) { could = true; break; }
        reorth(k + 1);
        dot(r, r, ds + 2, 1);
        lz_scale_kernel<<<G, 256, 0, st>>>(r, ds + 2, n, r);
        gemv_t(k + 1);
        p->launches += 2;
        GP_CUDA(cudaMemcpyAsync(h + 8, cvec, sizeof(double) * (k + 1), cudaMemcpyDeviceToHost, st));
        GP_CUDA(cudaStreamSynchronize(st));
      }
      GP_CUDA(cudaMemcpyAsync(Qt + (int64_t)(k + 1) * n, r, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
      if (!(fabs(beta) > 1e-6) || !could) break;
    } else {
      GP_CHECK(fetch(1));
      Th[(size_t)k * max_iter + k] = (float)h[0];
    }
  }
  int J = std::min(k + 1, num_iter);
  // zero anything outside the leading J x J block (a break leaves T[J-1][J] written, as the reference slices it off)
  for (int a = 0; a < max_iter; ++a)
    for (int b = 0; b < max_iter; ++b)
      if (a >= J || b >= J) Th[(size_t)a * max_iter + b] = 0.f;
  GP_CUDA(cudaMemcpyAsync(T, Th.data(), sizeof(float) * Th.size(), cudaMemcpyHostToDevice, st));
  GP_CUDA(cudaStreamSynchronize(st));
  GP_CUDA(cudaGetLastError());
  if (J_out) *J_out = J;
  return GP_OK;
}
