// slq.cu -- stochastic Lanczos quadrature log-determinant from the mBCG tridiagonals, on the device.
//
// Restates linear_operator.utils.lanczos.lanczos_tridiag_to_diag + StochasticLQ.to_dense (SURVEY.md
// Appendix A.5):  logdet ~= (n / t_p) sum_i sum_j (V_i[0,j])^2 log lambda_ij , eigenvalues < 0 masked.
// The reference ships the J x J tridiagonals to the CPU for torch.linalg.eigh when J < 32; here one thread per
// probe runs an implicit-shift QL iteration in fp64 that tracks only the first row of the eigenvector matrix.
#include "gp_common.cuh"

namespace gp {

constexpr int SLQ_JMAX = 256;

__global__ void slq_kernel(const float* __restrict__ TMAT, int n_tridiag, int ldt, int J, double scale,
                           double* __restrict__ out_per_probe, int* __restrict__ fail) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_tridiag) return;
  const float* T = TMAT + (size_t)i * ldt * ldt;
  double d[SLQ_JMAX], e[SLQ_JMAX], z[SLQ_JMAX];
  bool finite = true;
  for (int a = 0; a < J; ++a) {
    d[a] = (double)T[(size_t)a * ldt + a];
    e[a] = (a + 1 < J) ? (double)T[(size_t)(a + 1) * ldt + a] : 0.0;
    z[a] = (a == 0) ? 1.0 : 0.0;
    finite = finite && isfinite(d[a]) && isfinite(e[a]);
  }
  // A NaN / Inf entry would not stop the QL sweeps (fabs(NaN) <= x is false) and the mask below would then drop every NaN
  // eigenvalue, turning the probe's term into a silent 0.  The reference gets NaN (eigh of a non-finite T), so write NaN.
  if (!finite) {
    out_per_probe[i] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  const int n = J;
  for (int l = 0; l < n; ++l) {
    int iter = 0, m;
    do {
      for (m = l; m < n - 1; ++m) {
        double dd = fabs(d[m]) + fabs(d[m + 1]);
        if (fabs(e[m]) <= 2.3e-16 * dd) break;
      }
      if (m != l) {
        if (iter++ == 100) { *fail = 1; break; }
        double g = (d[l + 1] - d[l]) / (2.0 * e[l]);
        double r = hypot(g, 1.0);
        g = d[m] - d[l] + e[l] / (g + copysign(r, g));
        double s = 1.0, c = 1.0, pp = 0.0;
        int q;
        for (q = m - 1; q >= l; --q) {
          double f = s * e[q], b = c * e[q];
          r = hypot(f, g);
          e[q + 1] = r;
          if (r == 0.0) { d[q + 1] -= pp; e[m] = 0.0; break; }
          s = f / r; c = g / r;
          g = d[q + 1] - pp;
          r = (d[q] - g) * s + 2.0 * c * b;
          pp = s * r;
          d[q + 1] = g + pp;
          g = c * r - b;
          f = z[q + 1];
          z[q + 1] = s * z[q] + c * f;
          z[q] = c * z[q] - s * f;
        }
        if (r == 0.0 && q >= l) continue;
        d[l] -= pp; e[l] = g; e[m] = 0.0;
      }
    } while (m != l);
  }
  double acc = 0.0;
  for (int a = 0; a < n; ++a)
    if (d[a] >= 0.0) acc += z[a] * z[a] * log(d[a]);  // negative eigenvalues: vector zeroed, value -> 1 (log 1 = 0)
  out_per_probe[i] = scale * acc;
}

}  // namespace gp

using namespace gp;

extern "C" int gp_slq_logdet(gp_plan* p, const float* TMAT, int n_tridiag, int ldt, int J, int64_t n, double* logdet_out) {
  GP_REQUIRE(p != nullptr, GP_E_STATE, "null plan");
  GP_REQUIRE(n_tridiag >= 1 && n_tridiag <= 64 && J >= 1 && J <= SLQ_JMAX && J <= ldt, GP_E_SHAPE,
             "bad SLQ shape n_tridiag=%d J=%d ldt=%d", n_tridiag, J, ldt);
  GP_CHECK(p->tmat_tmp.ensure(sizeof(double) * 64 + 64));
  double* d_out = p->tmat_tmp.as<double>();
  int* d_fail = reinterpret_cast<int*>(d_out + 64);
  GP_CUDA(cudaMemsetAsync(d_fail, 0, sizeof(int), p->stream));
  slq_kernel<<<1, 64, 0, p->stream>>>(TMAT, n_tridiag, ldt, J, (double)n / (double)n_tridiag, d_out, d_fail);
  p->launches++;
  GP_CUDA(cudaGetLastError());
  double* h = reinterpret_cast<double*>(static_cast<char*>(p->pinned) + PIN_SLQ);
  GP_CUDA(cudaMemcpyAsync(h, d_out, sizeof(double) * 64 + sizeof(int), cudaMemcpyDeviceToHost, p->stream));
  GP_CUDA(cudaStreamSynchronize(p->stream));
  double s = 0.0;
  for (int i = 0; i < n_tridiag; ++i) s += h[i];
  *logdet_out = s;  // a probe whose leading block holds a NaN / Inf wrote NaN: the log-det is NaN, as in InvQuadLogdet.forward
  if (*reinterpret_cast<int*>(h + 64)) {
    set_error("tridiagonal eigen-solver (implicit QL) did not converge within 100 sweeps for at least one probe; the SLQ log-determinant is unreliable");
    return GP_W_EIG_NOT_CONVERGED;
  }
  return GP_OK;
}
