/*
 * gp_bbmm.h -- C ABI of the H100-native BBMM exact-GP engine (libgpbbmm.so).
 *
 * Drop-in boundary for ONE hot path of cornellius-gp/gpytorch: the mBCG / SLQ evaluation of
 * the exact-GP marginal log likelihood.  Plain pointers and sizes only; no torch types.
 * Every entry point names the reference interface it replaces (paths relative to
 * /root/reference/gpytorch unless noted; "linear_operator" = the pinned third-party
 * dependency linear_operator>=0.6.1, setup.py:44, whose source is not vendored).
 *
 * Conventions
 *  - all device buffers are caller-owned (torch caching allocator in the Python host),
 *    row-major fp32 unless stated, and must stay alive until the stream work finishes;
 *  - every call enqueues on the cudaStream_t passed at plan creation (as void*) and
 *    returns an int status (GP_OK == 0); nothing throws, nothing calls exit();
 *  - hyper-parameters arrive as already-constrained host scalars (module.py /
 *    constraints/constraints.py stay in PyTorch, SURVEY.md section 2 row 12);
 *  - there is NO CPU fallback: every function needs a CUDA device.
 */
#ifndef GP_BBMM_H
#define GP_BBMM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* status codes (SURVEY.md section 8b "Errors"): mapped by the binding to RuntimeError /
 * NumericalWarning (utils/warnings.py:5) / NanError (utils/errors.py:8-22). */
enum {
  GP_OK = 0,
  GP_E_SHAPE = 1,         /* bad sizes / unsupported configuration            */
  GP_E_CUDA = 2,          /* a CUDA runtime call failed (gp_last_error())     */
  GP_E_NAN_MVM = 3,       /* "NaNs encountered when trying to perform matrix-vector multiplication" */
  GP_W_NOT_CONVERGED = 4, /* CG hit max_iter above tolerance (NumericalWarning) */
  GP_W_PIVCHOL_NAN = 5,   /* NaN in pivoted Cholesky -> preconditioner dropped  */
  GP_E_NCCL = 6,
  GP_E_STATE = 7,         /* call order violated (data / hypers not set)      */
  GP_W_EIG_NOT_CONVERGED = 8 /* tridiagonal QL iteration hit its sweep limit: the SLQ log-det is unreliable (NumericalWarning) */
};

/* Plan settings.  Ten settings change what a plan's operator is: a low-rank correction (lr, gp_plan_set_lowrank), task indices
 * (tsk, gp_plan_set_tasks), Kronecker (krn, gp_plan_set_kron), derivative observations (drv, gp_plan_set_deriv), a kernel product
 * (prd, gp_plan_set_product), additive (add, gp_plan_set_additive), spectral mixture (spm, gp_plan_set_spectral), periodic (per,
 * gp_plan_set_periodic), rational quadratic (rq, gp_plan_set_hypers_rq) and polynomial (ply, gp_plan_set_hypers_poly).  A call on a
 * plan carrying a setting it does not support (x below) returns GP_E_STATE with "<call> is not available on <plan> (<setter>)", naming
 * the call, the setting and its setter; a plan another plan takes in is refused the same way, as a data plan, or with "<call>: <plan>
 * as a factor|term is not available (<setter>)".  The low-rank correction, the one setting that coexists with others, is named first.
 * A re-check runs before every call on the taking plan once the plan it took in was re-packed.  SKI, kernel-sum and row-sharded
 * plans are checked separately, as each call describes.
 *                                                 lr  tsk krn drv prd add spm per rq  ply
 *   gp_plan_set_backend                           .   .   .   x   x   x   x   .   .   .
 *   gp_plan_set_hypers_rq                         .   x   x   x   x   x   x   x   .   .
 *   gp_plan_set_hypers_poly                       .   x   x   x   x   x   x   x   .   .
 *   gp_plan_set_comm with more than one rank      .   .   .   .   x   x   x   x   x   x
 *   gp_plan_set_ski                               .   x   x   x   x   x   x   x   x   x
 *   gp_ski_input_grad                             x   x   x   x   x   .   .   .   .   .
 *   gp_plan_set_tasks                             .   .   x   x   x   x   x   x   x   x
 *   gp_plan_set_tasks (after SKI / sum checks)    x   .   .   .   .   .   .   .   .   .
 *   gp_plan_set_additive                          .   x   x   x   x   .   x   x   x   x
 *   gp_plan_set_spectral                          .   x   x   x   x   x   .   x   x   x
 *   gp_plan_set_periodic                          .   x   x   x   x   x   x   .   x   x
 *   gp_plan_set_sum                               .   x   x   x   x   x   x   x   .   .
 *   gp_plan_set_product                           x   x   x   x   .   x   x   x   x   x
 *   gp_plan_set_kron                              x   x   .   x   x   x   x   x   x   x
 *   gp_plan_set_deriv                             x   x   x   .   x   x   x   x   x   x
 *   gp_plan_set_deriv_kind                        x   x   x   .   x   x   x   x   x   x
 *   gp_plan_set_lowrank                           .   x   x   x   x   .   .   .   .   .
 *   gp_kmv_input_grad                             x   x   x   x   x   x   x   x   .   .
 *   gp_kdense_input_grad                          x   x   x   x   x   x   x   x   .   .
 *   gp_pivoted_cholesky                           x   .   .   .   .   .   .   .   .   .
 *   gp_precond_build                              x   .   .   .   .   .   .   .   .   .
 *   gp_ciq_precond_build                          x   .   .   .   .   .   .   .   .   .
 *   gp_precond_probes                             x   .   .   .   .   .   .   .   .   .
 *   gp_bilinear_grad                              x   .   .   .   .   .   .   .   .   .
 *   gp_mbcg with a preconditioner                 x   .   .   .   .   .   .   .   .   .
 *   gp_ciq_sqrt_matmul_precond                    x   .   .   .   .   .   .   .   .   .
 *   gp_plan_set_kron (as the data plan)           .   .   .   .   x   x   x   x   x   x
 *   gp_plan_set_deriv (as the data plan)          .   .   .   .   x   x   x   x   x   x
 *   gp_plan_set_deriv_kind (as the data plan)     .   .   .   .   x   x   x   x   x   x
 *   gp_plan_set_kron data plan (re-check)         x   x   .   .   .   .   .   .   x   x
 *   gp_plan_set_deriv(_kind) data plan (re-check) x   x   .   .   .   .   .   .   .   .
 *   gp_plan_set_product, a factor                 .   .   .   .   x   x   x   x   x   x
 *   kernel product, a factor (re-check)           x   x   .   .   .   .   .   .   x   x
 *   gp_plan_set_sum, a term                       .   .   .   .   x   x   x   .   .   .
 *   kernel sum, a term (re-check)                 .   x   .   .   .   .   .   .   .   .
 */

/* covariance function kinds: kernels/rbf_kernel.py:68-85, kernels/matern_kernel.py:85-110, kernels/rq_kernel.py (GP_RQ is set
 * through gp_plan_set_hypers_rq only, which also gives alpha), kernels/polynomial_kernel.py (GP_POLY is set through
 * gp_plan_set_hypers_poly only, which also gives the power and the offset) */
enum { GP_RBF = 0, GP_MATERN12 = 1, GP_MATERN32 = 2, GP_MATERN52 = 3, GP_RQ = 4, GP_POLY = 5 };

/* which fused K.V kernel runs: GP_BACKEND_TCGEN05 = wgmma/bulk-TMA 3xTF32 tensor-core kernel
 * (the name is historical),
 * GP_BACKEND_SIMT = fp32 CUDA-core kernel (bring-up / cross-check / d > 41). */
enum { GP_BACKEND_AUTO = 0, GP_BACKEND_TCGEN05 = 1, GP_BACKEND_SIMT = 2, GP_BACKEND_SKI = 3 /* set by gp_plan_set_ski */,
       GP_BACKEND_SUM = 4 /* set by gp_plan_set_sum */, GP_BACKEND_KRON = 5 /* set by gp_plan_set_kron */,
       GP_BACKEND_DERIV = 6 /* set by gp_plan_set_deriv */, GP_BACKEND_PRODUCT = 7 /* set by gp_plan_set_product */ };

typedef struct gp_plan gp_plan;   /* opaque: repacked X, workspaces, stream, comm */
typedef struct gp_comm gp_comm;   /* opaque: NCCL communicator for row-sharded runs */

const char* gp_version(void);
const char* gp_last_error(void);          /* thread-local text of the last failure */
const char* gp_status_string(int status);

/* ---- plan ------------------------------------------------------------------------- */

/* Create a plan on `device` working on `stream` (a cudaStream_t, NULL = legacy default).
 * Replaces nothing 1:1; it is the "optional opaque handle" of SURVEY.md section 8b Ownership. */
int gp_plan_create(gp_plan** out, int device, void* stream);
int gp_plan_destroy(gp_plan* plan);
int gp_plan_set_backend(gp_plan* plan, int backend);

/* Training / test inputs.  X1 [n1, d] (ld1 floats per row), X2 [n2, d] or NULL (X2 == X1:
 * the x1_eq_x2 branch of sq_dist, kernels/kernel.py:26-49, incl. its exact diagonal).
 * Row-sharded runs pass row_begin/row_count: this rank owns output rows
 * [row_begin, row_begin+row_count) of K (multi_device_kernel.py:38,56-62); row_count<=0 = all. */
int gp_plan_set_data(gp_plan* plan, const float* X1, int64_t n1, int64_t ld1,
                     const float* X2, int64_t n2, int64_t ld2, int d,
                     int64_t row_begin, int64_t row_count);

/* Hyper-parameters: kind, lengthscale (host array, n_ls == 1 or d [ARD]), outputscale
 * (scale_kernel.py:108-118), noise sigma^2 (noise_models.py:57-92; added iff X2 == X1 and
 * the call asks for it).  Re-packs X on the device; call again whenever they change. */
int gp_plan_set_hypers(gp_plan* plan, int kind, const float* lengthscale, int n_ls,
                       float outputscale, float noise);

/* Per-row noise diagonal D (FixedNoiseGaussianLikelihood, likelihoods/gaussian_likelihood.py:245-363; FixedGaussianNoise,
 * noise_models.py:150-190): K_hat = K + diag(d).  `diag` is a device pointer to n2 floats (caller-owned, must outlive the plan's
 * use of it) that replaces the scalar noise in every product / solve / preconditioner / probe; NULL restores the scalar. */
int gp_plan_set_noise_diag(gp_plan* plan, const float* diag, int64_t n);

/* SKI / KISS-GP (kernels/grid_interpolation_kernel.py:132-213, kernels/grid_kernel.py:107-177, utils/interpolation.py:15-167):
 * the plan's operator becomes K_ski = W (T_0 x ... x T_{d-1}) W^T with cubic interpolation onto a regular grid; grid_lo[i] /
 * grid_step[i] are the first node and the spacing of dimension i (utils/grid.py:142-180), grid_sizes[i] in [4, 131072], d <= 4;
 * a grid with a dimension over 128 also needs prod_i grid_sizes[i] * 16 < 2^31 (GP_E_SHAPE otherwise).  Dimensions up to 128
 * nodes multiply by their dense Toeplitz factor, larger ones by its generating column, skipping the exactly-zero far band.
 * Call after gp_plan_set_data (square operator); products, mBCG, SLQ, gp_mll (without preconditioner) and gp_lanczos then run
 * on the interpolated operator, and gp_kdiag, gp_krows, gp_pivoted_cholesky, gp_precond_build, gp_precond_probes, gp_mbcg with W,
 * gp_ciq_precond_build and gp_ciq_sqrt_matmul_precond accept it (a preconditioned SKI MLL combines these primitives).  Out-of-bounds inputs fail like the reference ("Received data that was out of bounds ..."). */
int gp_plan_set_ski(gp_plan* plan, const int* grid_sizes, const float* grid_lo, const float* grid_step, int d);

/* KISS-GP prediction on the grid (InterpolatedPredictionStrategy, models/exact_prediction_strategies.py:481-827: mean_cache,
 * covar_cache, exact_predictive_mean / exact_predictive_covar).  Both take a packed SKI plan (gp_plan_set_ski + gp_plan_set_hypers)
 * over n points; grid matrices are row-major [M][t] (M = prod G_i) in the reference's flat grid order, dimension 0 slowest
 * (utils/interpolation.py:157-163).  t >= 1 is arbitrary, ld >= t.  GP_E_STATE on a non-SKI plan, GP_E_SHAPE for t < 1, ld < t
 * or a row-sharded plan.
 *  gp_ski_grid_matmul:   OUT[M, t] = s K_uu W^T V for V [n, t] over the plan's points (the grid caches c = s K_uu W^T alpha and
 *                        C = s K_uu W^T R);
 *  gp_ski_interp_matmul: OUT[n, t] = W C for C [M, t] (the reference's left_interp; W is never expanded, every call with the same
 *                        C returns bit-identical results). */
int gp_ski_grid_matmul(gp_plan* plan, const float* V, int64_t ldv, int t, float* OUT, int64_t ldo);
int gp_ski_interp_matmul(gp_plan* plan, const float* C, int64_t ldc, int t, float* OUT, int64_t ldo);

/* Input gradient of a SKI operator (deep kernel learning through KISS-GP): DX[n, d] (lddx >= d) = dF/dX of
 * F = sum_ic L_ic (K_ski R)_ic, K_ski = s W K_uu W^T, L and R [n, t] over the plan's points (ldl, ldr >= t, any t >= 1), in raw input
 * units.  Only W depends on X: the derivative of the Keys cubic weights, exactly 0 in the one-hot first / last grid cells, as the
 * reference's autograd through Interpolation.interpolate gives.  The gradient pass has no atomics; its grid blocks come from the
 * SKI scatter (per-tile atomic adds), so repeated calls agree to fp32 rounding.  A non-finite L
 * or R gives NaN.  GP_E_STATE on a non-SKI plan or one with a low-rank correction; GP_E_SHAPE for a row-sharded plan, t < 1 or
 * bad leading dimensions. */
int gp_ski_input_grad(gp_plan* plan, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, float* DX, int64_t lddx);

/* Kernel sums (AdditiveKernel, kernels/kernel.py:592-621: k = k_1 + ... + k_m, each term with its own covariance function,
 * lengthscale(s), outputscale and active dimensions): `plan` becomes the operator  sum_t K_t  (+ its own noise), where every
 * K_t is a ready plan over the same rows (same n1 / n2 / row shard / stream; the data pointers may differ: active_dims).
 * Call after gp_plan_set_data on `plan`; gp_plan_set_hypers on `plan` (before or after) supplies the sum's noise, its kind /
 * lengthscale / outputscale are ignored.  The terms stay owned by the caller and must outlive `plan`; re-packing a term (gp_plan_set_hypers on it) is
 * picked up by the next call on `plan`.  One K.V of the sum = one fused kernel launch per term into disjoint partial slots,
 * reduced by the same finish kernels; gp_pivoted_cholesky evaluates rows of the sum.  n_terms in [1, 4].
 * Hyper-parameter gradients: gp_bilinear_grad on each term plan. */
int gp_plan_set_sum(gp_plan* plan, gp_plan* const* terms, int n_terms);

/* Kernel products (ProductKernel, kernels/kernel.py:547-551, :634-690: k = k_1 * ... * k_m, each factor with its own covariance
 * function, lengthscale(s), outputscale and active dimensions; the reference multiplies the dense N x N matrices): `plan` becomes
 * the operator  S prod_f k_f  (+ its own noise / per-row diagonal where a call adds it), S = prod_f s_f, where every factor is a
 * ready plain plan (tensor-core or SIMT backend, any kind, scalar or ARD lengthscale) over the same rows, device and stream (the
 * data pointers may differ: active_dims).  Call after gp_plan_set_data on `plan`; gp_plan_set_hypers on `plan` (before or after)
 * supplies the noise only.  The factors stay owned by the caller and must outlive `plan`; re-packing a factor (gp_plan_set_hypers
 * on it) is picked up by the next call on `plan`.  n_factors in [2, 4]; NULL / 0 clears.  One K.V is ONE launch that forms
 * prod_f k_f per pair in registers with one ex2: two tensor-core factors with KP_a + KP_b <= 128 run the wgmma kernel
 * (gp_plan_info reports kpad = KP_a + KP_b), everything else with a total padded width <= 128 the CUDA-core kernel.
 * gp_kmv, gp_krows, gp_kdiag (square and cross), gp_pivoted_cholesky, gp_precond_build, gp_precond_probes, gp_mbcg, gp_slq_logdet,
 * gp_mll, gp_lanczos, gp_ciq_sqrt_matmul, gp_ciq_precond_build, gp_ciq_sqrt_matmul_precond, gp_plan_set_noise_diag and
 * gp_time_kmv_kernel run on it.  gp_bilinear_grad returns, factor after factor, the gradients of that factor's lengthscale(s)
 * (1 or d_f entries, sum_f n_ls_f in all; total padded width <= 64) and in grad_os dF/dS of the combined scale (dF/ds_f = S / s_f
 * dF/dS).  A SKI, sum, Kronecker, derivative or row-sharded factor returns GP_E_SHAPE. */
int gp_plan_set_product(gp_plan* plan, gp_plan* const* factors, int n_factors);

/* Additive GPs (the reference's ScaleKernel(RBFKernel(batch_shape=[D], ard_num_dims=1)) over X.mT.unsqueeze(-1), then .sum(dim=-3)
 * or utils/sum_interaction_terms.py, both dense): `plan` becomes the operator
 *   K(x, x') = sum_{m=1}^{M} e_m(c_1, .., c_D),   c_i = comp_scale[i] k(x_i, x'_i)   (+ its noise / per-row diagonal where a call adds it)
 * with e_m the elementary symmetric polynomial of degree m and k the plan's kind (RBF or Matern) over column i alone, with
 * lengthscale l_i.  M = min(max_degree, D): M = 1 is the sum of the components, M >= 2 adds every interaction term up to degree M.
 * The plan is a plain plan whose data has d = n_comp = D columns (1 <= D <= 32) and whose gp_plan_set_hypers gives D lengthscales
 * (before or after this call); its outputscale is ignored, its noise kept.  max_degree in [1, 8]; comp_scale: host [D], > 0.
 * comp_scale = NULL or n_comp = 0 clears the setting.  Square and cross plans; the plan runs its own CUDA-core kernels, which form e
 * per pair in registers by the positive recurrence e_m += c_i e_{m-1} (no cancellation).
 * gp_kmv, gp_krows, gp_kdiag (square: the constant sum_m e_m(comp_scale); cross: per pair), gp_pivoted_cholesky, gp_precond_build,
 * gp_precond_probes, gp_mbcg, gp_slq_logdet, gp_mll, gp_lanczos, gp_ciq_sqrt_matmul, gp_ciq_precond_build,
 * gp_ciq_sqrt_matmul_precond, gp_plan_set_noise_diag, gp_plan_set_lowrank and gp_time_kmv_kernel run on it.  gp_bilinear_grad returns
 * the D lengthscale gradients dF/dl_i in grad_ls and the D component-scale gradients dF/ds_i in grad_os, which must hold D doubles.
 * A non-finite input makes products, rows, the diagonal and gradients NaN.  A SKI, sum or row-sharded plan cannot become additive. */
int gp_plan_set_additive(gp_plan* plan, int max_degree, const float* comp_scale, int n_comp);

/* Spectral mixture kernels (the reference's SpectralMixtureKernel, kernels/spectral_mixture_kernel.py, dense over [Q, n, m, d]):
 * `plan` becomes the operator
 *   K(x, x') = S prod_{c<d} sum_{q<Q} w_q exp(-2 pi^2 v_qc^2 tau_c^2) cos(2 pi mu_qc tau_c),   tau = x - x'
 * (+ its noise / per-row diagonal where a call adds it), with w = weights[Q], mu = means[Q][d] and v = scales[Q][d] (host arrays,
 * row-major) and S the outputscale of gp_plan_set_hypers, which also gives the noise; the kind and lengthscale it passes are not
 * used.  As in the reference, the components of each dimension are summed before the product over the dimensions; for d = 1 this is
 * S sum_q w_q exp(-2 pi^2 v_q^2 tau^2) cos(2 pi mu_q tau).  The square diagonal is the constant S (sum_q w_q)^d.  A plain plan,
 * square or cross, after gp_plan_set_data, whose data has d columns.  1 <= Q <= 16, 1 <= d <= 8, Q d <= 32; anything else returns
 * GP_E_SHAPE.  Parameters are not checked: non-positive or non-finite values give what the formula gives.  Call it again whenever
 * the parameters change; weights = NULL or Q = 0 clears the setting.  The plan runs its own CUDA-core kernels on packed rows of the
 * fp32 inputs and their reduced phases frac(mu_qc x_c) (formed in fp64), so the cosine's argument stays below 2 pi in magnitude and
 * an entry's error does not grow with |x|.
 * gp_kmv, gp_krows, gp_kdiag, gp_pivoted_cholesky, gp_precond_build, gp_precond_probes, gp_mbcg, gp_slq_logdet, gp_mll, gp_lanczos,
 * gp_ciq_sqrt_matmul, gp_ciq_precond_build, gp_ciq_sqrt_matmul_precond, gp_plan_set_noise_diag, gp_plan_set_lowrank and
 * gp_time_kmv_kernel run on it.  gp_bilinear_grad returns Q (1 + 2d) doubles in grad_ls: dF/dw_q (Q), then dF/dmu_qc and dF/dv_qc
 * (Q d each, row-major); grad_os receives dF/dS.  A non-finite input makes products, rows, the diagonal and gradients NaN.  A SKI, sum or
 * row-sharded plan cannot become a spectral plan. */
int gp_plan_set_spectral(gp_plan* plan, int Q, const float* weights, const float* means, const float* scales, int d);

/* Periodic kernels (the reference's PeriodicKernel, kernels/periodic_kernel.py): `plan` becomes the operator
 *   K(x, x') = S exp(-2 sum_{c<d} sin^2(pi tau_c / p_c) / l_c),   tau = x - x'   (l_c not squared, as in the reference)
 * (+ its noise / per-row diagonal where a call adds it), with the n_period periods p = period[] (1: one period shared by every
 * dimension, or d), and the lengthscales l (1 or d), the outputscale S and the noise of gp_plan_set_hypers, whose kind must be
 * GP_RBF.  A plain plan, square or cross, after gp_plan_set_data, whose data has d columns; 1 <= d <= 16 and every period > 0 and
 * finite, else GP_E_SHAPE; a plan whose gp_plan_set_hypers kind is not GP_RBF returns GP_E_STATE, and so does gp_plan_set_hypers
 * with another kind on a periodic plan.  A failed call leaves the plan's previous setting in place.  Call it again whenever the
 * periods change; period = NULL or n_period = 0 clears the setting.  The
 * kernel is the RBF kernel of unit lengthscale over the embedding u_c(x) = (cos, sin)(2 pi x_c / p_c) / sqrt(l_c): the plan packs
 * u (2d columns, from phases reduced in fp64, so an entry's error does not grow with |x|) and from then on runs as a plain RBF
 * plan of width 2d, on the tensor-core backend (kpad = pad8(6d + 4)) or the CUDA-core one.
 * gp_kmv, gp_krows, gp_kdiag (the square diagonal is S), gp_pivoted_cholesky, gp_precond_build, gp_precond_probes, gp_mbcg,
 * gp_slq_logdet, gp_mll, gp_lanczos, gp_ciq_sqrt_matmul, gp_ciq_precond_build, gp_ciq_sqrt_matmul_precond, gp_plan_set_backend,
 * gp_plan_set_noise_diag, gp_plan_set_lowrank and gp_time_kmv_kernel run on it, and it may be a term of gp_plan_set_sum.
 * gp_bilinear_grad returns n_ls + n_period doubles in grad_ls, [dF/dl (n_ls) | dF/dp (n_period)] (a shared parameter receives the
 * sum over the dimensions), and dF/dS in grad_os; it is formed from tau directly, not through the embedding.  A non-finite input
 * makes the gradients NaN.  A SKI, sum or row-sharded plan cannot become a periodic plan. */
int gp_plan_set_periodic(gp_plan* plan, const float* period, int n_period, int d);

/* Rational quadratic kernels (the reference's RQKernel, kernels/rq_kernel.py): kind GP_RQ with its alpha, set together with the
 * lengthscales (1 or d), the outputscale S and the noise in one call:
 *   K(x, x') = S (1 + r^2 / (2 alpha))^-alpha,   r^2 = |(x - x') / l|^2
 * (+ its noise / per-row diagonal where a call adds it).  alpha must be > 0 and finite, and the lengthscales as for
 * gp_plan_set_hypers, else GP_E_SHAPE.  The call is all or nothing: a failed call leaves the plan's previous hyper-parameters in
 * place.  gp_plan_set_hypers with kind GP_RQ returns GP_E_SHAPE, so a plan never holds kind GP_RQ without its alpha; a later
 * gp_plan_set_hypers with another kind makes the plan a plain plan of that kind.  A plain plan, square or cross, on the tensor-core
 * backend or the CUDA-core one; the inputs are packed as for RBF with the constant C = 1, and alpha stays out of the packing.  Its
 * K.V evaluates log2(1 + t), t = r^2 / (2 alpha), with an absolute error O(2^-24 t) (a polynomial below t = 1/16), so an entry's
 * error does not grow with alpha (DESIGN 4.20).
 * gp_kmv, gp_krows, gp_kdiag (the square diagonal is S), gp_pivoted_cholesky, gp_precond_build, gp_precond_probes, gp_mbcg,
 * gp_slq_logdet, gp_mll, gp_lanczos, gp_ciq_sqrt_matmul, gp_ciq_precond_build, gp_ciq_sqrt_matmul_precond, gp_plan_set_backend,
 * gp_plan_set_noise_diag, gp_plan_set_lowrank (as the base), gp_kmv_input_grad, gp_kdense_input_grad and gp_time_kmv_kernel run on
 * it, and it may be a term of gp_plan_set_sum.  gp_bilinear_grad returns n_ls + 1 doubles in grad_ls, [dF/dl (n_ls) | dF/dalpha],
 * and dF/dS in grad_os; a non-finite input makes them NaN.  A SKI, sum or row-sharded plan cannot take this call (GP_E_STATE). */
int gp_plan_set_hypers_rq(gp_plan* plan, const float* lengthscale, int n_ls, float alpha, float outputscale, float noise);

/* Polynomial kernels (the reference's PolynomialKernel, kernels/polynomial_kernel.py): kind GP_POLY with its integer power p and
 * offset c, set together with the outputscale S and the noise in one call:
 *   K(x, x') = S (x . x' + c)^p
 * (+ its noise / per-row diagonal where a call adds it) over the raw inputs: no lengthscale and no centring.  x . x' + c may be
 * negative; an odd power keeps its sign.  1 <= p <= 8 and c finite and >= 0, else GP_E_SHAPE.  The call is all or nothing: a failed
 * call leaves the plan's previous hyper-parameters in place.  gp_plan_set_hypers with kind GP_POLY returns GP_E_SHAPE, so a plan
 * never holds kind GP_POLY without its power; a later gp_plan_set_hypers with another kind makes the plan a plain plan of that kind.
 * A plain plan, square or cross, on the tensor-core backend (the same widths as RBF: 3d + 4 <= the tensor-core limit) or the CUDA-core
 * one.  The tensor-core operands carry c in their spare columns, so GEMM1 gives a = x_i . x_j + c in 3xTF32 and the epilogue is
 * p - 1 multiplies at most (DESIGN 4.21).  The kernel is not stationary: its diagonal S (|x_i|^2 + c)^p varies from row to row.
 * gp_kmv, gp_krows, gp_kdiag (square: S (|x_i|^2 + c)^p per row; on a low-rank-corrected base that minus sum_j U_ij^2; on a sum with
 * a polynomial term the per-row sum of the terms' diagonals), gp_pivoted_cholesky (from that diagonal, first pivot its argmax,
 * earliest index on ties; a factor of a rank-deficient K ends, without GP_W_PIVCHOL_NAN, where no positive residual is left),
 * gp_precond_build, gp_precond_probes, gp_mbcg, gp_slq_logdet, gp_mll, gp_lanczos, gp_ciq_sqrt_matmul, gp_ciq_precond_build (its
 * trace from the same diagonal), gp_ciq_sqrt_matmul_precond, gp_plan_set_backend, gp_plan_set_noise_diag, gp_plan_set_lowrank (as
 * the base), gp_kmv_input_grad, gp_kdense_input_grad and gp_time_kmv_kernel run on it, and it may be a term of gp_plan_set_sum.
 * gp_bilinear_grad returns one double in grad_ls, [dF/dc], and dF/dS in grad_os (the power is not learned); a non-finite input makes
 * them NaN.  The input gradients use dk/dx_i = S p (x_i . x_j + c)^(p-1) x_j: every pair contributes, and on a square plan the
 * diagonal pair contributes 2 S p (|x_i|^2 + c)^(p-1) x_i.  A SKI, sum or
 * row-sharded plan cannot take this call (GP_E_STATE). */
int gp_plan_set_hypers_poly(gp_plan* plan, int power, float offset, float outputscale, float noise);

/* Low-rank correction (the lazy LOVE posterior covariance K** - K*x R R^T Kx*, models/exact_prediction_strategies.py:464-478,
 * which the reference keeps as test_test_covar + MatmulLinearOperator(root, -root^T)): the plan's operator becomes  s K - U U^T
 * (+ its noise / per-row diagonal where a call adds it).  U: device [n, r] fp32, leading dimension ldu, caller-owned, must outlive
 * the plan's use of it; 1 <= r <= 128.  U = NULL or r = 0 clears it.  Square, unsharded plans of every backend (tensor-core,
 * SIMT, kernel sum, SKI); GP_E_SHAPE otherwise.  The correction is one more partial slot of every product (U^T V reduced in a
 * fixed order: repeated products are bit-identical), so gp_kmv, gp_mbcg without W, gp_lanczos, gp_slq_logdet, gp_ciq_sqrt_matmul
 * and gp_mll (unpreconditioned) run on it; gp_kdiag returns diag(s K) - sum_j U_ij^2 and gp_krows the rows of s K - U U^T (also
 * for kernel sums); gp_mll skips its preconditioner.  A later
 * gp_plan_set_data / gp_plan_set_comm that changes the size or shards the plan makes every call that applies the correction
 * return GP_E_STATE until gp_plan_set_lowrank is called again. */
int gp_plan_set_lowrank(gp_plan* plan, const float* U, int64_t ldu, int r);

/* Hadamard multitask GPs (IndexKernel, kernels/index_kernel.py:18-117, multiplied into the data kernel as in
 * examples/03_Multitask_Exact_GPs/Hadamard_Multitask_GP_Regression.ipynb): with task ids set, the plan's operator becomes
 *     s K(x_i, x'_j) B[t_i, t'_j]   (+ its noise / per-row diagonal where a call adds it).
 * gp_plan_set_tasks: device int32 task ids, task1 [n1] and task2 [n2] (task2 = NULL on a square plan), 1 <= T <= 32; ids outside
 *   [0, T) return GP_E_SHAPE.  Call after gp_plan_set_data (new data drops the tasks); task1 = NULL clears them.  The ids are copied:
 *   the caller's arrays need not outlive the call.  GP_E_STATE on SKI and kernel-sum plans, GP_E_SHAPE on a row-sharded
 *   plan.
 * gp_plan_set_task_covar: B as a host array, row-major T x T (need not be symmetric or PSD: not checked); call again whenever it
 *   changes, like gp_plan_set_hypers.  Every call that applies the operator returns GP_E_STATE until it has been set.
 * Tensor-core and SIMT plans, square and cross: gp_kmv, gp_krows, gp_kdiag (s B[t_i, t_i]: not constant), gp_pivoted_cholesky
 * (first pivot = argmax of that diagonal, as for SKI), gp_precond_build / gp_precond_probes, gp_mbcg, gp_slq_logdet, gp_mll,
 * gp_lanczos, gp_ciq_* and gp_bilinear_grad (lengthscale(s) and outputscale of s K o B).  The input gradients (gp_kmv_input_grad,
 * gp_kdense_input_grad, gp_ski_input_grad) are refused.  One K.V is one launch of the plain fused kernel per column task over
 * that task's columns (rows and columns packed in task order), then B is applied row by row: no atomics, repeated calls agree bit
 * for bit.
 * gp_task_covar_grad: dB [T][T] (host, row-major) with dB[a][b] = s sum_{i: t_i = a} sum_{j: t'_j = b} (L_i . R_j) k(x_i, x'_j),
 * L [n1, t] (ldl), R [n2, t] (ldr), any t >= 1: the gradient of sum_ic L_ic ((s K o B) R)_ic with respect to B, at the cost of one
 * K.V per 16 columns.  Non-finite inputs give NaN. */
int gp_plan_set_tasks(gp_plan* plan, const int32_t* task1, const int32_t* task2, int T);
int gp_plan_set_task_covar(gp_plan* plan, const float* B, int T);
int gp_task_covar_grad(gp_plan* plan, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* dB);

/* Kronecker multitask GPs (MultitaskKernel, kernels/multitask_kernel.py:13-61, with every input observed for every task as in
 * examples/03_Multitask_Exact_GPs/Multitask_GP_Regression.ipynb): `plan` becomes the N1 T x N2 T operator
 *     (s K_data) (x) B   over interleaved rows i T + a (point i, task a)   (+ its noise / per-row diagonal where a call adds it),
 * where K_data is `data`'s operator.  `data` is a ready plain plan (tensor-core or SIMT, any kind, scalar or ARD lengthscale,
 * square or cross) on the same device and stream, caller-owned, and must outlive `plan`; re-packing it (gp_plan_set_hypers) is
 * picked up by the next call on `plan`.  data = NULL clears the operator.  1 <= T <= 32.  gp_plan_set_hypers on `plan` supplies the
 * noise only (as on a kernel sum); gp_plan_set_noise_diag takes N T entries.  B comes through gp_plan_set_task_covar(plan, B, T)
 * and its gradient through gp_task_covar_grad; gp_bilinear_grad on `plan` returns the gradients of data's lengthscale(s) and
 * outputscale.  One K.V of [N T, t] columns is ceil(T t / 16) launches of data's fused kernel on the B-mixed blocks
 * W[j, a t + c] = sum_b B[a, b] V[j T + b, c]: no atomics, repeated calls agree bit for bit.  gp_kmv, gp_krows, gp_kdiag,
 * gp_pivoted_cholesky, the preconditioner calls, gp_mbcg, gp_slq_logdet, gp_mll, gp_lanczos and gp_ciq_* run on it.
 * GP_E_SHAPE: a SKI, kernel-sum or row-sharded data plan, and gp_plan_set_comm with more than one rank on `plan`. */
int gp_plan_set_kron(gp_plan* plan, gp_plan* data, int T);

/* Missing observations on a Kronecker plan (settings.observation_nan_policy("mask") of the Python package): `plan` becomes the
 * n_rows x n_cols operator  P_r ((s K_data) (x) B) P_c^T  that keeps the interleaved rows `rows` and columns `cols` (host arrays,
 * strictly increasing, inside [0, N1 T) and [0, N2 T); copied to the device once).  NULL keeps every row or column; rows = cols =
 * NULL, or lists that name every row, remove the mask.  On a square plan the two masks must be equal (GP_E_SHAPE otherwise).  The
 * mask is part of the Kronecker setting: it survives gp_plan_set_kron with the same N1, N2 and T, as B does, and is dropped
 * otherwise.  gp_plan_set_noise_diag then takes n_rows entries (a diagonal set before is dropped when the row count changes).
 * Every call that runs on a Kronecker plan runs on the masked operator: K.V mixes the observed columns (zero elsewhere) through
 * the same launches of data's fused kernel and scatters the observed rows; gp_krows takes observed row indices and returns the
 * observed columns; gp_kdiag, gp_pivoted_cholesky (first pivot = argmax of the diagonal s B[a, a]), gp_bilinear_grad and
 * gp_task_covar_grad (L and R of n_rows and n_cols rows) are those of the masked operator.  GP_E_STATE: not a Kronecker plan. */
int gp_plan_set_kron_observed(gp_plan* plan, const int64_t* rows, int64_t n_rows, const int64_t* cols, int64_t n_cols);

/* Several latent processes (the linear model of coregionalisation, LCMKernel, kernels/lcm_kernel.py): `plan` becomes the
 * N1 T x N2 T operator
 *     sum_q (s_q K_q) (x) B_q,   q = 0 .. Q-1,   over interleaved rows i T + a   (+ its noise / per-row diagonal),
 * where K_q is data[q]'s operator and s_q its outputscale.  1 <= Q <= 4 (GP_E_SHAPE otherwise); every data[q] is a data plan as
 * gp_plan_set_kron takes it (the same roles and refusals), and the terms may differ in kind, lengthscale, backend and input rows
 * (active dimensions), but share N1, N2, squareness, device and stream (GP_E_SHAPE / GP_E_STATE otherwise).  data = NULL clears the
 * operator; Q = 1 is gp_plan_set_kron(plan, data[0], T).  One K.V is, per term, a B_q mix and ceil(T t / 16) launches of data[q]'s
 * fused kernel, then one scatter of sum_q s_q (term's product) in a fixed order (terms outer, splits inner); it is NaN when any
 * term has non-finite inputs or any B_q a non-finite entry.  gp_krows, gp_kdiag, gp_pivoted_cholesky (entries
 * sum_q s_q B_q[a, b] k_q, first pivot = argmax of the diagonal), the preconditioner calls, gp_mbcg, gp_slq_logdet, gp_mll,
 * gp_lanczos and gp_ciq_* run on it.  On a plan with Q > 1, gp_plan_set_task_covar, gp_task_covar_grad, gp_bilinear_grad and
 * gp_plan_set_kron_observed return GP_E_STATE (naming the call to use instead). */
int gp_plan_set_kron_terms(gp_plan* plan, gp_plan* const* data, int Q, int T);

/* B_0 .. B_{Q-1} of a plan set by gp_plan_set_kron_terms: Q row-major T x T host blocks back to back, in term order (copied). */
int gp_plan_set_kron_term_covars(gp_plan* plan, const float* B, int Q, int T);

/* Gradients of F = sum(L * (K R)) for L [N1 T, t] (leading dimension ldl) and R [N2 T, t] (ldr) on a Kronecker plan, in term
 * order: grad_ls = every term's lengthscale gradient(s) concatenated (1 or d per term), grad_os = the Q outputscale gradients,
 * dB = the Q T x T blocks dF/dB_q (row-major, back to back).  Per term these are gp_bilinear_grad's and gp_task_covar_grad's
 * passes with that term's B_q; the sums are fp64 in a fixed order, without atomics: repeated calls agree bit for bit. */
int gp_kron_terms_grad(gp_plan* plan, const float* L, int64_t ldl, const float* R, int64_t ldr, int t, double* grad_ls, double* grad_os,
                       double* dB);

/* GPs with derivative observations (RBFKernelGrad, kernels/rbf_kernel_grad.py:60-115, with the perfect shuffle of :99-102, as in
 * examples/08_Advanced_Usage/Simple_GP_Regression_Derivative_Information_{1d,2d}.ipynb): `plan` becomes the N1 (d+1) x N2 (d+1)
 * operator over interleaved rows i (d+1) + a (a = 0: f(x_i); a = 1..d: df/dx_a at x_i) with, for D = x_i - x'_j,
 * u_a = D_a / l_a^2 and k = s exp(-|D / l|^2 / 2),
 *     [value, value] = k,  [value, d/dx'_b] = k u_b,  [d/dx_a, value] = -k u_a,  [d/dx_a, d/dx'_b] = k (delta_ab / l_a^2 - u_a u_b)
 * (+ its noise / per-row diagonal where a call adds it).  `data` is a ready plain RBF plan (tensor-core or SIMT, scalar or ARD
 * lengthscale, square or cross, 1 <= d <= 16) on the same device and stream, caller-owned, and must outlive `plan`; the derivative
 * kernels read its packed inputs and hyper-parameters and never call its fused kernel.  Re-packing it (gp_plan_set_hypers) is
 * picked up by the next call on `plan`.  data = NULL clears the operator.  gp_plan_set_hypers on `plan` supplies the noise only (as
 * on a kernel sum); gp_plan_set_noise_diag takes N (d+1) entries.  One K.V is one launch of an fp32 SIMT kernel per 4 columns
 * (16 for d <= 4) and a fixed-order sum of its column-split partials: no atomics, repeated calls agree bit for bit.
 * gp_kmv, gp_krows, gp_kdiag (s, s / l_a^2 on a square plan), gp_pivoted_cholesky (first pivot = argmax of that diagonal), the
 * preconditioner calls, gp_mbcg, gp_slq_logdet, gp_mll, gp_lanczos and gp_ciq_* run on it; gp_bilinear_grad returns the gradients of
 * data's lengthscale(s) and outputscale.  A non-finite input makes products, rows, the diagonal and gradients NaN.
 * GP_E_SHAPE: a non-RBF, SKI, kernel-sum, Kronecker, derivative or row-sharded data plan, d > 16, and gp_plan_set_comm with more
 * than one rank on `plan`. */
int gp_plan_set_deriv(gp_plan* plan, gp_plan* data);

/* The same value / gradient operator for another covariance (kernels/matern52_kernel_grad.py): kind = GP_RBF is
 * gp_plan_set_deriv; kind = GP_MATERN52 takes a ready plain Matern-5/2 data plan and gives, with D = x_i - x'_j, u_a = D_a / l_a^2,
 * rho = sqrt(5 |D / l|^2), e = exp(-rho), A = (5/3) (1 + rho) e, B = (25/3) e and the data plan's outputscale s,
 *     [0, 0] = s (1 + rho + rho^2 / 3) e,  [0, b] = s A u_b,  [a, 0] = -s A u_a,  [a, b] = s (A delta_ab / l_a^2 - B u_a u_b);
 * gp_kdiag returns s and (5/3) s / l_a^2 on a square plan.  Every call and refusal of gp_plan_set_deriv applies.  The plan
 * remembers `kind`: a data plan whose covariance later differs is refused by the next call (GP_E_SHAPE).  Another kind: GP_E_SHAPE. */
int gp_plan_set_deriv_kind(gp_plan* plan, gp_plan* data, int kind);

/* ---- kernel seam (LazyEvaluatedKernelTensor, lazy/lazy_evaluated_kernel_tensor.py) --- */

/* OUT[n1_local, t] = K(X1,X2) V [+ noise * V when add_noise and X2 == X1].
 * Replaces LazyEvaluatedKernelTensor._matmul (:245-276) / KernelLinearOperator._matmul
 * (kernels/keops/rbf_kernel.py:44-55); K is never written to HBM.  V [n2, t] ldv, OUT ldo. */
int gp_kmv(gp_plan* plan, const float* V, int64_t ldv, int t, float* OUT, int64_t ldo, int add_noise);

/* OUT[m, n2] = K(X1[idx], X2): row extraction, LazyEvaluatedKernelTensor._getitem (:136-243);
 * idx is a DEVICE int64 array; an index outside [0, n1) gives a row of NaN (every backend).  SKI plans: exact entries
 * s prod_k w_ik^T T_k w_jk from the separable form, m <= 65535. */
int gp_krows(gp_plan* plan, const int64_t* idx, int64_t m, float* OUT, int64_t ldo);

/* OUT[n1] = diag K(X1,X1): LazyEvaluatedKernelTensor._diagonal (:107-133).  SKI plans: s prod_k w_ik^T T_k w_ik (not constant). */
int gp_kdiag(gp_plan* plan, float* OUT);

/* d/d(theta) sum_ij sum_s Lf[i,s] K_theta(x_i,x_j) Rt[j,s]: LazyEvaluatedKernelTensor.
 * _bilinear_derivative (:69-105) + RBFCovariance/MaternCovariance.backward
 * (functions/rbf_covariance.py:26-29, matern_covariance.py:52-56).
 * grad_ls: host double[n_ls]; grad_os: host double (d/d outputscale).  Lf [n1,s], Rt [n2,s]. */
int gp_bilinear_grad(gp_plan* plan, const float* Lf, int64_t ldl, const float* Rt, int64_t ldr,
                     int s, double* grad_ls, double* grad_os);

/* Input gradients (the autograd of RBFKernel.forward / MaternKernel.forward's slow branch, kernels/rbf_kernel.py:68-85,
 * kernels/matern_kernel.py:86-107, w.r.t. x1 / x2): DX1 = dF/dX1 [n1][d] (ld1), DX2 = dF/dX2 [n2][d] (ld2), in raw input units
 * with the outputscale folded in and the noise excluded, for F = sum_ic G_ic (K V)_ic; G [n1, t] ldg, V [n2, t] ldv, any t >= 1.
 * Either output may be NULL; on a square plan (X2 == X1) DX1 gets the total gradient and DX2 must be NULL.  A pair at distance 0
 * contributes 0 for the stationary kinds; on a polynomial plan (GP_POLY) every pair contributes S p a^(p-1) x_j, a = x_i . x_j + c,
 * the diagonal pair of a square plan 2 S p a_ii^(p-1) x_i.  A non-finite input gives NaN outputs.  Repeated calls give identical bits (no atomics).
 * GP_E_SHAPE on SKI, kernel-sum (call on every term) and row-sharded plans, for bad shapes, t < 1 or d > 64; GP_E_STATE on a
 * plan with a low-rank correction. */
int gp_kmv_input_grad(gp_plan* plan, const float* G, int64_t ldg, const float* V, int64_t ldv, int t,
                      float* DX1, int64_t ld1, float* DX2, int64_t ld2);
/* the same for F = sum_ij W_ij K_ij, W [n1][n2] (ldw >= n2): the input gradient of the dense block gp_krows returns */
int gp_kdense_input_grad(gp_plan* plan, const float* W, int64_t ldw, float* DX1, int64_t ld1, float* DX2, int64_t ld2);

/* ---- solver seam (linear_operator) --------------------------------------------------- */

/* Greedy pivoted partial Cholesky of K(X1,X1) (outputscale included, no noise):
 * linear_operator.functions._pivoted_cholesky, surfaced at gpytorch/__init__.py:146-173.
 * Lt [rank, n] row-major (= L^T), piv int64[rank] (device), *rank_out <= rank.  Dense, kernel-sum and SKI plans; for SKI the
 * initial diagonal is not constant: the first pivot is its argmax (earliest index on ties) and the error is sum|diag| / max diag.
 * Kernel sums and SKI need the cooperative (persistent) kernel. */
int gp_pivoted_cholesky(gp_plan* plan, int rank, float error_tol, float* Lt, int64_t* piv,
                        int* rank_out);

/* Preconditioner for K + noise I from Lt [k, n]: W [n, k] with P^{-1} v = (v - W W^T v)/noise,
 * log det P.  AddedDiagLinearOperator._preconditioner / _init_cache_for_constant_diag
 * (linear_operator); W spans the same space as the reference's Q[:n] (W W^T == Q Q^T). */
int gp_precond_build(gp_plan* plan, const float* Lt, int k, float* W, double* logdet_out);

/* z = L eps1 + sqrt(noise) eps2 ~ N(0, P): the probe draw of InvQuadLogdet.forward
 * (linear_operator) with the base samples supplied.  eps1 [k, tp], eps2 [n, tp], Z [n, tp]. */
int gp_precond_probes(gp_plan* plan, const float* Lt, int k, const float* eps1, const float* eps2,
                      int tp, float* Z);

/* modified batched preconditioned CG on (K + noise I) with K applied by the fused kernel:
 * linear_operator.utils.linear_cg (signature attested at
 * variational/ciq_variational_strategy.py:56-64).  RHS/SOLVES [n, t] (t <= 16 per call),
 * W [n,k] or NULL.  TMAT fp32 [n_tridiag, max_tridiag_iter, max_tridiag_iter] (zero-filled by
 * the call; the leading J x J block is valid, J -> *tridiag_size).  resid_out host float[t]. */
int gp_mbcg(gp_plan* plan, const float* RHS, int64_t ldr, int t, int n_tridiag, float tolerance,
            int max_iter, int max_tridiag_iter, const float* W, int k, float* SOLVES, int64_t lds,
            float* TMAT, int* iters_out, int* tridiag_size, float* resid_out);

/* log det estimate from the mBCG tridiagonals: lanczos_tridiag_to_diag + StochasticLQ.to_dense
 * (linear_operator.utils.lanczos / stochastic_lq).  TMAT [n_tridiag, ldt, ldt] device fp32,
 * leading J x J blocks used; result (n / n_tridiag) sum_i sum_j (V_i[0,j])^2 log lambda_ij. */
int gp_slq_logdet(gp_plan* plan, const float* TMAT, int n_tridiag, int ldt, int J, int64_t n,
                  double* logdet_out);

/* Lanczos tridiagonalisation with full re-orthogonalisation of (K + noise I):
 * linear_operator.utils.lanczos.lanczos_tridiag (root_inv_decomposition,
 * models/exact_prediction_strategies.py:268-272).  INIT [n], Q [max_iter, n] row-major
 * (= Q^T), T [max_iter, max_iter]; *J_out = steps run. */
int gp_lanczos(gp_plan* plan, const float* INIT, int max_iter, float tol, float* Qt, float* T,
               int* J_out);

/* OUT = K_hat * sum_q w_q (K_hat + tau_q I)^{-1} B  ~=  K_hat^{1/2} B  (contour integral quadrature);
 * B, OUT [n, t] (t <= 16), tau/w host double[Q] (1 <= Q <= 32, tau_q >= 0, finite);
 * resid_out host float[Q*t]: final |phi| / ||b_c|| per shift and column; *iters_out = iterations run.
 * Multi-shift MINRES on K_hat = the plan's operator with its noise (the closure of gp_mbcg), one Lanczos process per column
 * shared by all shifts (msMINRES, Pleiss et al. 2020, arXiv 2006.11267; the reference's CIQ sampler,
 * linear_operator.utils.contour_integral_quad / minres, behind settings.ciq_samples).  Square, unsharded plans only. */
int gp_ciq_sqrt_matmul(gp_plan* plan, const float* B, int64_t ldb, int t, const double* tau, const double* w, int Q,
                       float tol, int max_iter, float* OUT, int64_t ldo, int* iters_out, float* resid_out);

/* Split factor of the pivoted-Cholesky preconditioner P = L L^T + D for the CIQ sampler, from Lt [k, n] (1 <= k <= 128):
 * U [n, k] with F^-1 = (I - U U^T) D^-1/2 for F = D^1/2 (I + M M^T)^1/2, M = D^-1/2 L (eigh of L^T D^-1 L in fp64 on the host);
 * *trace_resid_out = tr(K - L L^T) in fp64 (SKI plans: the fp64 sum of the SKI diagonal).  Needs noise > 0 (all d > 0); square,
 * unsharded plans.
 * A non-finite Gram returns GP_W_PIVCHOL_NAN (the caller drops the preconditioner). */
int gp_ciq_precond_build(gp_plan* plan, const float* Lt, int k, float* U, double* trace_resid_out);

/* Preconditioned CIQ: OUT = K_hat F^-T sum_q w_q (A + tau_q I)^-1 B with A = F^-1 K_hat F^-T and U [n, k] from
 * gp_ciq_precond_build, i.e. OUT ~= F A^{1/2} B ~ N(0, K_hat) for B ~ N(0, I) (a different root than gp_ciq_sqrt_matmul's).
 * Arguments, status codes and the stop rule (on A's shifted residuals) as gp_ciq_sqrt_matmul. */
int gp_ciq_sqrt_matmul_precond(gp_plan* plan, const float* B, int64_t ldb, int t, const float* U, int k, const double* tau,
                               const double* w, int Q, float tol, int max_iter, float* OUT, int64_t ldo, int* iters_out,
                               float* resid_out);

/* one-shot: MultivariateNormal.log_prob (distributions/multivariate_normal.py:221-252) through
 * inv_quad_logdet (:249), i.e. pivoted Cholesky -> preconditioner -> probes -> mBCG -> SLQ. */
typedef struct gp_mll_opts {
  int num_probes;          /* settings.num_trace_samples (10)                    */
  int precond_rank;        /* settings.max_preconditioner_size (15; C2 uses 100) */
  int min_precond_size;    /* settings.min_preconditioning_size (2000)           */
  float precond_tol;       /* settings.preconditioner_tolerance (1e-3)           */
  float cg_tol;            /* settings.cg_tolerance (1.0)                        */
  int max_cg_iter;         /* settings.max_cg_iterations (1000)                  */
  int max_tridiag_iter;    /* settings.max_lanczos_quadrature_iterations (20)    */
} gp_mll_opts;

typedef struct gp_mll_result {
  double inv_quad, logdet, logdet_precond, log_prob, mll;
  int cg_iters, tridiag_size, precond_rank, status_flags;
  float resid[16];
} gp_mll_result;

/* y_minus_mean [n]; eps1 [precond_rank, tp], eps2 [n, tp] N(0,1) base samples, rademacher [n, tp]
 * (used when no preconditioner applies); solve_out [n] = K_hat^{-1}(y - mu) or NULL. */
int gp_mll(gp_plan* plan, const float* y_minus_mean, const float* eps1, const float* eps2,
           const float* rademacher, const gp_mll_opts* opts, float* solve_out, gp_mll_result* res);

/* ---- multi-GPU (one process per GPU; replaces MultiDeviceKernel, multi_device_kernel.py:14-95) */
int gp_comm_unique_id(uint8_t out[128]);                 /* rank 0, then broadcast by the host */
int gp_comm_init(gp_comm** out, const uint8_t id[128], int rank, int world);
int gp_comm_destroy(gp_comm* comm);
int gp_plan_set_comm(gp_plan* plan, gp_comm* comm);      /* NULL = single GPU */

/* ---- introspection for bench.py --------------------------------------------------- */
int64_t gp_kernel_launches(gp_plan* plan);               /* kernels launched by this plan so far */
int gp_plan_info(gp_plan* plan, int* backend, int* nsplit, int* kpad, int* n_sm);
/* Times `reps` back-to-back launches of the fused K.V kernel ALONE (after `warmup` untimed ones) with CUDA
 * events on the plan's stream; V [n2, t].  *ms_per_launch is the average device time of one launch.  On a plan with task ids a
 * "launch" is the whole K o B product (V gather and tiles, one launch per column task, combine). */
int gp_time_kmv_kernel(gp_plan* plan, const float* V, int64_t ldv, int t, int warmup, int reps, float* ms_per_launch);

#ifdef __cplusplus
}
#endif
#endif /* GP_BBMM_H */
