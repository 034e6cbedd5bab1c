/* agp.h -- C ABI of libagp.so, the Hopper-native (sm_90a) exact-GP engine that sits
 * behind AbstractGPs.jl's dense hot path.
 *
 * The reference (pure Julia, /root/reference) has no FFI; the two seams a drop-in uses are
 * Julia multiple dispatch on FiniteGP / PosteriorGP (SURVEY.md s1, s8b).  Each entry point
 * below names the reference method(s) it replaces (path:line relative to /root/reference).
 * The Julia shim that `ccall`s these symbols is julia/AGPBlackwell.jl; the identical symbols
 * are driven from Python ctypes in abstractgps.jl_b200/_cabi.py (the only host toolchain in
 * this image).  See INTEGRATION.md.
 *
 * Conventions
 *   - all functions return int32_t status (AGP_OK == 0); no exception crosses the ABI.
 *   - every data pointer is HOST memory owned by the caller unless the ctx was switched
 *     with agp_set_memspace(ctx, AGP_MEM_DEVICE) (then X / Y / Xs / Z-normals / outputs that
 *     are arrays are DEVICE pointers on the ctx's GPU; scalars-out stay host).
 *   - element type is `dtype` (AGP_F32 / AGP_F64) for every array argument.
 *   - points: AGP_POINT_MAJOR   = ColVecs(X),  X is D x N column-major (a point is contiguous)
 *             AGP_FEATURE_MAJOR = RowVecs(X),  X is N x D column-major
 *   - matrices out are column-major (Julia layout).
 *   - calls are blocking (stream-synchronised before return) and a ctx is not re-entrant.
 */
#ifndef AGP_H
#define AGP_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct agp_ctx agp_ctx;           /* device, streams, workspace arena, (NCCL comm)      */
typedef struct agp_post agp_post;         /* device-resident factor L (=U'), alpha, x, kernel     */
typedef struct agp_vfe_post agp_vfe_post; /* device-resident VFE cache (m_e, Lambda, U, alpha, z) */

enum { AGP_F32 = 0, AGP_F64 = 1 };
enum { AGP_SE = 0, AGP_MATERN12 = 1, AGP_MATERN32 = 2, AGP_MATERN52 = 3, AGP_LINEAR = 4 };
/* factor-only families (valid inside an agp_kernel_composite, AGP_ERR_UNSUPPORTED at top level) and the composite tag */
enum { AGP_RQ = 5, AGP_PERIODIC = 6, AGP_WHITE = 7, AGP_CONSTANT = 8, AGP_COMPOSITE = 9 };
enum { AGP_T_NONE = 0, AGP_T_SCALE = 1, AGP_T_ARD = 2 };
enum { AGP_POINT_MAJOR = 0, AGP_FEATURE_MAJOR = 1 };
enum { AGP_MEM_HOST = 0, AGP_MEM_DEVICE = 1 };

enum {
  AGP_OK = 0,
  AGP_ERR_NOT_POSDEF = 1,   /* -> Julia PosDefException(info); info via agp_last_info()      */
  AGP_ERR_DIM_MISMATCH = 2, /* -> DimensionMismatch (src/sparse_approximations.jl:290-294)   */
  AGP_ERR_UNSUPPORTED = 3,
  AGP_ERR_CUDA = 4,
  AGP_ERR_NCCL = 5,
  AGP_ERR_INVALID = 6
};

/* One factor of a composite kernel: a base kernel over its own input transform.  With d2 the squared Euclidean distance
 * of the transformed inputs x~, y~ (KernelFunctions definitions):
 *   AGP_SE / AGP_MATERN12 / 32 / 52   as the single-kernel families
 *   AGP_LINEAR     x~ . y~ + c                                  (param = c)
 *   AGP_RQ         (1 + d2 / (2 alpha))^(-alpha), alpha > 0     (param = alpha)
 *   AGP_PERIODIC   exp(-1/2 sum_i (sinpi(x~_i - y~_i) / r_i)^2), r > 0 (r == NULL -> ones)
 *   AGP_WHITE      1 if x~ == y~, else 0
 *   AGP_CONSTANT   c                                            (param = c)
 * with_lengthscale(PeriodicKernel(r), p) is an AGP_PERIODIC factor with ScaleTransform(1/p). */
typedef struct {
  int32_t family, transform; /* AGP_SE..AGP_CONSTANT; AGP_T_* of this factor's inputs */
  double scale;              /* ScaleTransform s */
  double param;              /* RQ alpha | Linear c | Constant c */
  const void* ard;           /* ARD v, D values of `dtype`, HOST */
  const void* r;             /* Periodic r, D values of `dtype`, HOST (NULL -> ones) */
} agp_kernel_factor;

/* K(x, y) = sum_t variance[t] * prod_{f in term t} kappa_f(T_f x, T_f y): KernelSum / KernelProduct / ScaledKernel trees
 * flattened into a sum of product terms.  At most 8 terms and 8 factors in all. */
typedef struct {
  int32_t nterms;                   /* 1..8 */
  const int32_t* nfactors;          /* per term, >= 1, total <= 8 */
  const double* variance;           /* v_t per term */
  const agp_kernel_factor* factors; /* concatenated term by term */
} agp_kernel_composite;

/* sigma_f^2 * (kappa o transform): KernelFunctions ScaledKernel / TransformedKernel with
 * ScaleTransform(s) | ARDTransform(v); with_lengthscale(k,l) == scale 1/l.
 * Reference call sites: src/base_gp.jl:70,72,74.
 * family == AGP_COMPOSITE: the kernel is `composite` (transform must be AGP_T_NONE and variance 1; scale, linear_c and
 * ard are ignored).  The single-GPU exact path (agp_gram, agp_fit, agp_rand and the agp_post_* calls on its handle)
 * accepts it; the VFE entry points and distributed contexts return AGP_ERR_UNSUPPORTED.  Out-of-range counts, a missing
 * ARD array, alpha <= 0 or r <= 0 give AGP_ERR_INVALID.  `composite` is read only for that family. */
typedef struct {
  int32_t family;    /* AGP_SE ... AGP_LINEAR, AGP_COMPOSITE */
  int32_t transform; /* AGP_T_* */
  double variance;   /* sigma_f^2 */
  double scale;      /* ScaleTransform s */
  double linear_c;   /* LinearKernel c */
  const void* ard;   /* ARDTransform v: D values in `dtype`, HOST memory always */
  const agp_kernel_composite* composite; /* AGP_COMPOSITE only; HOST; copied by the call (handles keep their own copy) */
} agp_kernel;

/* ZeroMean / ConstMean / CustomMean-evaluated-to-a-vector (src/mean_function.jl:27,40,52-55) */
typedef struct {
  int32_t kind; /* 0 zero, 1 const, 2 vector */
  double c;
  const void* v; /* `dtype`, length = number of points; HOST memory always */
} agp_mean;

/* Diagonal Sigma_y: Fill(sigma^2) or per-point vector (src/finite_gp_projection.jl:13-21) */
typedef struct {
  int32_t kind; /* 0 scalar, 1 per-point vector */
  double s;
  const void* v; /* `dtype`; HOST memory always */
} agp_noise;

typedef struct {
  int32_t tile_nb;       /* OUTER panel width (multiple of 128); 0 -> auto (512 from n_pad >= 8192, else 128) */
  int32_t fp64_mode;     /* -1 auto (int8 slices from n_pad >= 8192), 0 = DMMA mma.sync trailing update,
                            1 = int8-sliced (Ozaki) trailing update on wgmma s8 x s8 */
  int32_t fp32_mode;     /* -1 auto (int8 slices from n_pad >= 4096), 0 = FFMA tile kernels, 1 = int8-sliced trailing update /
                            triangular solves on wgmma s8 x s8 (4 seven-bit slices cover the fp32 significand) */
  int32_t lookahead;     /* 0 off, 1: overlap the next panel with the bulk of the trailing update, 2 (default): additionally
                            split the bulk so that the chain waits only for the panel-after-next block (DMMA path) */
  int32_t use_graph;     /* reserved */
  int32_t ozaki_slices;  /* slices of the int8 fp64 path; 0 -> 6.  6: six balanced 8-bit digits (21 int8 MMAs per fp64 MAC,
                            error <= 2^-43.4 2^(e_i+e_j) K) in the Cholesky's trailing updates, seven 7-bit slices in
                            the substitutions and VFE products; 5, 7, 8: that many 7-bit slices everywhere
                            ((S + 1.06) 2^-7S 2^(e_i+e_j) K; 7 -> 2^-46) */
  int32_t profile_kernels; /* 1: CUDA events around every trailing-update launch (agp_last_timings[7]); default 0 */
  int32_t reserved[9];
} agp_config; /* NULL -> defaults; env AGP_NB, AGP_FP64_MODE, AGP_FP32_MODE, AGP_LOOKAHEAD, AGP_OZAKI_S, AGP_OZAKI_S32 override at agp_init */

/* ---- context ------------------------------------------------------------------------- */
int32_t agp_init(agp_ctx** ctx, int32_t device, const agp_config* cfg);
/* one process per GPU, NCCL across processes (rank 0 creates the id, host code ships it) */
int32_t agp_nccl_unique_id(void* out128);
int32_t agp_init_dist(agp_ctx** ctx, int32_t device, int32_t rank, int32_t nranks,
                      int32_t grid_p, int32_t grid_q, const void* nccl_unique_id128,
                      const agp_config* cfg);
int32_t agp_destroy(agp_ctx* ctx);
const char* agp_last_error(const agp_ctx* ctx);
int64_t agp_last_info(const agp_ctx* ctx); /* LAPACK-style failing pivot (1-based) after NOT_POSDEF */
int32_t agp_set_memspace(agp_ctx* ctx, int32_t memspace);
int32_t agp_set_config(agp_ctx* ctx, const agp_config* cfg); /* change the tunables of a live ctx (bench / tests) */
int32_t agp_get_config(const agp_ctx* ctx, agp_config* out);
const char* agp_version(void);

/* instrumentation for bench.py: per-phase device times (CUDA events on the launching stream)
 * of the LAST call: out[0]=total [1]=h2d [2]=gram [3]=cholesky [4]=solves [5]=d2h [6]=predict
 * [7]=trailing-update kernels only (sum), all in ms; returns number of doubles written. */
int32_t agp_last_timings(const agp_ctx* ctx, double* out, int32_t n);
int64_t agp_launch_count(const agp_ctx* ctx); /* kernels launched by this ctx so far */

/* ---- Gram only: cov(f, x) / cov(f, x, z) / cov(fx)  ---------------------------------------
 * replaces kernelmatrix(k,x[,z]) at src/base_gp.jl:70,74 and `C + Sigma_y`
 * src/finite_gp_projection.jl:96,135.  Z == NULL -> symmetric N x N (+ noise on the diagonal
 * when noise != NULL); else N x M cross-Gram.  K_out column-major, leading dim N. */
int32_t agp_gram(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, int32_t layout, const void* X,
                 int64_t N, int32_t D, const void* Z, int64_t M, const agp_noise* noise,
                 void* K_out);

/* ---- fused fit: ONE Gram + ONE Cholesky -> logpdf for S columns of Y, alpha, posterior ------
 * replaces logpdf(::FiniteGP, Y) src/finite_gp_projection.jl:306-311 (+ _sqmahal :325-326,
 * tr_Xt_invA_X / diag_Xt_invA_X src/util/common_covmat_ops.jl:90,101) AND
 * posterior(fx, y) src/exact_gpr_posterior.jl:29-35 (alpha = C \ (y - m) for column 0 of Y).
 * Y: N x S column-major.  logpdf_out: S values (`dtype`).  alpha_out: N values or NULL.
 * post_out: NULL or receives a handle owning the device-resident factor. */
int32_t agp_fit(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean,
                const agp_noise* noise, int32_t layout, const void* X, int64_t N, int32_t D,
                const void* Y, int32_t S, void* logpdf_out, void* alpha_out, agp_post** post_out);

/* mean_and_var(::PosteriorGP, x*) src/exact_gpr_posterior.jl:85-90 (+ mean :60-62, var :68-70);
 * with noise != NULL also mean_and_var(::FiniteGP) src/finite_gp_projection.jl:154-158.
 * mean_s == NULL -> the prior mean given at fit time (zero/const only). */
int32_t agp_post_mean_var(agp_post* p, int32_t layout, const void* Xs, int64_t M,
                          const agp_mean* mean_s, const agp_noise* noise_s, void* mean_out,
                          void* var_out);
/* mean_and_cov(::PosteriorGP, x*) src/exact_gpr_posterior.jl:78-83 (Xt_invA_X
 * src/util/common_covmat_ops.jl:54-58).  cov_out M x M column-major. */
int32_t agp_post_mean_cov(agp_post* p, int32_t layout, const void* Xs, int64_t M,
                          const agp_mean* mean_s, void* mean_out, void* cov_out);
/* logpdf(f_post(x*, Sigma*), Y): src/finite_gp_projection.jl:306-311 (matrix Y :313-318) for a
 * FiniteGP over a PosteriorGP -- mean_and_cov(f_post, x*) src/exact_gpr_posterior.jl:78-83 is formed on
 * the device, Sigma* (noise_s; NULL -> 1e-18) added, factored in place; the M x M covariance never visits
 * the host.  Y is M x S column-major, S <= 128; logpdf_out[S].  AGP_ERR_NOT_POSDEF as agp_fit. */
int32_t agp_post_logpdf(agp_post* p, int32_t layout, const void* Xs, int64_t M,
                        const agp_mean* mean_s, const agp_noise* noise_s, const void* Y, int32_t S,
                        void* logpdf_out);
/* rand(f_post(x*, Sigma*), S): src/finite_gp_projection.jl:233-240, out = m* + chol(C* + Sigma*).U' Z with
 * caller-supplied standard normals Z (M x S column-major) as agp_rand. */
int32_t agp_post_rand(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                      const agp_noise* noise_s, const void* Z, int32_t S, void* out);
/* EXPERIMENTAL -- compiled, not yet validated on a device (SURVEY s8f rank 1).  Gradient of logpdf(fx, y) with
 * respect to the hyper-parameters, from the factor and alpha that agp_fit left in the handle: what reverse-mode AD
 * returns through the reference's logpdf (test/finite_gp_projection.jl:152-178, examples/1-mauna-loa/script.jl:200-242).
 * grad_out (double, 5 + D entries): [0] d/d variance, [1] d/d ScaleTransform s, [2] d/d LinearKernel c,
 * [3] d/d sigma^2 (scalar noise; = 1/2 tr W), [4] d/d ConstMean c, [5 + d] d/d ARDTransform v_d.
 * noise_diag_out (N elements of the handle's dtype, or NULL): d/d sigma_i^2 for per-point noise, and -- via
 * d/d m_i = alpha_i -- the caller already holds the gradient w.r.t. a vector mean.
 * Composite handle (AGP_COMPOSITE): grad_out has agp_post_grad_len(p) entries.  [0..2] are 0, [3] and [4] as above, and
 * from [5] each term in order takes d/d variance[t], then, for each of its factors in order: d/d s (Scale) or d/d v[0..D)
 * (ARD), then d/d param (RQ alpha, Linear c, Constant c), then d/d r[0..D) (Periodic).  A White factor's entries are 0
 * (the kernel is piecewise constant in its inputs' transform). */
int32_t agp_post_logpdf_grad(agp_post* p, double* grad_out, void* noise_diag_out);
/* The same gradient and, in the same call, the gradient of logpdf(fx, y) with respect to the input points -- what
 * reverse-mode AD returns for `x` through the reference's logpdf (test/finite_gp_projection.jl:162-173), and what trains
 * a feature network under the GP (examples/2-deep-kernel-learning).  With W = alpha alpha' - C^-1, for point i and
 * input dimension d:
 *   x_grad[i, d] = sum_j W_ij d1k(x_i, x_j)_d      (j over all points, j == i included)
 * d1 the derivative in the FIRST argument, taken with respect to the untransformed input (the Scale / ARD chain factor
 * is included).  Per factor, leaving out the variances (with t the Scale s, the ARD v or 1, x~ = t x):
 *   SE / Matern / RQ   2 kappa'(d2) t^2 (x_i - x_j)          Linear   t^2 x_j   (so the diagonal term t^2 x_i counts)
 *   Periodic           kappa (-pi t_d / (2 r_d^2)) sinpi(2 t_d (x_i - x_j)_d)   White / Constant   0
 * and the product rule over a composite's terms.  Coincident points (x~_i == x~_j, i == j included) contribute exactly 0
 * for every stationary factor: the limit for SE, Matern 3/2 and 5/2, RQ and Periodic, and the zero subgradient of
 * Matern 1/2, which is not differentiable there.  Finite inputs never give NaN.  Summed in fp64 whatever the dtype, in a
 * fixed order: two calls on the same handle give the same bits.
 * grad_out and noise_diag_out are as agp_post_logpdf_grad's; either may be NULL (that part is then not reduced).
 * x_grad_out: N x D values of the handle's dtype in `layout` -- AGP_POINT_MAJOR: D x N column-major, AGP_FEATURE_MAJOR:
 * N x D column-major; a DEVICE pointer under AGP_MEM_DEVICE; NULL: not computed.  C^-1 (the ~N^3 part) is formed once
 * for everything requested.  Like agp_post_logpdf_grad this is the gradient for the one column of Y whose alpha the
 * handle holds, and only for a handle straight from agp_fit: an extended handle gives AGP_ERR_UNSUPPORTED.  A layout
 * other than the two gives AGP_ERR_INVALID.  agp_post_logpdf_grad(p, g, nd) is agp_post_logpdf_grad_x(p, g, nd,
 * AGP_POINT_MAJOR, NULL). */
int32_t agp_post_logpdf_grad_x(agp_post* p, double* grad_out, void* noise_diag_out, int32_t layout, void* x_grad_out);
/* The gradient of sum_s w_s logpdf(fx, Y[:, s]) for a matrix Y (N x S column-major, any S >= 1) from the factor of the
 * handle, with w = lp_bar the cotangent of the S-vector of logpdfs: what reverse-mode AD returns through the reference's
 * logpdf(fx, Y::AbstractMatrix) and loglikelihood(fx, Y) (test/finite_gp_projection.jl:165-178; w = 1 for loglikelihood).
 * With delta_s = Y[:, s] - m, alpha_s = C^-1 delta_s, A = [alpha_1 .. alpha_S] and
 *   W = A diag(w) A' - (sum_s w_s) C^-1
 * the outputs are the reductions of agp_post_logpdf_grad_x with this W in place of alpha alpha' - C^-1:
 *   d/d theta = 1/2 sum_ij W_ij dK_ij/dtheta,  d/d sigma^2 = 1/2 tr W,  d/d sigma_i^2 = 1/2 W_ii,
 *   x_grad[i, d] = sum_j W_ij d1k(x_i, x_j)_d,  mbar = A w (d/d m_i),  d/d ConstMean c = sum_i mbar_i,
 *   y_bar = -A diag(w)  (N x S column-major, the cotangent of Y).
 * The pullback is evaluated at this Y, which need not be the one the handle was fit with.  mean: the prior mean at the
 * handle's points (host arrays); NULL means the handle's zero or constant mean.  The handle keeps no vector mean, so a
 * CustomMean's values must be passed again.  lp_bar: S host doubles; NULL means all ones.
 * grad_out (double): the layout of agp_post_logpdf_grad -- 5 + D for a single kernel, agp_post_grad_len(p) for a
 * composite; [3] is 1/2 tr W, [4] sum_i mbar_i.  noise_diag_out, mean_diag_out (N values each) and y_bar_out (N x S) have
 * the handle's dtype; x_grad_out is in `layout`, as agp_post_logpdf_grad_x's.  Under AGP_MEM_DEVICE, Y and these four are
 * DEVICE pointers.  Every output may be NULL, and its work is skipped (C^-1, the rank-S updates and the reductions run
 * only for grad_out, noise_diag_out or x_grad_out).
 * Arithmetic: that of agp_post_logpdf_grad_x in the handle's dtype (V = L^-1, C^-1 and A in T, the sums in fp64), so at
 * S = 1, w = 1 the two agree to the dtype's rounding.  A = V' (L^-1 Delta) is formed on the tile GEMM in column chunks of
 * up to 1024.  Cost: the logpdf gradient's ~2 N^3 flop (V and C^-1 = V'V), plus ~N^2 S for the substitution of the
 * columns, 2 N^2 S for A and N^2 S for the lower half of the rank-S update: ~4 N^2 S flop.  Memory: besides the handle,
 * two N x N buffers of T (as agp_post_logpdf_grad_x), two N x min(S, 1024) chunk buffers and, for a host Y, the copy of
 * one chunk of it; nothing else grows with S.
 * Determinism: noise_diag_out, mean_diag_out, x_grad_out and y_bar_out are formed in a fixed order (two calls give the
 * same bits), grad_out[4] too; the other entries of grad_out leave their CTAs through fp64 atomics and agree to rounding.
 * Errors: S < 1, a NULL Y, a bad layout, or a vector mean with a NULL v: AGP_ERR_INVALID; an extended handle:
 * AGP_ERR_UNSUPPORTED; a failed device allocation: AGP_ERR_CUDA. */
int32_t agp_post_logpdf_grad_cols(agp_post* p, const agp_mean* mean, const void* Y, int32_t S, const double* lp_bar,
                                  double* grad_out, void* noise_diag_out, void* mean_diag_out, int32_t layout,
                                  void* x_grad_out, void* y_bar_out);
/* The gradient of the held-out log-likelihood of a posterior,
 *   F = sum_s w_s logpdf(posterior(fx, y)(x*, Sigma*), Y*[:, s]),   w = lp_bar (S host doubles; NULL means ones),
 * with respect to both sides of the problem: the kernel, the training noise, mean, targets and inputs of the handle, and
 * the test noise, mean, targets and inputs -- what reverse-mode AD returns through the reference's
 * logpdf(posterior(fx, y)(x_test, s2), y_test) (examples/0-intro-1d/script.jl's model score).  p must come straight
 * from agp_fit; y is its target column 0.  With C = K_xx + Sigma_y = L L', delta = y - m, alpha = C^-1 delta,
 * mu* = m* + K_sx alpha, Sigma = K_ss - K_sx C^-1 K_xs + Sigma*, E = Y* - mu* 1', B = Sigma^-1 E,
 * P = C^-1 K_xs = V'A (V = L^-1, A = L^-1 K_xs) and beta = P mubar:
 *   Sigmabar = 1/2 (B diag(w) B' - (sum w) Sigma^-1),  mubar = B w,  Ybar* = -B diag(w)
 *   Kbar_ss = Sigmabar,  Kbar_sx = mubar alpha' - 2 Sigmabar P' (M x N),  Cbar = Kbar_xx = P Sigmabar P' - 1/2 (beta alpha' + alpha beta')
 *   ybar = beta,  mbar = -beta at x,  mbar* = mubar,  d/d sigma_i^2 = Cbar_ii,  d/d sigma*_m^2 = Sigmabar_mm,
 *   d/d ConstMean c = sum mubar - sum beta,  d/d theta = <Cbar, dK_xx> + <Kbar_sx, dK_sx> + <Sigmabar, dK_ss>
 *   x_grad[i]  = 2 sum_j Cbar_ij d1k(x_i, x_j) + sum_m Kbar_sx[m, i] d2k(x*_m, x_i)
 *   xs_grad[m] = 2 sum_m' Sigmabar_mm' d1k(x*_m, x*_m') + sum_i Kbar_sx[m, i] d1k(x*_m, x_i)
 * (d1 / d2 as agp_post_logpdf_grad_x's, through the Scale / ARD chain).  The three kernel blocks are reduced as one
 * symmetric W = [2 Cbar, Kbar_xs; Kbar_sx, 2 Sigmabar] over the stacked points [x; x*], by the reductions of
 * agp_post_logpdf_grad_x, so a composite handle is covered as a single kernel is.
 * Inputs: Xs (M points in `layout`), mean_s (the prior mean at x*, as agp_post_logpdf's; NULL means the handle's zero or
 * constant mean), noise_s (Sigma*; NULL means 1e-18), Ys (M x S column-major, any S >= 1).
 * Outputs, each may be NULL and its work is then skipped: lp_out (S values, logpdf of each column), grad_out (double, the
 * layout of agp_post_logpdf_grad: 5 + D for a single kernel, agp_post_grad_len(p) for a composite; [3] d/d sigma^2 of
 * the training scalar noise, [4] d/d ConstMean c), noise_diag_out, mean_diag_out and y_bar_out (N values each),
 * x_grad_out (N x D in `layout`), noise_s_diag_out and mean_s_diag_out (M values each), ys_bar_out (M x S) and
 * xs_grad_out (M x D in `layout`).  Every output but grad_out has the handle's dtype; under AGP_MEM_DEVICE, Xs, Ys and
 * those outputs are DEVICE pointers.  The gradient of a scalar test noise is the sum of noise_s_diag_out.
 * Arithmetic: the handle's dtype for the factors, V, P and the products, fp64 for the reductions (as
 * agp_post_logpdf_grad_x); the error of fp32 handles grows with cond(C), and the kernel gradient of a Linear prior at
 * N >> D, a difference of nearly equal terms, can be off by tens of percent in fp32 (DESIGN s6): use an fp64 handle
 * there.  Cost: the forward of agp_post_logpdf (N^2 M for A, M^3 / 3 for the factor of Sigma), M^3 for
 * Sigma^-1, 4 M^2 S for the columns, then, when a kernel, noise, x or x* output or one of the training-side outputs is
 * asked for, ~N^3 for V, 2 N^2 M for P, 2 N M^2 for Kbar_sx, N^2 M for Cbar (the lower half), and the reductions over
 * (N + M)^2 / 2 pairs.  Memory, besides the handle, in elements of the handle's dtype: about NM + 3 M^2 while Sigma is
 * factored and inverted, N^2 + 2 NM + M^2 while V is live (V, K_xs / A, P, Sigmabar), then (N + M)^2 + NM + M^2 for the
 * stacked W (which also holds the 2 NM elements of its unused upper block), P and Sigmabar: each buffer is freed when it
 * is dead, so the peak is the last.  Add two M x min(S, 1024) chunk buffers.  S goes through in chunks of up to 1024 columns.
 * Determinism: every per-point output and grad_out[3], grad_out[4] are formed in a fixed order (two calls give the same
 * bits); the other entries of grad_out leave their CTAs through fp64 atomics and agree to rounding.
 * Errors: a bad layout, S < 1, a NULL Ys or Xs, or a vector mean / noise with a NULL v: AGP_ERR_INVALID; M < 1:
 * AGP_ERR_DIM_MISMATCH; an extended handle: AGP_ERR_UNSUPPORTED; a Sigma that is not positive definite:
 * AGP_ERR_NOT_POSDEF (agp_last_info gives the pivot); a failed device allocation: AGP_ERR_CUDA.  VFE posteriors are not
 * covered. */
int32_t agp_post_pred_logpdf_grad(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                                  const agp_noise* noise_s, const void* Ys, int32_t S, const double* lp_bar, void* lp_out,
                                  double* grad_out, void* noise_diag_out, void* mean_diag_out, void* y_bar_out,
                                  void* x_grad_out, void* noise_s_diag_out, void* mean_s_diag_out, void* ys_bar_out,
                                  void* xs_grad_out);
/* Pullback of agp_post_rand at the same arguments: what reverse-mode AD returns through the reference's
 * rand(rng, posterior(fx, y)(x*, Sigma*), S) (test/finite_gp_projection.jl:105-127 over a posterior), for Monte Carlo
 * acquisition functions (q-EI, q-NEI, q-KG) and losses built on reparameterised posterior samples.  p must come straight
 * from agp_fit.  With C = K_xx + Sigma_y = L L', alpha = C^-1 (y - m), A = L^-1 K_xs, P = C^-1 K_xs = L^-T A,
 * mu* = m* + K_sx alpha, Sigma = K_ss + Sigma* - A'A = L* L*', out = mu* 1' + L* Z, Obar the cotangent of out (M x S
 * column-major, like Z) and V* = L*^-1:
 *   z_bar = L*' Obar,  mubar = Obar 1,  Sigmabar = 1/2 V*' Q V*,  Q symmetric with the lower triangle (diagonal included)
 *           of z_bar Z'   (agp_rand_grad's Cholesky pullback, applied to L*)
 * and from Sigmabar and mubar the formulas of agp_post_pred_logpdf_grad, unchanged:
 *   Kbar_sx = mubar alpha' - 2 Sigmabar P',  Cbar = P Sigmabar P' - 1/2 (beta alpha' + alpha beta'),  beta = P mubar,
 *   ybar = beta,  mbar = -beta at x,  mbar* = mubar,  d/d sigma_i^2 = Cbar_ii,  d/d sigma*_m^2 = Sigmabar_mm,
 *   d/d ConstMean c = sum mubar - sum beta,  both input gradients from the stacked W over [x; x*].
 * Inputs: Xs, mean_s, noise_s as agp_post_rand's (NULL mean_s: the handle's zero or constant mean; NULL noise_s: 1e-18),
 * Z and out_bar (M x S each, any S >= 1).
 * Outputs, each may be NULL and its work is then skipped: grad_out (double, the layout of agp_post_logpdf_grad: 5 + D for
 * a single kernel, agp_post_grad_len(p) for a composite; [3] d/d sigma^2 of the training scalar noise, [4] d/d ConstMean
 * c), noise_diag_out, mean_diag_out and y_bar_out (N values each), x_grad_out (N x D in `layout`), noise_s_diag_out and
 * mean_s_diag_out (M values each), z_bar_out (M x S) and xs_grad_out (M x D in `layout`).  Every output but grad_out has
 * the handle's dtype; under AGP_MEM_DEVICE, Xs, Z, out_bar and those outputs are DEVICE pointers.  The gradient of a
 * scalar test noise is the sum of noise_s_diag_out.
 * Cost: the forward of agp_post_rand (N^2 M for A, M^3 / 3 for the factor of Sigma, M^2 S for the sample), then M^2 S for
 * z_bar and, when a kernel, noise, x or x* output is asked for, ~5 M^3 for the head (V* M^3 / 3 .. M^3, Q V* 2 M^3,
 * V*' (Q V*) 2 M^3); when any training-side output is asked for, N^2 M for P (a multi-column backward substitution on
 * L, on the int8-sliced tensor cores above the forward substitution's threshold), then 2 N M^2 for Kbar_sx, N^2 M for
 * Cbar (the lower half) and the reductions over (N + M)^2 / 2 pairs.  There is no N^3 term: V = L^-1 is never formed.
 * Memory, besides the handle, in elements of the handle's dtype: about NM + 4 M^2 + 3 MS for the forward and the head,
 * then NM + M^2 + (N + M)^2 for P, Sigmabar and the stacked W (which also holds the 2 NM elements of its unused upper
 * block); no other N x N buffer is allocated.
 * Arithmetic: the handle's dtype for the factors, V*, P and the products, fp64 for the row sums of Obar and the
 * reductions (as agp_post_pred_logpdf_grad; an fp32 handle keeps only its transformed fp32 points, so there is no fp64
 * refit).  The fp32 error grows with cond(C) and cond(Sigma) (DESIGN s6).
 * Determinism: every per-point output, z_bar_out and grad_out[3], grad_out[4] are formed in a fixed order (two calls give
 * the same bits); the other entries of grad_out leave their CTAs through fp64 atomics and agree to rounding.
 * Errors: a bad layout, S < 1, a NULL Xs, Z or out_bar, or a vector mean / noise with a NULL v: AGP_ERR_INVALID; M < 1:
 * AGP_ERR_DIM_MISMATCH; an extended handle: AGP_ERR_UNSUPPORTED; a Sigma that is not positive definite:
 * AGP_ERR_NOT_POSDEF (agp_last_info gives the pivot); a failed device allocation: AGP_ERR_CUDA.  VFE posteriors are not
 * covered. */
int32_t agp_post_rand_grad(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                           const agp_noise* noise_s, const void* Z, int32_t S, const void* out_bar, double* grad_out,
                           void* noise_diag_out, void* mean_diag_out, void* y_bar_out, void* x_grad_out,
                           void* noise_s_diag_out, void* mean_s_diag_out, void* z_bar_out, void* xs_grad_out);
/* Pullback of agp_post_mean_var at the cotangents mean_bar and var_bar of its two outputs: what reverse-mode AD returns
 * through the reference's mean_and_var(posterior(fx, y)(x*, Sigma*)), for analytic acquisition functions (expected
 * improvement, probability of improvement, UCB: closed forms in mu* and sigma^2 maximised over x*) and losses on
 * predicted means.  p must come straight from agp_fit.  With C = K_xx + Sigma_y = L L', alpha = C^-1 (y - m),
 * A = L^-1 K_xs and P = C^-1 K_xs = L^-T A, mu*_j = m*_j + (K_sx alpha)_j and sigma^2_j = k(x*_j, x*_j) - |A e_j|^2
 * (+ sigma*^2_j); with mbar = mean_bar and vbar = var_bar these are agp_post_pred_logpdf_grad's formulas at
 * mubar = mbar and Sigmabar = diag(vbar):
 *   Kbar_sx[j, n] = mbar_j alpha_n - 2 vbar_j P[n, j],  beta = P mbar,  Cbar = P diag(vbar) P' - 1/2 (beta alpha' + alpha beta'),
 *   ybar = beta,  mbar = -beta at x,  d/d sigma_i^2 = Cbar_ii,  d/d ConstMean c = sum mbar - sum beta,
 *   xs_grad[j] = sum_n Kbar_sx[j, n] d1k(x*_j, x_n) + 2 vbar_j d1k(x*_j, x*_j)
 * (d1 as agp_post_logpdf_grad_x's, through the Scale / ARD chain; the last term is nonzero only through Linear factors and
 * products that contain them).  At x* the gradients with respect to the test mean and test noise are mbar and vbar
 * themselves, so the call does not return them; neither the test mean nor the test noise enters the gradient, so the call
 * takes neither.  A test point on a training point adds exactly 0 through every stationary factor (Matern 1/2: its zero
 * subgradient, as agp_post_logpdf_grad_x).
 * Inputs: Xs (M points in `layout`, as agp_post_mean_var's), mean_bar and var_bar (M values of the handle's dtype each;
 * NULL means zeros).
 * Outputs, each may be NULL and its work is then skipped: grad_out (double, the layout of agp_post_logpdf_grad: 5 + D for
 * a single kernel, agp_post_grad_len(p) for a composite; [3] d/d sigma^2 of the training scalar noise, [4] d/d ConstMean
 * c), noise_diag_out, mean_diag_out and y_bar_out (N values each), x_grad_out (N x D in `layout`) and xs_grad_out (M x D
 * in `layout`).  Every output but grad_out has the handle's dtype; under AGP_MEM_DEVICE, Xs, mean_bar, var_bar and those
 * outputs are DEVICE pointers.
 * Routes, one per output: xs_grad_out always comes from one pass over the N x M pairs (x*_j, x_n) that forms Kbar_sx from
 * P on the fly; grad_out, noise_diag_out and x_grad_out come from agp_post_pred_logpdf_grad's stacked reductions over
 * [x; x*] with Sigmabar = diag(vbar); y_bar_out and mean_diag_out alone need only beta, one GEMV.  Passing NULL for every
 * training-side output gives the test-side-only call an optimiser over x* needs.
 * Cost: N^2 M for A (K_xs, then a multi-column forward substitution) and N^2 M for P (a backward substitution on L; both on
 * the int8-sliced tensor cores above the substitutions' threshold), then N M D for the x* pass; when a kernel, noise or
 * x output is asked for, 2 N M^2 for Kbar_sx, N^2 M for Cbar (the lower half) and the reductions over (N + M)^2 / 2 pairs.
 * There is no N^3 or M^3 term: neither L^-1, C^-1 nor the posterior covariance is formed.
 * Memory, besides the handle, in elements of the handle's dtype: about NM for A and P (P overwrites A) and O((N + M) D)
 * for the x* pass when no kernel, noise or x output is asked for (no N x N or (N + M)^2 buffer); otherwise 2 NM briefly,
 * then NM + M^2 + (N + M)^2 for P, Sigmabar and the stacked W.
 * Arithmetic: the handle's dtype for K_xs, A, P and the products, fp64 for the x* pass (its weights and sums) and the
 * reductions.  The fp32 error grows with cond(C) through P (DESIGN s6).
 * Determinism: every per-point output and grad_out[3], grad_out[4] are formed in a fixed order (the x* pass writes
 * per-CTA fp64 partials summed in a fixed order: two calls give the same bits); the other entries of grad_out leave their
 * CTAs through fp64 atomics and agree to rounding.
 * Errors: a bad layout or a NULL Xs: AGP_ERR_INVALID; M < 1: AGP_ERR_DIM_MISMATCH; an extended handle:
 * AGP_ERR_UNSUPPORTED; a failed device allocation: AGP_ERR_CUDA.  VFE posteriors are not covered. */
int32_t agp_post_mean_var_grad(agp_post* p, int32_t layout, const void* Xs, int64_t M, const void* mean_bar,
                               const void* var_bar, double* grad_out, void* noise_diag_out, void* mean_diag_out,
                               void* y_bar_out, void* x_grad_out, void* xs_grad_out);
/* number of doubles agp_post_logpdf_grad writes: 5 + D for a single kernel, the layout above for a composite */
int64_t agp_post_grad_len(const agp_post* p);
/* V = U' \ B (N x nrhs, column-major): backs Xt_invA_X / diag_Xt_invA_X / Xt_invA_Y /
 * tr_Xt_invA_X on a device factor, src/util/common_covmat_ops.jl:54-60,90,101. */
int32_t agp_post_solve_lower(agp_post* p, const void* B, int64_t nrhs, void* V_out);
/* C.U for p.data.C.U compatibility (test/exact_gpr_posterior.jl:40): N x N column-major upper */
int32_t agp_post_factor_export(agp_post* p, void* U_out);
int32_t agp_post_logdet(agp_post* p, double* logdet_out); /* logdet(C) = 2 sum log U_ii */
int64_t agp_post_n(const agp_post* p);
/* sequential conditioning: posterior(fx::FiniteGP{<:PosteriorGP}, y) src/exact_gpr_posterior.jl:46-56
 * via update_chol src/util/common_covmat_ops.jl:38-42.  alpha_out receives the N1+N2 re-solved weights
 * (or NULL).  post_out != NULL: a NEW handle is returned and p stays valid (the reference's value
 * semantics -- both posteriors usable, both to be freed); post_out == NULL: p is extended in place. */
int32_t agp_post_extend(agp_post* p, int32_t layout, const void* X2, int64_t N2, const void* y2,
                        const agp_mean* mean2, const agp_noise* noise2, void* alpha_out,
                        agp_post** post_out);
int32_t agp_post_free(agp_post* p);

/* rand(rng, fx, S) / _rand! src/finite_gp_projection.jl:233-237,271-277: out = m + U' Z with the
 * caller's standard normals Z (N x S column-major) -- the RNG stream stays host-defined. */
int32_t agp_rand(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean,
                 const agp_noise* noise, int32_t layout, const void* X, int64_t N, int32_t D,
                 const void* Z, int32_t S, void* out);
/* Pullback of agp_rand at the same arguments: what reverse-mode AD returns through the reference's rand(rng, fx, S)
 * (test/finite_gp_projection.jl:105-127), for reparameterised Monte Carlo objectives and losses built on prior samples.
 * With out = m + L Z, C = K + Sigma_y = L L', Obar the cotangent of out (N x S column-major, like Z) and V = L^-1:
 *   z_bar = L' Obar                                   (N x S column-major, the cotangent of the normals Z)
 *   mbar_i = sum_s Obar_is;  d/d ConstMean c = sum_i mbar_i
 *   2 Cbar = V' Q V,  Q symmetric with the lower triangle (diagonal included) of z_bar Z'    (Murray 2016, symmetric form:
 *            Lbar = tril(Obar Z'), and the lower triangle of L' Lbar is that of z_bar Z')
 * and with W = 2 Cbar, exactly the reductions of agp_post_logpdf_grad_x with alpha = 0 and C^-1 replaced by -V'QV:
 *   d/d theta = 1/2 sum_ij W_ij dK_ij/dtheta,  d/d sigma^2 = 1/2 tr W,  d/d sigma_i^2 = 1/2 W_ii,
 *   x_grad[i, d] = sum_j W_ij d1k(x_i, x_j)_d.
 * grad_out (double): the layout of agp_post_logpdf_grad -- 5 + D for a single kernel, agp_post_grad_len's composite layout
 * for AGP_COMPOSITE; [3] is d/d sigma^2 of a scalar noise, [4] d/d ConstMean c.
 * noise_diag_out / mean_diag_out: N values of `dtype` (d/d sigma_i^2, d/d m_i); x_grad_out: N x D values of `dtype` in
 * `layout`, as agp_post_logpdf_grad_x's; z_bar_out: N x S values of `dtype`.  Under AGP_MEM_DEVICE, X, Z, out_bar and these
 * four are DEVICE pointers.  Every output may be NULL, and its work is skipped (z_bar is formed whatever is requested; V,
 * Q and the reductions only when grad_out, noise_diag_out or x_grad_out is requested).  A vector (CustomMean) mean and
 * per-point noise are constants of X: the caller chains through mean_diag_out and noise_diag_out.
 * Cost: the factor-only fit, then ~4 N^3 flop on the tile GEMM and the forward substitution (the substitution on the
 * identity N^3, Q V 2 N^3, the lower half of V' (Q V) N^3), ~2x the logpdf gradient's.  Memory: the factor plus three
 * N x N fp64 buffers whatever the dtype: (N + 128) N 8 + 3 N^2 8 bytes, plus O(N) terms (the int8-slice workspace of
 * the substitution, ~7 kB per row) -- an estimate, ~65 GB at N = 45 000; the largest N that fits has not been measured.
 * For AGP_F32 the pullback is formed in fp64 on the problem converted to fp64 and its outputs rounded to fp32: V'QV
 * carries terms of the order of cond(C) that cancel.  mean_diag_out and grad_out[4] are summed in a fixed order; the
 * other outputs are those of the reductions of agp_post_logpdf_grad_x (noise_diag_out and x_grad_out in a fixed order:
 * two calls give the same bits).  Errors: a bad layout, S < 0, or a NULL X, or NULL Z / out_bar with S > 0:
 * AGP_ERR_INVALID; a distributed context: AGP_ERR_UNSUPPORTED; C not positive definite: AGP_ERR_NOT_POSDEF with
 * agp_last_info, as agp_rand; a failed device allocation: AGP_ERR_CUDA. */
int32_t agp_rand_grad(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                      int32_t layout, const void* X, int64_t N, int32_t D, const void* Z, int32_t S,
                      const void* out_bar, double* grad_out, void* noise_diag_out, void* mean_diag_out,
                      void* x_grad_out, void* z_bar_out);

/* ---- VFE (Titsias) -------------------------------------------------------------------------
 * approx_log_evidence(::VFE)/elbo src/sparse_approximations.jl:248-254 with
 * _compute_intermediates :289-305 and tr_Cf_invSigma_y :307-313; dtc_out (optional) is the DTC
 * objective :282-286.  Only diagonal Sigma_y (as in the reference, :307-313). */
int32_t agp_vfe_elbo(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean,
                     const agp_noise* noise, int32_t layout, const void* X, int64_t N, int32_t D,
                     const void* Zind, int64_t M, const agp_noise* jitter, const void* y,
                     void* elbo_out, void* dtc_out);
/* Gradient of approx_log_evidence(VFE | DTC, fx, y), src/sparse_approximations.jl:248-254 / :282-286: what reverse-mode
 * AD returns through the reference when a sparse GP is trained.  objective 0 = elbo, 1 = DTC.  With s_i = sigma_i^2,
 * delta = s^-1/2 (y - m), K_zz + J = L_z L_z', A = L_z^-1 K_zx S^-1/2, Lam = I + A A', m_e = Lam^-1 A delta, V_z = L_z^-1
 * and c = 1 (elbo) | 0 (DTC):
 *   Kbar_zx = V_z' H V_z K_zx S^-1 + V_z' m_e (delta o s^-1/2)',  H = c I - Lam^-1 - m_e m_e'
 *   Kbar_zz = -1/2 V_z' E V_z,  E = c (Lam - I) - I + Lam^-1 + m_e m_e';   kdiagbar_i = -c / (2 s_i)
 *   d/d theta = sum Kbar_zz o dK_zz + sum Kbar_zx o dK_zx + sum kdiagbar o dkdiag
 *   d/d z_m = 2 sum_m' Kbar_zz[m, m'] d1k(z_m, z_m') + sum_n Kbar_zx[m, n] d1k(z_m, x_n)
 *   d/d s_i = -1/(2 s_i) + c kdiag_i/(2 s_i^2) - q_i/(2 s_i) - deltabar_i delta_i/(2 s_i),  d/d m_i = -s_i^-1/2 deltabar_i
 *   with u = K_zx' V_z' m_e, q_i = sum_m Kbar_zx[m, i] K_zx[m, i], deltabar = -delta + s^-1/2 o u.
 * value_out: 1 value of `dtype`, computed by the pass agp_vfe_elbo makes (for fp32 that fp32 pass itself); it agrees with
 * agp_vfe_elbo's value to rounding, not bit for bit, because that pass sums its scalars with fp64 atomics.
 * grad_out (double, 5 + D, NULL allowed): the layout of agp_post_logpdf_grad -- [3] is d/d sigma^2 of a scalar noise
 * (the sum of the per-point derivatives), [4] d/d ConstMean c (the sum of the per-point ones).
 * noise_diag_out / mean_diag_out: N values of `dtype` (d/d sigma_i^2, d/d m_i) or NULL.
 * z_grad_out: M x D values of `dtype` in `layout` (AGP_POINT_MAJOR: D x M column-major, AGP_FEATURE_MAJOR: M x D
 * column-major), with respect to the untransformed inducing points, or NULL; a DEVICE pointer under AGP_MEM_DEVICE, as are
 * noise_diag_out and mean_diag_out.  Coincident points contribute 0 for the stationary families (agp_post_logpdf_grad_x).
 * Single kernels only (the kernels agp_vfe_elbo accepts).  For AGP_F32 the gradient is formed in fp64 on the problem
 * converted to fp64 (its own pass 1 included) and rounded to fp32 at the end: the adjoints are differences of terms up
 * to ~1e5 times larger than the result, which fp32 arithmetic cannot carry.  G = R K_zx runs on the int8-slice product
 * where pass 1's long-K product does (M >= 1024 under the automatic policy), on the tile GEMM otherwise.  The gradient
 * with respect to X is agp_vfe_elbo_grad_x's; the gradient with respect to the jitter is not formed.
 * Summed in fp64.  noise_diag_out, mean_diag_out and z_grad_out are summed in a fixed order (two calls give the same bits);
 * the grad_out sums leave their CTAs through fp64 atomics, so two calls agree to rounding.  Errors: an objective other
 * than 0 / 1 or a bad layout: AGP_ERR_INVALID; composite kernels and distributed contexts: AGP_ERR_UNSUPPORTED;
 * K_zz + J or Lam not positive definite: AGP_ERR_NOT_POSDEF with agp_last_info, as agp_vfe_elbo. */
int32_t agp_vfe_elbo_grad(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                          int32_t layout, const void* X, int64_t N, int32_t D, const void* Zind, int64_t M,
                          const agp_noise* jitter, const void* y, int32_t objective, void* value_out, double* grad_out,
                          void* noise_diag_out, void* mean_diag_out, void* z_grad_out);
/* The same outputs and, from the same passes, the gradient with respect to the training inputs X -- what reverse-mode AD
 * returns for `x` through the reference's elbo, and what trains a feature network under a sparse GP
 * (examples/2-deep-kernel-learning).  For data point n and input dimension d, with respect to the untransformed input:
 *   x_grad[n, d] = sum_m Kbar_zx[m, n] dk(z_m, x_n)/dx_n[d] + kdiagbar_n dkdiag(x_n)/dx_n[d],   kdiagbar_n = -c / (2 s_n)
 * With t the Scale s, the ARD v or 1 and x~ = t x:
 *   SE / Matern   x_grad[n, d] = -sigma^2 t_d sum_m Kbar_zx[m, n] q(d2_mn) (z~_md - x~_nd),  q = kappa'(r) / r, the
 *                 coefficient of z_grad's K_zx part with the opposite sign; coincident points contribute exactly 0 (for
 *                 Matern 1/2 the zero subgradient); the kdiag term is 0
 *   Linear        x_grad[n, d] = sigma^2 t_d (sum_m Kbar_zx[m, n] z~_md - c x~_nd / s_n)   (the second term is kdiag's)
 * The mean and per-point noise are constants of X: the caller chains through mean_diag_out and noise_diag_out.
 * x_grad_out: N x D values of `dtype` in `layout` (AGP_POINT_MAJOR: D x N column-major, AGP_FEATURE_MAJOR: N x D
 * column-major), a DEVICE pointer under AGP_MEM_DEVICE; NULL: not computed.  Summed in fp64 in a fixed order (two calls
 * give the same bits); the chunking of the data changes only the rounding.  Per chunk of the streamed pass it adds two
 * launches (vfe_x_grad_kernel, vfe_x_finish_kernel); for AGP_F32 it is formed on the fp64 path like the rest and
 * narrowed at the end.  Errors as agp_vfe_elbo_grad.  agp_vfe_elbo_grad(...) is agp_vfe_elbo_grad_x(..., NULL). */
int32_t agp_vfe_elbo_grad_x(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                            int32_t layout, const void* X, int64_t N, int32_t D, const void* Zind, int64_t M,
                            const agp_noise* jitter, const void* y, int32_t objective, void* value_out, double* grad_out,
                            void* noise_diag_out, void* mean_diag_out, void* z_grad_out, void* x_grad_out);
/* posterior(::VFE, fx, y) src/sparse_approximations.jl:58-75 */
int32_t agp_vfe_fit(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean,
                    const agp_noise* noise, int32_t layout, const void* X, int64_t N, int32_t D,
                    const void* Zind, int64_t M, const agp_noise* jitter, const void* y,
                    agp_vfe_post** out);
/* mean_and_var(::ApproxPosteriorGP, x*) src/sparse_approximations.jl:212-217 */
int32_t agp_vfe_mean_var(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t Ms,
                         void* mean_out, void* var_out);
/* EXPERIMENTAL -- composed of validated kernels, not yet run on a device.
 * mean_and_cov(::ApproxPosteriorGP, x*) src/sparse_approximations.jl:205-210 (cov :187-190); cov_out M x M column-major,
 * no observation noise.  The prior mean at x* is the handle's Zero/Const mean (a closure mean is added by the host). */
int32_t agp_vfe_mean_cov(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t M, void* mean_out,
                         void* cov_out);
/* logpdf(f_approx_post(x*, Sigma*), Y) and rand(f_approx_post(x*, Sigma*), S): src/finite_gp_projection.jl:306-318,
 * :233-240 over the approximate posterior -- C* + Sigma* is formed and factored on the device like agp_post_logpdf. */
int32_t agp_vfe_post_logpdf(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t M, const agp_noise* noise_s,
                            const void* Y, int32_t S, void* logpdf_out);
int32_t agp_vfe_post_rand(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t M, const agp_noise* noise_s,
                          const void* Z, int32_t S, void* out);
int32_t agp_vfe_post_free(agp_vfe_post* p);

/* Device-pointer entry points (AGP_MEM_DEVICE and the agp_debug_* hooks): the library runs on its OWN non-blocking streams
 * and returns after synchronising them, so results are complete on return -- but the CALLER must make sure the device
 * buffers it passes in are complete (synchronise the stream that produced them) before the call. */
/* ---- test hook for the int8-sliced fp64 trailing update (csrc/umma_ozaki.cu): DEVICE pointers;
 * C (M x N, ldc, fp64) -= P P' (lower tiles when lower_only), P = M x K fp64 (lda), S in 5..8 slices. */
int32_t agp_debug_ozaki_syrk(agp_ctx* ctx, void* C_dev, int64_t ldc, const void* P_dev, int64_t lda, int64_t M,
                             int64_t N, int32_t K, int32_t S, int32_t lower_only);

/* general product on the same int8-slice path: C (M x N, N % 128 == 0) += sign * A B' with fp32 or fp64 operands and output,
 * row-contiguous (element (r,k) at [r + k*ld]) or k-major ([k + r*ld]) operands; B_dev == NULL: B = A, lower tiles only.
 * S = number of 7-bit slices (3..5 for fp32 output, 4..8 for fp64). */
int32_t agp_debug_ozaki_gemm(agp_ctx* ctx, void* C_dev, int32_t c_is_float, int64_t ldc, const void* A_dev, int32_t a_is_float,
                             int32_t a_kmajor, int64_t lda, int64_t M, const void* B_dev, int32_t b_is_float, int32_t b_kmajor,
                             int64_t ldb, int64_t N, int32_t K, int32_t S, double sign);
/* same kernel through the block-cyclic column map of the multi-GPU trailing update (the strip-table tile enumeration):
 * P has m_panel rows; row r of C (M x N local columns, N % 128 == 0) pairs with panel row r + a_off, local column n with
 * panel row (n / b_tile_width) * b_tile_stride + n % b_tile_width + b_off; lower tiles only (relative to panel rows). */
int32_t agp_debug_ozaki_syrk_map(agp_ctx* ctx, void* C_dev, int64_t ldc, const void* P_dev, int64_t lda, int64_t m_panel,
                                 int64_t M, int64_t N, int32_t K, int32_t S, int64_t b_tile_stride, int64_t b_tile_width,
                                 int64_t b_off, int64_t a_off);
/* the six-slice eight-bit format of the fp64 path (ozaki_slices = 6), K % 64 == 0 and K <= 16384 (else
 * AGP_ERR_UNSUPPORTED), fp64 operands and C, C (M x N, N % 128 == 0) += sign * A B':
 *  - B_dev != NULL: rectangular product of A (M rows) and B (N rows), each row-contiguous or k-major (*_kmajor);
 *    m_panel, b_tile_stride, b_tile_width, b_off and a_off must be 0;
 *  - B_dev == NULL: A is a panel of m_panel rows, lower tiles only; row r of C pairs with panel row r + a_off, column n
 *    with panel row (n / b_tile_width) * b_tile_stride + n % b_tile_width + b_off (stride 0: n + b_off), all in
 *    multiples of 128 -- the closed-form walk when stride == 0 and a_off == b_off, the strip table otherwise. */
int32_t agp_debug_ozaki8(agp_ctx* ctx, void* C_dev, int64_t ldc, const void* A_dev, int32_t a_kmajor, int64_t lda,
                         int64_t m_panel, const void* B_dev, int32_t b_kmajor, int64_t ldb, int64_t M, int64_t N, int32_t K,
                         double sign, int64_t b_tile_stride, int64_t b_tile_width, int64_t b_off, int64_t a_off);

/* ---- test hook for the tile GEMM (csrc/gemm.cu): DEVICE pointers, dtype AGP_F32 | AGP_F64, one launch on the caller's
 * buffers.  C (M x N, ldc) = beta C + alpha op(A) op(B), alpha = -1 if alpha_neg else +1, beta = 1 if beta_one else 0;
 * A(m,k) at A[m + k*lda] (a_kmajor = 0) or A[k + m*lda]; B(k,n) at B[n + k*ldb] (b_kmajor = 0) or B[k + n*ldb].  C == A
 * or C == B (the same pointer) selects the in-place kernels.  lower_only skips tiles above the diagonal, trmm_lower
 * reads A as lower triangular (K cut at the end of each row tile); column n of C takes B's column
 * (n / w) * b_tile_stride + n % w + b_off (w = b_tile_width, 0 -> 128) when b_tile_stride != 0.  Operands that break
 * the contract of GemmArgs (csrc/kernels.h) are refused with AGP_ERR_INVALID before anything is launched. */
int32_t agp_debug_gemm(agp_ctx* ctx, int32_t dtype, const void* A_dev, int32_t a_kmajor, int64_t lda, const void* B_dev,
                       int32_t b_kmajor, int64_t ldb, void* C_dev, int64_t ldc, int64_t M, int64_t N, int64_t K,
                       int32_t alpha_neg, int32_t beta_one, int32_t lower_only, int32_t trmm_lower, int64_t b_tile_stride,
                       int64_t b_tile_width, int64_t b_off);

/* routes of one step of the blocked Cholesky: how the 128 x 128 diagonal block is factored and the panel below it solved */
#define AGP_PANEL_SPLIT_SUBST 0 /* fp64: factor-only kernel, panel by blocked substitution, inverse on a side stream */
#define AGP_PANEL_SPLIT_GEMM 1  /* fp64: factor-only kernel, strip inverse, panel by one in-place GEMM with the inverse */
#define AGP_PANEL_FUSED 2       /* fused factor + inverse kernel, panel by the in-place GEMM (fp32's only route) */
/* ---- test hook for one panel step (csrc/potrf.cu): DEVICE pointers.  Factors the 128 x 128 block at A (lda, lower
 * triangle read) in place (L, upper triangle zeroed), solves the rows_below rows under it, A21 <- A21 L^-T, and writes
 * Dinv (128 x 128, = inv(L)), logdet[blk] = sum_j log L_jj and, at the first non-positive pivot j (1-based) of the
 * block, info = blk * 128 + j unless info is already nonzero.  Returns once every stream has finished.  fp32 panels need
 * rows_below % 4 == 0 (the panel GEMM's contract; AGP_ERR_INVALID otherwise, before anything runs). */
int32_t agp_debug_panel(agp_ctx* ctx, int32_t dtype, int32_t route, void* A_dev, int64_t lda, int64_t rows_below,
                        int32_t blk, void* Dinv_dev, double* logdet_dev, int32_t* info_dev);

/* ---- host-only helpers of the 2D block-cyclic tile map (no GPU needed; used by the CPU
 * world_size-2 tests): owner rank of tile (i,j) on a P x Q grid and local tile counts. */
int32_t agp_bc_owner(int32_t ti, int32_t tj, int32_t grid_p, int32_t grid_q);
int64_t agp_bc_local_tiles(int32_t ntiles, int32_t rank, int32_t grid_p, int32_t grid_q);

#ifdef __cplusplus
}
#endif
#endif /* AGP_H */
