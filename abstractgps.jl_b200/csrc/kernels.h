// kernels.h -- launch-level interface between the engine (engine.cu) and the sm_90a kernels.
// All matrices are column-major.  TILE = 128 is the factorisation tile edge: every matrix the
// Cholesky touches is padded to a multiple of TILE (identity padding), so kernels on that path
// see no ragged edges; the generic GEMM still bounds-checks for the prediction path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define AGP_TILE 128

// ---- composite kernels: sum of product terms, K = sum_t v_t prod_{f in t} kappa_f (agp.h agp_kernel_composite) -------
#define AGP_COMP_MAX 8
// accumulator kinds: the distances a composite kernel needs, one register block each
enum { COMP_ACC_SQ = 0,    // sum_d (w_d diff_d)^2           (raw: w = 1, shared by every Scale/None stationary factor)
       COMP_ACC_DOT = 1,   // sum_d w_d^2 x_d y_d            (raw: w = 1, shared by every Scale/None Linear factor)
       COMP_ACC_PER = 2 }; // sum_d (sinpi(w_d diff_d) rinv_d)^2   (one per Periodic factor)

struct CompFactor {
  int family, transform;
  int acc;      // accumulator slot; -1: Constant (needs none)
  int term;     // term index
  double s, s2; // Scale s and s^2 applied to a shared raw accumulator (1 otherwise)
  double param; // RQ alpha | Linear c | Constant c
  // gradient slots (indices into grad_out; -1: none): Scale s, param, ARD v base, Periodic r base
  int g_s, g_p, g_w, g_r;
};

struct CompositeDesc {  // passed by value (__grid_constant__); per-dimension weights live in a device array
  int nterms, nfactors, nacc;
  double variance[AGP_COMP_MAX];
  int g_var[AGP_COMP_MAX];       // gradient slot of each term's variance
  CompFactor f[AGP_COMP_MAX];
  int acc_kind[AGP_COMP_MAX];
  // device weights (element type T): accumulator a's w at [2a*D, 2a*D + D), its rinv (Periodic) at [(2a+1)*D, ...)
  const void* w;
};

struct GramParams {
  int family;        // AGP_SE ...
  double variance;   // sigma_f^2
  double linear_c;
  int symmetric;     // 1: Xb == Xa, exact-zero self distance, optional noise on the diagonal
  int lower_only;    // 1: skip 64x64 tiles strictly above the diagonal
  int64_t valid_a;   // rows >= valid_a are padding
  int64_t valid_b;   // cols >= valid_b are padding
  int noise_kind;    // -1 none, 0 scalar, 1 vector
  double noise_s;
  const void* noise_v;  // device, T
  const unsigned char* mask_a;  // optional per-row validity (extended posteriors); overrides valid_a
  const unsigned char* mask_b;
  int64_t noise_off;  // noise_v index offset for the diagonal (block Gram of an extension)
  int64_t diag_off;   // column index offset: column gj of this launch is global column gj + diag_off
  const CompositeDesc* comp;  // family == AGP_COMPOSITE: host copy of the descriptor (its weights are on the device)
};

// op(A) is M x K, op(B) is K x N, C is M x N (ldc).  C = beta*C + alpha*op(A)op(B), alpha in {+1,-1}.
// Contract (launch_gemm checks it on the host and launches nothing, returning nonzero, when it fails):
//  - A and B 16-byte aligned, lda and ldb even (fp64) or multiples of 4 (fp32): the operands are read in 16-byte loads;
//    fp32 also needs C 16-byte aligned, ldc % 4 == 0 and M % 4 == 0 (the epilogue stores float4 and checks only m < M);
//  - lda >= K (A K-major) or M, ldb >= K (B K-major) or 1 + the highest B column the column map reads, ldc >= M;
//  - K even (fp64) or K % 4 == 0 (fp32) when either operand is K-major: a load of k .. k+1 (k+3) checks only k < K, and
//    a NaN past K times the other operand's zero fill would still poison the sum;
//  - C == A: a_kmajor = 0, ldc == lda, N <= 128; C == B: b_kmajor = 1, ldc == ldb, M <= 128, no column map.  One CTA then
//    owns every row (column) of the aliased operand it reads and reads all of them before its epilogue;
//  - column map: stride, width and b_off >= 0, the width a multiple of the instantiation's column tile (fp64: 128 when C
//    aliases an operand, else 64; fp32: 128), and for an MN-major B the shift a multiple of the load width.
// C overlapping an operand only partly (sharing columns but not rows, say) is the caller's business and is not checked.
// Tiles: fp64 64 x 128 (C == A), 128 x 128 (C == B), 128 x 64 otherwise; fp32 128 x 128.  lower_only skips whole tiles,
// trmm_lower cuts K at the end of the row tile, so A is read above its diagonal inside the tile's band.
struct GemmArgs {
  const void* A; int64_t lda; int a_kmajor;  // 0: A(m,k) at A[m + k*lda]   1: A(m,k) at A[k + m*lda]
  const void* B; int64_t ldb; int b_kmajor;  // 0: B(k,n) at B[n + k*ldb]   1: B(k,n) at B[k + n*ldb]
  void* C; int64_t ldc;
  int64_t M, N, K;
  int alpha_neg;     // 1 -> alpha = -1 else +1
  int beta_one;      // 1 -> beta = 1 else 0
  int lower_only;    // 1 -> skip tiles with tile_n > tile_m (SYRK on a diagonal-anchored C)
  int trmm_lower;    // 1 -> A is lower triangular M x K anchored at (0,0): limit k <= row tile end
  // block-cyclic column gather (multi-GPU trailing update): local column n of C takes its B rows from
  // n_src = (n / 128) * b_tile_stride + n % 128 + b_off; 0 = identity.  The lower-only test uses n_src.
  int64_t b_tile_stride, b_off;
  int64_t b_tile_width;  // width of a distribution block in columns (0 -> 128)
};

template <typename T> void launch_prep_points(const T* X, int layout, int64_t n, int64_t n_pad, int D,
                                              int transform, double scale, const T* ard, T* Xt,
                                              cudaStream_t s);
template <typename T> void launch_gram(const T* Xa, const T* Xb, int64_t na_pad, int64_t nb_pad, int D,
                                       T* K, int64_t ldk, const GramParams& p, cudaStream_t s);
template <typename T> void launch_kdiag(const T* Xt, int64_t n, int D, int family, double variance,
                                        double linear_c, T* out, cudaStream_t s, const CompositeDesc* comp = nullptr);
// border rows: E[s, j] = Y[j + s*ldy] - mean_j  (j < n, s < S), 0 elsewhere; E is TILE x n_pad at
// rows [n_pad, n_pad+TILE) of the factor matrix (leading dimension lda).
template <typename T> void launch_border_init(T* A, int64_t lda, int64_t n, int64_t n_pad, const T* Y,
                                              int64_t ldy, int S, int mean_kind, double mean_c,
                                              const T* mean_v, cudaStream_t s);
// same for a block of `ncols` columns of a column-distributed factor: A points at the block's first
// column, border rows start at row_off, column c of the block is global point col0 + c (valid if < n)
template <typename T> void launch_border_init_cols(T* A, int64_t lda, int64_t row_off, int64_t col0, int64_t ncols,
                                                   int64_t n, const T* Y, int64_t ldy, int S, int mean_kind,
                                                   double mean_c, const T* mean_v, cudaStream_t s);
// diagonal block factorisation + inverse: A (TILE x TILE at Ablk, lda) -> L in place (upper zeroed),
// Dinv = inv(L) (TILE x TILE col-major, lower), logdet_part[blk] = sum log L_jj, info (first bad pivot, 1-based).
// One fused kernel; the fp64 factorisation uses it only on the AGP_PANEL_FUSED route (agp.h), the split kernels below
// otherwise.
template <typename T> void launch_potrf_diag(T* Ablk, int64_t lda, T* Dinv, double* logdet_part, int blk,
                                             int* info, cudaStream_t s);
template <typename T> int launch_gemm(const GemmArgs& g, cudaStream_t s);  // 0: launched (or nothing to do); else refused
// fp64 split schedule: factor-only diagonal block, 8-CTA strip inverse (off the critical path), and the
// panel TRSM by blocked substitution that does not need the 128x128 inverse
int potrf_split_enabled();
void launch_potrf_factor_f64(double* Ablk, int64_t lda, double* logdet_part, int blk, int* info, cudaStream_t s);
void launch_trtri_f64(const double* Ablk, int64_t lda, double* Dinv, cudaStream_t s);
void launch_trsm_sub_f64(double* A21, int64_t lda, int64_t M, const double* Lkk, cudaStream_t s);
// v extraction from the border rows + sqmahal: r[s*n_pad + j] = E[s, j], sq[s] = sum_j E[s,j]^2
template <typename T> void launch_extract_v(const T* A, int64_t lda, int64_t n_pad, int S, T* r, double* sq,
                                            cudaStream_t s);
// whole backward substitution in one persistent launch; flags_and_ticket: nblk+1 ints (zeroed inside)
template <typename T> void launch_bwd_solve(const T* A, int64_t lda, const T* Dinv, int nblk, T* r,
                                            int* flags_and_ticket, cudaStream_t s);
// distributed (column-cyclic) backward substitution pieces
template <typename T> void launch_bwd_diag(const T* Dinv_i, const T* r_i, T* alpha_i, cudaStream_t s);
template <typename T> void launch_bwd_update_local(const T* Lloc, int64_t lda, int i_blk, const T* alpha_i, T* r, int nloc,
                                                   int rank, int nranks, int G, cudaStream_t s);
template <typename T> void launch_bwd_update_local_multi(const T* Lloc, int64_t lda, int i_lo, int Gn, const T* alpha_lo, T* r,
                                                         int nloc, int rank, int nranks, int G, int64_t j_min, int64_t j_max,
                                                         cudaStream_t s);
template <typename T> void launch_bwd_block_solve(const T* Lblk, int64_t lda, const T* Dinv_blk, const T* r_blk, T* alpha_blk,
                                                  int Gn, cudaStream_t s);
template <typename T> void launch_finalize_logpdf(const double* logdet_part, int nblk, const double* sq, int S,
                                                  int64_t n, T* out, double* logdet_out, cudaStream_t s);
// mu[j] = mean_j + sum_i B[i + j*ldb] * alpha[i]
template <typename T> void launch_gemv_t(const T* B, int64_t ldb, int64_t n, int64_t m, const T* alpha,
                                         int mean_kind, double mean_c, const T* mean_v, T* mu, cudaStream_t s);
// var[j] = kdiag[j] - sum_i V[i + j*ldv]^2 (+ noise)
template <typename T> void launch_colsumsq_var(const T* V, int64_t ldv, int64_t n, int64_t m, const T* kdiag,
                                               int noise_kind, double noise_s, const T* noise_v, T* var,
                                               cudaStream_t s);
// out[i + j*ldo] = (i<=j) ? L[j + i*lda] : 0     (U = L')
template <typename T> void launch_export_upper(const T* A, int64_t lda, int64_t n, T* U, int64_t ldo,
                                               cudaStream_t s);
template <typename T> void launch_add_mean_cols(T* out, int64_t ldo, int64_t n, int S, int mean_kind,
                                                double mean_c, const T* mean_v, cudaStream_t s);
// C[i + j*ldc] = Kss[i + j*ldc] - C[...]  and symmetrise (mean_and_cov epilogue)
template <typename T> void launch_cov_finish(T* C, int64_t ldc, const T* Kss, int64_t m, cudaStream_t s);
template <typename T> void launch_fill(T* p, int64_t n, double v, cudaStream_t s);
// out[i] = y[i] - mean_i
template <typename T> void launch_sub_mean(const T* y, int64_t n, int mean_kind, double mean_c, const T* mean_v, T* out, cudaStream_t s);
// out[i + j*ldo] = Y[i + j*ldy] - mean_i for i < n, j < nc; 0 elsewhere in the n_pad x nc_pad block
template <typename T> void launch_sub_mean_cols(const T* Y, int64_t ldy, int64_t n, int64_t nc, int mean_kind, double mean_c,
                                                const T* mean_v, T* out, int64_t ldo, int64_t n_pad, int64_t nc_pad, cudaStream_t s);
// p[i] *= v for i < n
template <typename T> void launch_scale(T* p, int64_t n, double v, cudaStream_t s);
// y[m] += sum_n A[m + n*lda] * x[n]   (rows coalesced)
template <typename T> void launch_gemv_n_acc(const T* A, int64_t lda, int64_t m, int64_t n, const T* x, T* y, cudaStream_t s);
// out[j] += sign * sum_i V[i + j*ldv]^2
template <typename T> void launch_colsumsq_acc(const T* V, int64_t ldv, int64_t n, int64_t m, double sign, T* out, cudaStream_t s);
// zero the strict upper triangle of every TILE x TILE diagonal block of an n_pad x n_pad factor
template <typename T> void launch_zero_diag_upper(T* A, int64_t lda, int64_t n_pad, cudaStream_t s);
// U(i,j) = L(map[j], map[i]) for i <= j (map == nullptr -> identity)
template <typename T> void launch_export_upper_map(const T* A, int64_t lda, int64_t n, const int64_t* map, T* U, int64_t ldo, cudaStream_t s);
template <typename T> void launch_copy2d(const T* src, int64_t lds, T* dst, int64_t ldd, int64_t rows,
                                         int64_t cols, cudaStream_t s);
// generic small helpers for VFE
template <typename T> void launch_scale_cols(T* B, int64_t ldb, int64_t rows, int64_t cols, const T* colscale,
                                             cudaStream_t s);  // B[:,j] *= colscale[j]
// EXPERIMENTAL (grad.cu): fused reduction of the logpdf gradient over the lower triangle; sums has 5 + D doubles (zeroed
// by the caller), noise_diag (n, optional) receives 1/2 W_ii
template <typename T> void launch_grad_reduce(const T* Xt, int D, int64_t n, int64_t n_pad, const T* Cinv, int64_t ldc,
                                              const T* alpha, int family, double linear_c, int want_ard, double* sums,
                                              T* noise_diag, cudaStream_t s);
// composite kernels (grad.cu): the same reduction for a sum of product terms over untransformed points; sums is indexed
// by the descriptor's gradient slots (zeroed by the caller) and holds sum_ij w_ij dK_ij/dtheta (times 1/2 by the caller),
// sums[3] = sum_i W_ii, sums[4] = sum_i alpha_i
template <typename T> void launch_composite_grad_reduce(const T* Xt, int D, int64_t n, int64_t n_pad, const T* Cinv, int64_t ldc,
                                                        const T* alpha, const CompositeDesc& cd, double* sums, T* noise_diag,
                                                        cudaStream_t s);
// input gradient (grad_x.cu): out (n x D values in `layout`, agp.h) = mult * chain_d * sum_j W_ij d1k(x_i, x_j)_d over the
// descriptor cd on the points X (n x D, point-major); chain_d = ard[d], or 1 when ard is null.  part: workspace of
// grad_x_part_len(n, D, cd.nacc) doubles (zeroed inside)
int64_t grad_x_part_len(int64_t n, int D, int nacc);
template <typename T> void launch_grad_x(const T* X, int D, int64_t n, const T* Cinv, int64_t ldc, const T* alpha,
                                         const CompositeDesc& cd, double mult, const T* ard, int layout, double* part,
                                         T* out, cudaStream_t s);
// test-point gradient of mean_and_var over a posterior (post_xs_grad.cu): out (m x D values in `layout`) = mult * chain_d *
// (sum_n Kbar_sx[j, n] d1k(x*_j, x_n)_d + 2 vbar_j d1k(x*_j, x*_j)_d), Kbar_sx[j, n] = mbar_j alpha_n - 2 vbar_j P[n + j*ldp],
// over the descriptor cd on the test points Xs (m x D) and the training points X (n x D), both point-major; mbar and vbar
// hold m values.  part: workspace of cross_grad_x_part_len(m, n, D, cd.nacc) doubles (zeroed inside)
int64_t cross_grad_x_part_len(int64_t m, int64_t n, int D, int nacc);
template <typename T> void launch_cross_grad_x(const T* Xs, int64_t m, const T* X, int64_t n, int D, const T* P, int64_t ldp,
                                               const T* alpha, const T* mbar, const T* vbar, const CompositeDesc& cd,
                                               double mult, const T* ard, int layout, double* part, T* out, cudaStream_t s);
// gradient of the VFE objectives (vfe_grad.cu).  H = c I - Lam^-1 - m_e m_e', E = c D - I + Lam^-1 + m_e m_e' (m_pad x m_pad,
// full, 0 outside M x M) from Lam^-1 (full), D = Lam - I (lower storage) and m_e
template <typename T> void launch_vfe_hz(const T* Laminv, const T* Dl, int64_t ldd, const T* me, int64_t M, int64_t m_pad,
                                         double c, T* H, T* E, cudaStream_t s);
// row blocks and the column ranges of the inducing-point partials for chunks of up to `cap` points
void vfe_cross_shape(int64_t m_pad, int64_t cap, int* nrb, int* nsplit);
// one chunk: hyper-parameter sums (grad_reduce units, 5 + D), column sums q / u (qpart / upart: nrb rows of ldq) and the
// inducing-point partials zpart (nsplit x D x m_pad, accumulated across chunks) from G = R K_zx,c (ldg) and r
template <typename T> void launch_vfe_cross_grad(const T* Zt, int64_t M, int64_t m_pad, const T* Xc, int64_t nc, int D,
                                                 const T* G, int64_t ldg, const T* r, const T* delta, const T* isn, int family,
                                                 double variance, double linear_c, int want_ard, int nsplit, double* sums,
                                                 double* qpart, double* upart, int64_t ldq, double* zpart, cudaStream_t s);
// one chunk: noise / mean adjoints per point, their sums nm[0..1], and the kdiag term of the hyper-parameter sums
template <typename T> void launch_vfe_point_grad(const double* qpart, const double* upart, int64_t ldq, int nrb, int64_t nc,
                                                 const T* delta, const T* isn, const T* kd, int noise_kind, double noise_s,
                                                 const T* noise_v, double c, const T* Xc, int D, int linear, double linear_c,
                                                 int want_ard, double* sums, double* nm, T* noise_diag, T* mean_diag,
                                                 cudaStream_t s);
// out (M x D in `layout`) = zz + mult * chain_d * sum_q zpart[q]  (chain_d = ard[d], or 1 when ard is null)
template <typename T> void launch_vfe_z_finish(const double* zpart, int nsplit, int64_t ldz, int64_t M, int D, double mult,
                                               const T* ard, int layout, const T* zz, T* out, cudaStream_t s);
// gradient of the VFE objectives with respect to the training inputs (vfe_grad_x.cu): the row ranges of the partials for
// chunks of up to `cap` points; one chunk's partials (nsplit x (D + 1) x ldx doubles, overwritten) from the same G and r
// as launch_vfe_cross_grad; then out (N x D in `layout`, rows c0 .. c0 + nc) from them (c = 1 elbo | 0 DTC)
void vfe_x_shape(int64_t m_pad, int64_t cap, int* nsplit);
template <typename T> void launch_vfe_x_grad(const T* Zt, int64_t M, int64_t m_pad, const T* Xc, int64_t nc, int D,
                                             const T* G, int64_t ldg, const T* r, const T* delta, const T* isn, int family,
                                             int nsplit, double* xpart, int64_t ldx, cudaStream_t s);
template <typename T> void launch_vfe_x_finish(const double* xpart, int nsplit, int64_t ldx, int64_t nc, int D, const T* Xc,
                                               const T* isn, int linear, double variance, double c, double mult,
                                               const T* ard, int layout, int64_t N, int64_t c0, T* out, cudaStream_t s);
// out[i] = (D)in[i]: the fp32 problems of the VFE gradient are converted to fp64 and back (vfe_grad.cu)
template <typename S, typename D> void launch_cast(const S* in, D* out, int64_t n, cudaStream_t s);
template <typename T> void launch_add_diag(T* A, int64_t lda, int64_t n, double v, cudaStream_t s);
// pullback of rand (rand_grad.cu): A(i, j) = A(j, i) for i < j < n (the strict lower triangle copied onto the upper one),
// and out[i] = sum_{s < S} A[i + s*lda] in fp64, in order
template <typename T> void launch_symmetrize_lower(T* A, int64_t lda, int64_t n, cudaStream_t s);
template <typename T> void launch_rowsum(const T* A, int64_t lda, int64_t n, int S, double* out, cudaStream_t s);
template <typename T> void launch_sumsq(const T* p, int64_t n, double* out, cudaStream_t s);  // out += sum p^2
template <typename T> void launch_vfe_prep(const T* y, int64_t n, int mean_kind, double mean_c, const T* mean_v,
                                           int noise_kind, double noise_s, const T* noise_v, const T* kdiag,
                                           T* delta, T* inv_sqrt_noise, double* scal /*[0]=logdet_sy [1]=sum d^2 [2]=tr*/,
                                           cudaStream_t s);

// true exactly once per (call site, current device): guards cudaFuncSetAttribute, which is a per-device setting
static inline bool agp_first_use_on_device(uint64_t* mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const uint64_t bit = 1ull << (dev & 63);
  if (*mask & bit) return false;
  *mask |= bit;
  return true;
}

int64_t agp_kernel_launches();
void agp_count_launch();  // global counter (all kernels above bump it)
