// solve.cu -- K6/K7/K8: blocked triangular solves with one right-hand side, reductions (sqmahal,
// logdet, column sums of squares), predictive-mean GEMV and small element-wise helpers.
// Replaces `C \ delta` (/root/reference/src/exact_gpr_posterior.jl:33), tr_At_A / diag_At_A
// (/root/reference/src/util/common_covmat_ops.jl:64-67), `C_xcond_x' * alpha`
// (/root/reference/src/exact_gpr_posterior.jl:87) and the logpdf assembly
// (/root/reference/src/finite_gp_projection.jl:309-310).  All HBM-bound: one coalesced pass over
// the data, warp-shuffle reductions, fp64 accumulation of every scalar.
#include "kernels.h"
#include "agp.h"

namespace {
constexpr int TB = AGP_TILE;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__global__ void border_init_kernel(T* __restrict__ A, int64_t lda, int64_t n, int64_t n_pad, const T* __restrict__ Y,
                                   int64_t ldy, int S, int mean_kind, T mean_c, const T* __restrict__ mean_v) {
  // one thread per (s, j), s fastest: each column's TILE border entries are contiguous in memory.
  int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= n_pad * TB) return;
  const int s = (int)(idx & (TB - 1));
  const int64_t j = idx >> 7;
  T v = 0;
  if (s < S && j < n) {
    T m = (mean_kind == 0) ? (T)0 : (mean_kind == 1 ? mean_c : mean_v[j]);
    v = Y[j + (int64_t)s * ldy] - m;
  }
  A[(n_pad + s) + j * lda] = v;
}

template <typename T>
__global__ void extract_v_kernel(const T* __restrict__ A, int64_t lda, int64_t n_pad, int S, T* __restrict__ r,
                                 double* __restrict__ sq) {
  // block s handles border row s
  const int s = blockIdx.x;
  double acc = 0.0;
  for (int64_t j = threadIdx.x; j < n_pad; j += blockDim.x) {
    T v = A[(n_pad + s) + j * lda];
    r[(int64_t)s * n_pad + j] = v;
    acc += (double)v * (double)v;
  }
  __shared__ double red[32];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    sq[s] = t;
  }
}

// 128-term column dot product split over a thread pair: thread (output o = tid>>1, half h = tid&1) streams
// 64 CONTIGUOUS elements of column o with independent loads (all in flight at once); the two halves meet
// through one shuffle in the caller.
template <typename T>
__device__ __forceinline__ double col_dot_half(const T* __restrict__ col, const T* __restrict__ vec_s, int h) {
  double acc0 = 0.0, acc1 = 0.0;
  const T* c = col + h * (TB / 2);
  const T* v = vec_s + h * (TB / 2);
#pragma unroll 16
  for (int j = 0; j < TB / 2; j += 2) {
    acc0 = fma((double)c[j], (double)v[j], acc0);
    acc1 = fma((double)c[j + 1], (double)v[j + 1], acc1);
  }
  return acc0 + acc1;
}

// ------------------------------------------------------------------------------------------------
// Persistent backward substitution  L' alpha = v  in ONE launch (replaces nblk dependent launches).
// CTA "b" (claimed through an atomic ticket so that producers always start before consumers) owns
// block b of the vector: it streams the tiles L(k, b), k = nblk-1 .. b+1, applying
// r_b -= L(k,b)' alpha_k as soon as CTA k publishes alpha_k (release/acquire flag in global memory),
// then computes alpha_b = inv(L_bb)' r_b from a copy of Dinv_b prefetched into shared memory at
// kernel start, and publishes it.  The tile for step k is loaded into registers BEFORE waiting on
// the flag, so the HBM/L2 latency of the factor is off the critical chain.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
template <typename T> struct Vec16;
template <> struct Vec16<double> { using type = double2; static constexpr int N = 2; };
template <> struct Vec16<float> { using type = float4; static constexpr int N = 4; };

template <typename T>
__device__ __forceinline__ void load_half_col(const T* __restrict__ col, T (&t)[TB / 2]) {
  using V = typename Vec16<T>::type;
  constexpr int VN = Vec16<T>::N;
  const V* p = reinterpret_cast<const V*>(col);
#pragma unroll
  for (int i = 0; i < TB / 2 / VN; ++i) {
    V v = __ldcg(p + i);
    const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
    for (int j = 0; j < VN; ++j) t[i * VN + j] = e[j];
  }
}

template <typename T>
__global__ void __launch_bounds__(256, 1) bwd_solve_kernel(const T* __restrict__ A, int64_t lda, const T* __restrict__ Dinv,
                                                            int nblk, T* r, int* flags, int* ticket) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sD = reinterpret_cast<T*>(smem_raw);  // Dinv_b, TB x TB col-major
  __shared__ T rb[TB];
  __shared__ T ak[TB];
  __shared__ int sb;
  const int tid = threadIdx.x, o = tid >> 1, h = tid & 1;
  if (tid == 0) sb = nblk - 1 - atomicAdd(ticket, 1);
  __syncthreads();
  const int b = sb;
  {  // prefetch Dinv_b -> smem (cp.async, 16 B per request)
    const T* Dk = Dinv + (int64_t)b * TB * TB;
    constexpr int VN = Vec16<T>::N;
    for (int q = tid; q < TB * TB / VN; q += 256) {
      unsigned sa = (unsigned)__cvta_generic_to_shared(sD + q * VN);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(Dk + q * VN));
    }
    asm volatile("cp.async.commit_group;" ::);
  }
  if (tid < TB) rb[tid] = __ldcg(r + (int64_t)b * TB + tid);
  for (int k = nblk - 1; k > b; --k) {
    T tile[TB / 2];
    load_half_col<T>(A + (int64_t)k * TB + ((int64_t)b * TB + o) * lda + h * (TB / 2), tile);
    if (tid == 0) {
      while (ld_acquire(flags + k) == 0) { }
    }
    __syncthreads();
    if (tid < TB) ak[tid] = __ldcg(r + (int64_t)k * TB + tid);
    __syncthreads();
    double a0 = 0.0, a1 = 0.0;
    const T* av = ak + h * (TB / 2);
#pragma unroll
    for (int j = 0; j < TB / 2; j += 2) {
      a0 = fma((double)tile[j], (double)av[j], a0);
      a1 = fma((double)tile[j + 1], (double)av[j + 1], a1);
    }
    double acc = a0 + a1;
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (h == 0) rb[o] -= (T)acc;
    // rb[o] is private to this thread pair; ak is rewritten only after the next barrier pair
  }
  asm volatile("cp.async.wait_group 0;" ::);
  __syncthreads();
  {  // alpha_b[o] = sum_j Dinv(j, o) r_b[j]
    double a0 = 0.0, a1 = 0.0;
    const T* col = sD + o * TB + h * (TB / 2);
    const T* rv = rb + h * (TB / 2);
#pragma unroll 16
    for (int j = 0; j < TB / 2; j += 2) {
      a0 = fma((double)col[j], (double)rv[j], a0);
      a1 = fma((double)col[j + 1], (double)rv[j + 1], a1);
    }
    double acc = a0 + a1;
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (h == 0) r[(int64_t)b * TB + o] = (T)acc;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) st_release(flags + b, 1);
}


template <typename T>
__global__ void border_init_cols_kernel(T* __restrict__ A, int64_t lda, int64_t row_off, int64_t col0, int64_t ncols,
                                        int64_t n, const T* __restrict__ Y, int64_t ldy, int S, int mean_kind, T mean_c,
                                        const T* __restrict__ mean_v) {
  int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= ncols * TB) return;
  const int s = (int)(idx & (TB - 1));
  const int64_t c = idx >> 7, j = col0 + c;
  T v = 0;
  if (s < S && j < n) {
    T m = (mean_kind == 0) ? (T)0 : (mean_kind == 1 ? mean_c : mean_v[j]);
    v = Y[j + (int64_t)s * ldy] - m;
  }
  A[(row_off + s) + c * lda] = v;
}

// distributed backward substitution pieces (column-cyclic factor): alpha_i = Dinv_i' r_i on the owner,
// then every rank applies r_j -= L(i,j)' alpha_i to its local column blocks j < i.
template <typename T>
__global__ void __launch_bounds__(256) bwd_diag_kernel(const T* __restrict__ Dinv_i, const T* __restrict__ r_i, T* __restrict__ alpha_i) {
  __shared__ T rk[TB];
  const int tid = threadIdx.x, o = tid >> 1, h = tid & 1;
  if (tid < TB) rk[tid] = r_i[tid];
  __syncthreads();
  double acc = col_dot_half<T>(Dinv_i + o * TB, rk, h);
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  if (h == 0) alpha_i[o] = (T)acc;
}
template <typename T>
__global__ void __launch_bounds__(256) bwd_update_local_kernel(const T* __restrict__ Lloc, int64_t lda, int i_blk,
                                                                const T* __restrict__ alpha_i, T* __restrict__ r,
                                                                int rank, int nranks, int G) {
  // CTA c handles local 128-column block lj = c; distribution blocks are G*128 columns wide:
  // global 128-block j = ((lj / G) * nranks + rank) * G + lj % G; only j < i is touched
  __shared__ T ak[TB];
  const int lj = blockIdx.x;
  const int64_t j = ((int64_t)(lj / G) * nranks + rank) * G + (lj % G);
  if (j >= i_blk) return;
  const int tid = threadIdx.x, o = tid >> 1, h = tid & 1;
  if (tid < TB) ak[tid] = alpha_i[tid];
  __syncthreads();
  const T* tile = Lloc + (int64_t)i_blk * TB + ((int64_t)lj * TB + o) * lda;
  double acc = col_dot_half<T>(tile, ak, h);
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  if (h == 0) r[j * TB + o] -= (T)acc;
}

// the same for a whole distribution block of G inner 128-blocks received in ONE broadcast: r_j -= sum_g L(i_lo+g, j)' alpha_{i_lo+g}
// for the local column blocks j < i_lo (a rank that does not own the block has no column inside it)
template <typename T>
__global__ void __launch_bounds__(256) bwd_update_local_multi_kernel(const T* __restrict__ Lloc, int64_t lda, int i_lo, int Gn,
                                                                      const T* __restrict__ alpha_lo, T* __restrict__ r,
                                                                      int rank, int nranks, int G, int64_t j_min, int64_t j_max) {
  __shared__ T ak[8 * TB];
  const int lj = blockIdx.x;
  const int64_t j = ((int64_t)(lj / G) * nranks + rank) * G + (lj % G);
  if (j >= i_lo || j < j_min || j >= j_max) return;
  const int tid = threadIdx.x, o = tid >> 1, h = tid & 1;
  for (int q = tid; q < Gn * TB; q += 256) ak[q] = alpha_lo[q];
  __syncthreads();
  double acc = 0.0;
  for (int g = 0; g < Gn; ++g) {
    const T* tile = Lloc + (int64_t)(i_lo + g) * TB + ((int64_t)lj * TB + o) * lda;
    acc += col_dot_half<T>(tile, ak + g * TB, h);
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  if (h == 0) r[j * TB + o] -= (T)acc;
}

template <typename T>
__global__ void finalize_logpdf_kernel(const double* __restrict__ logdet_part, int nblk, const double* __restrict__ sq,
                                       int S, int64_t n, T* __restrict__ out, double* __restrict__ logdet_out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double ld = 0.0;
    for (int b = 0; b < nblk; ++b) ld += logdet_part[b];
    ld *= 2.0;
    if (logdet_out) *logdet_out = ld;
    const double log2pi = 1.8378770664093454835606594728112;
    for (int s = 0; s < S; ++s) out[s] = (T)(-0.5 * ((double)n * log2pi + ld + sq[s]));
  }
}

template <typename T>
__global__ void gemv_t_kernel(const T* __restrict__ B, int64_t ldb, int64_t n, int64_t m, const T* __restrict__ alpha,
                              int mean_kind, T mean_c, const T* __restrict__ mean_v, T* __restrict__ mu) {
  const int64_t j = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= m) return;
  double acc = 0.0;
  const T* col = B + j * ldb;
  for (int64_t i = lane; i < n; i += 32) acc += (double)col[i] * (double)alpha[i];
  acc = warp_sum(acc);
  if (lane == 0) {
    T mj = (mean_kind == 0) ? (T)0 : (mean_kind == 1 ? mean_c : mean_v[j]);
    mu[j] = mj + (T)acc;
  }
}

template <typename T>
__global__ void colsumsq_var_kernel(const T* __restrict__ V, int64_t ldv, int64_t n, int64_t m, const T* __restrict__ kdiag,
                                    int noise_kind, T noise_s, const T* __restrict__ noise_v, T* __restrict__ var) {
  const int64_t j = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= m) return;
  double acc = 0.0;
  const T* col = V + j * ldv;
  for (int64_t i = lane; i < n; i += 32) { double v = (double)col[i]; acc += v * v; }
  acc = warp_sum(acc);
  if (lane == 0) {
    T v = kdiag[j] - (T)acc;
    if (noise_kind == 0) v += noise_s;
    else if (noise_kind == 1) v += noise_v[j];
    var[j] = v;
  }
}

template <typename T>
__global__ void export_upper_kernel(const T* __restrict__ A, int64_t lda, int64_t n, T* __restrict__ U, int64_t ldo) {
  // 32x32 smem transpose: U(i,j) = L(j,i) for i <= j
  __shared__ T tile[32][33];
  const int64_t bi = blockIdx.x * 32, bj = blockIdx.y * 32;  // output block rows bi.., cols bj..
  // read L(bj + y, bi + x) coalesced along rows of L (first index)
  for (int y = threadIdx.y; y < 32; y += 8) {
    int64_t lr = bj + threadIdx.x, lc = bi + y;  // L(lr, lc)
    T v = 0;
    if (lr < n && lc < n && lr >= lc) v = A[lr + lc * lda];
    tile[y][threadIdx.x] = v;  // tile[lc-bi][lr-bj]
  }
  __syncthreads();
  for (int y = threadIdx.y; y < 32; y += 8) {
    int64_t ui = bi + threadIdx.x, uj = bj + y;  // U(ui, uj) = L(uj, ui) = tile[ui-bi][uj-bj]
    if (ui < n && uj < n) U[ui + uj * ldo] = tile[threadIdx.x][y];
  }
}

template <typename T>
__global__ void add_mean_cols_kernel(T* __restrict__ out, int64_t ldo, int64_t n, int S, int mean_kind, T mean_c,
                                     const T* __restrict__ mean_v) {
  int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= n * S) return;
  int64_t s = idx / n, i = idx - s * n;
  T m = (mean_kind == 0) ? (T)0 : (mean_kind == 1 ? mean_c : mean_v[i]);
  out[i + s * ldo] += m;
}

template <typename T>
__global__ void cov_finish_kernel(T* __restrict__ C, int64_t ldc, const T* __restrict__ Kss, int64_t m) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t j = blockIdx.y;
  if (i >= m || j >= m) return;
  C[i + j * ldc] = Kss[i + j * ldc] - C[i + j * ldc];
}

template <typename T>
__global__ void fill_kernel(T* p, int64_t n, T v) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

template <typename T>
__global__ void copy2d_kernel(const T* __restrict__ src, int64_t lds, T* __restrict__ dst, int64_t ldd, int64_t rows,
                              int64_t cols) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t j = blockIdx.y;
  if (i < rows && j < cols) dst[i + j * ldd] = src[i + j * lds];
}

template <typename T>
__global__ void scale_cols_kernel(T* __restrict__ B, int64_t ldb, int64_t rows, int64_t cols, const T* __restrict__ cs) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t j = blockIdx.y;
  if (i < rows && j < cols) B[i + j * ldb] *= cs[j];
}

template <typename T>
__global__ void add_diag_kernel(T* A, int64_t lda, int64_t n, T v) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) A[i + i * lda] += v;
}

template <typename T>
__global__ void sumsq_kernel(const T* __restrict__ p, int64_t n, double* out) {
  double acc = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    double v = (double)p[i];
    acc += v * v;
  }
  acc = warp_sum(acc);
  __shared__ double red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    atomicAdd(out, t);
  }
}

// VFE prep (/root/reference/src/sparse_approximations.jl:296-300,307-313): delta = (y-m)/sqrt(s2),
// inv_sqrt_noise, logdet(Sigma_y), sum delta^2, tr(Cf Sigma_y^-1)
template <typename T>
__global__ void vfe_prep_kernel(const T* __restrict__ y, int64_t n, int mean_kind, T mean_c, const T* __restrict__ mean_v,
                                int noise_kind, T noise_s, const T* __restrict__ noise_v, const T* __restrict__ kdiag,
                                T* __restrict__ delta, T* __restrict__ isn, double* __restrict__ scal) {
  double a0 = 0, a1 = 0, a2 = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    T s2 = (noise_kind == 0) ? noise_s : noise_v[i];
    T m = (mean_kind == 0) ? (T)0 : (mean_kind == 1 ? mean_c : mean_v[i]);
    T is = (T)1 / (T)sqrt((double)s2);
    T d = (y[i] - m) * is;
    delta[i] = d;
    isn[i] = is;
    a0 += log((double)s2);
    a1 += (double)d * (double)d;
    a2 += (double)kdiag[i] / (double)s2;
  }
  a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
  if ((threadIdx.x & 31) == 0) { atomicAdd(scal + 0, a0); atomicAdd(scal + 1, a1); atomicAdd(scal + 2, a2); }
}

template <typename T>
__global__ void gemv_n_acc_kernel(const T* __restrict__ A, int64_t lda, int64_t m, int64_t n, const T* __restrict__ x,
                                  T* __restrict__ y) {
  // block handles 256 rows; grid.y splits the n range; partial sums accumulate with atomics (fp order
  // varies in the last bits only; the VFE scalars tolerate it and are documented as such)
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t per = (n + gridDim.y - 1) / gridDim.y;
  const int64_t n0 = blockIdx.y * per, n1 = (n0 + per < n) ? n0 + per : n;
  if (i >= m) return;
  double acc = 0.0;
  for (int64_t j = n0; j < n1; ++j) acc = fma((double)A[i + j * lda], (double)x[j], acc);
  atomicAdd(y + i, (T)acc);
}

template <typename T>
__global__ void colsumsq_acc_kernel(const T* __restrict__ V, int64_t ldv, int64_t n, int64_t m, T sign, T* __restrict__ out) {
  const int64_t j = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= m) return;
  double acc = 0.0;
  const T* col = V + j * ldv;
  for (int64_t i = lane; i < n; i += 32) { double v = (double)col[i]; acc += v * v; }
  acc = warp_sum(acc);
  if (lane == 0) out[j] += sign * (T)acc;
}

template <typename T>
__global__ void zero_diag_upper_kernel(T* __restrict__ A, int64_t lda) {
  const int64_t b = blockIdx.x;
  T* blk = A + b * TB + b * TB * lda;
  for (int idx = threadIdx.x; idx < TB * TB; idx += blockDim.x) {
    int c = idx >> 7, i = idx & 127;
    if (i < c) blk[i + (int64_t)c * lda] = (T)0;
  }
}

template <typename T>
__global__ void export_upper_map_kernel(const T* __restrict__ A, int64_t lda, int64_t n, const int64_t* __restrict__ map,
                                        T* __restrict__ U, int64_t ldo) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t j = blockIdx.y;
  if (i >= n || j >= n) return;
  T v = 0;
  if (i <= j) v = A[map[j] + map[i] * lda];
  U[i + j * ldo] = v;
}

template <typename T>
__global__ void sub_mean_kernel(const T* __restrict__ y, int64_t n, int mean_kind, T mean_c, const T* __restrict__ mean_v,
                                T* __restrict__ out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  T m = (mean_kind == 0) ? (T)0 : (mean_kind == 1 ? mean_c : mean_v[i]);
  out[i] = y[i] - m;
}

// one column block of Y - m, zero-padded to n_pad rows and gridDim.y columns (the multi-column logpdf gradient)
template <typename T>
__global__ void sub_mean_cols_kernel(const T* __restrict__ Y, int64_t ldy, int64_t n, int64_t nc, int mean_kind, T mean_c,
                                     const T* __restrict__ mean_v, T* __restrict__ out, int64_t ldo, int64_t n_pad) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t j = blockIdx.y;
  if (i >= n_pad) return;
  T v = (T)0;
  if (i < n && j < nc) v = Y[i + j * ldy] - ((mean_kind == 0) ? (T)0 : (mean_kind == 1 ? mean_c : mean_v[i]));
  out[i + j * ldo] = v;
}

template <typename T>
__global__ void scale_kernel(T* __restrict__ p, int64_t n, T v) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] *= v;
}
}  // namespace

template <typename T>
void launch_border_init(T* A, int64_t lda, int64_t n, int64_t n_pad, const T* Y, int64_t ldy, int S, int mean_kind,
                        double mean_c, const T* mean_v, cudaStream_t s) {
  border_init_kernel<T><<<(unsigned)((n_pad * TB + 255) / 256), 256, 0, s>>>(A, lda, n, n_pad, Y, ldy, S, mean_kind, (T)mean_c, mean_v);
  agp_count_launch();
}
template <typename T>
void launch_extract_v(const T* A, int64_t lda, int64_t n_pad, int S, T* r, double* sq, cudaStream_t s) {
  if (S <= 0) return;
  extract_v_kernel<T><<<S, 256, 0, s>>>(A, lda, n_pad, S, r, sq);
  agp_count_launch();
}
template <typename T>
void launch_bwd_solve(const T* A, int64_t lda, const T* Dinv, int nblk, T* r, int* flags_and_ticket, cudaStream_t s) {
  const size_t smem = (size_t)TB * TB * sizeof(T);
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  if (agp_first_use_on_device(&configured)) {
    cudaFuncSetAttribute(bwd_solve_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  cudaMemsetAsync(flags_and_ticket, 0, (size_t)(nblk + 1) * sizeof(int), s);
  bwd_solve_kernel<T><<<nblk, 256, smem, s>>>(A, lda, Dinv, nblk, r, flags_and_ticket, flags_and_ticket + nblk);
  agp_count_launch();
}
template <typename T>
void launch_finalize_logpdf(const double* logdet_part, int nblk, const double* sq, int S, int64_t n, T* out,
                            double* logdet_out, cudaStream_t s) {
  finalize_logpdf_kernel<T><<<1, 32, 0, s>>>(logdet_part, nblk, sq, S, n, out, logdet_out);
  agp_count_launch();
}
template <typename T>
void launch_gemv_t(const T* B, int64_t ldb, int64_t n, int64_t m, const T* alpha, int mean_kind, double mean_c,
                   const T* mean_v, T* mu, cudaStream_t s) {
  if (m <= 0) return;
  gemv_t_kernel<T><<<(unsigned)((m + 7) / 8), 256, 0, s>>>(B, ldb, n, m, alpha, mean_kind, (T)mean_c, mean_v, mu);
  agp_count_launch();
}
template <typename T>
void launch_colsumsq_var(const T* V, int64_t ldv, int64_t n, int64_t m, const T* kdiag, int noise_kind, double noise_s,
                         const T* noise_v, T* var, cudaStream_t s) {
  if (m <= 0) return;
  colsumsq_var_kernel<T><<<(unsigned)((m + 7) / 8), 256, 0, s>>>(V, ldv, n, m, kdiag, noise_kind, (T)noise_s, noise_v, var);
  agp_count_launch();
}
template <typename T>
void launch_export_upper(const T* A, int64_t lda, int64_t n, T* U, int64_t ldo, cudaStream_t s) {
  if (n <= 0) return;
  dim3 grid((unsigned)((n + 31) / 32), (unsigned)((n + 31) / 32));
  export_upper_kernel<T><<<grid, dim3(32, 8), 0, s>>>(A, lda, n, U, ldo);
  agp_count_launch();
}
template <typename T>
void launch_add_mean_cols(T* out, int64_t ldo, int64_t n, int S, int mean_kind, double mean_c, const T* mean_v,
                          cudaStream_t s) {
  if (mean_kind == 0 || n * S <= 0) return;
  add_mean_cols_kernel<T><<<(unsigned)((n * S + 255) / 256), 256, 0, s>>>(out, ldo, n, S, mean_kind, (T)mean_c, mean_v);
  agp_count_launch();
}
template <typename T>
void launch_cov_finish(T* C, int64_t ldc, const T* Kss, int64_t m, cudaStream_t s) {
  if (m <= 0) return;
  dim3 grid((unsigned)((m + 255) / 256), (unsigned)m);
  cov_finish_kernel<T><<<grid, 256, 0, s>>>(C, ldc, Kss, m);
  agp_count_launch();
}
template <typename T>
void launch_fill(T* p, int64_t n, double v, cudaStream_t s) {
  if (n <= 0) return;
  fill_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, n, (T)v);
  agp_count_launch();
}
template <typename T>
void launch_copy2d(const T* src, int64_t lds, T* dst, int64_t ldd, int64_t rows, int64_t cols, cudaStream_t s) {
  if (rows <= 0 || cols <= 0) return;
  dim3 grid((unsigned)((rows + 255) / 256), (unsigned)cols);
  copy2d_kernel<T><<<grid, 256, 0, s>>>(src, lds, dst, ldd, rows, cols);
  agp_count_launch();
}
template <typename T>
void launch_scale_cols(T* B, int64_t ldb, int64_t rows, int64_t cols, const T* cs, cudaStream_t s) {
  if (rows <= 0 || cols <= 0) return;
  dim3 grid((unsigned)((rows + 255) / 256), (unsigned)cols);
  scale_cols_kernel<T><<<grid, 256, 0, s>>>(B, ldb, rows, cols, cs);
  agp_count_launch();
}
template <typename T>
void launch_add_diag(T* A, int64_t lda, int64_t n, double v, cudaStream_t s) {
  if (n <= 0) return;
  add_diag_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(A, lda, n, (T)v);
  agp_count_launch();
}
template <typename T>
void launch_sumsq(const T* p, int64_t n, double* out, cudaStream_t s) {
  if (n <= 0) return;
  int blocks = (int)((n + 1023) / 1024);
  if (blocks > 592) blocks = 592;
  sumsq_kernel<T><<<blocks, 256, 0, s>>>(p, n, out);
  agp_count_launch();
}
template <typename T>
void launch_vfe_prep(const T* y, int64_t n, int mean_kind, double mean_c, const T* mean_v, int noise_kind, double noise_s,
                     const T* noise_v, const T* kdiag, T* delta, T* isn, double* scal, cudaStream_t s) {
  if (n <= 0) return;
  int blocks = (int)((n + 1023) / 1024);
  if (blocks > 592) blocks = 592;
  vfe_prep_kernel<T><<<blocks, 256, 0, s>>>(y, n, mean_kind, (T)mean_c, mean_v, noise_kind, (T)noise_s, noise_v, kdiag, delta, isn, scal);
  agp_count_launch();
}

template <typename T>
void launch_gemv_n_acc(const T* A, int64_t lda, int64_t m, int64_t n, const T* x, T* y, cudaStream_t s) {
  if (m <= 0 || n <= 0) return;
  int ysplit = (int)((n + 2047) / 2048);
  if (ysplit > 64) ysplit = 64;
  dim3 grid((unsigned)((m + 255) / 256), (unsigned)ysplit);
  gemv_n_acc_kernel<T><<<grid, 256, 0, s>>>(A, lda, m, n, x, y);
  agp_count_launch();
}
template <typename T>
void launch_colsumsq_acc(const T* V, int64_t ldv, int64_t n, int64_t m, double sign, T* out, cudaStream_t s) {
  if (m <= 0) return;
  colsumsq_acc_kernel<T><<<(unsigned)((m + 7) / 8), 256, 0, s>>>(V, ldv, n, m, (T)sign, out);
  agp_count_launch();
}
template <typename T>
void launch_zero_diag_upper(T* A, int64_t lda, int64_t n_pad, cudaStream_t s) {
  if (n_pad <= 0) return;
  zero_diag_upper_kernel<T><<<(unsigned)(n_pad / TB), 256, 0, s>>>(A, lda);
  agp_count_launch();
}
template <typename T>
void launch_export_upper_map(const T* A, int64_t lda, int64_t n, const int64_t* map, T* U, int64_t ldo, cudaStream_t s) {
  if (n <= 0) return;
  dim3 grid((unsigned)((n + 255) / 256), (unsigned)n);
  export_upper_map_kernel<T><<<grid, 256, 0, s>>>(A, lda, n, map, U, ldo);
  agp_count_launch();
}

template <typename T>
void launch_sub_mean(const T* y, int64_t n, int mean_kind, double mean_c, const T* mean_v, T* out, cudaStream_t s) {
  if (n <= 0) return;
  sub_mean_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(y, n, mean_kind, (T)mean_c, mean_v, out);
  agp_count_launch();
}
template <typename T>
void launch_sub_mean_cols(const T* Y, int64_t ldy, int64_t n, int64_t nc, int mean_kind, double mean_c, const T* mean_v, T* out,
                          int64_t ldo, int64_t n_pad, int64_t nc_pad, cudaStream_t s) {
  if (n_pad <= 0 || nc_pad <= 0) return;
  dim3 grid((unsigned)((n_pad + 255) / 256), (unsigned)nc_pad);
  sub_mean_cols_kernel<T><<<grid, 256, 0, s>>>(Y, ldy, n, nc, mean_kind, (T)mean_c, mean_v, out, ldo, n_pad);
  agp_count_launch();
}
template <typename T>
void launch_scale(T* p, int64_t n, double v, cudaStream_t s) {
  if (n <= 0) return;
  scale_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, n, (T)v);
  agp_count_launch();
}

template <typename T>
void launch_border_init_cols(T* A, int64_t lda, int64_t row_off, int64_t col0, int64_t ncols, int64_t n, const T* Y,
                             int64_t ldy, int S, int mean_kind, double mean_c, const T* mean_v, cudaStream_t s) {
  if (ncols <= 0) return;
  border_init_cols_kernel<T><<<(unsigned)((ncols * TB + 255) / 256), 256, 0, s>>>(A, lda, row_off, col0, ncols, n, Y, ldy, S,
                                                                                  mean_kind, (T)mean_c, mean_v);
  agp_count_launch();
}
template <typename T>
void launch_bwd_diag(const T* Dinv_i, const T* r_i, T* alpha_i, cudaStream_t s) {
  bwd_diag_kernel<T><<<1, 256, 0, s>>>(Dinv_i, r_i, alpha_i);
  agp_count_launch();
}
template <typename T>
void launch_bwd_update_local(const T* Lloc, int64_t lda, int i_blk, const T* alpha_i, T* r, int nloc, int rank, int nranks,
                             int G, cudaStream_t s) {
  if (nloc <= 0) return;
  bwd_update_local_kernel<T><<<nloc, 256, 0, s>>>(Lloc, lda, i_blk, alpha_i, r, rank, nranks, G);
  agp_count_launch();
}
template <typename T>
void launch_bwd_update_local_multi(const T* Lloc, int64_t lda, int i_lo, int Gn, const T* alpha_lo, T* r, int nloc, int rank,
                                   int nranks, int G, int64_t j_min, int64_t j_max, cudaStream_t s) {
  if (nloc <= 0 || Gn <= 0 || j_max <= j_min) return;
  bwd_update_local_multi_kernel<T><<<nloc, 256, 0, s>>>(Lloc, lda, i_lo, Gn, alpha_lo, r, rank, nranks, G, j_min, j_max);
  agp_count_launch();
}
template void launch_bwd_update_local_multi<float>(const float*, int64_t, int, int, const float*, float*, int, int, int, int, int64_t, int64_t, cudaStream_t);
template void launch_bwd_update_local_multi<double>(const double*, int64_t, int, int, const double*, double*, int, int, int, int, int64_t, int64_t, cudaStream_t);

// one outer block of the distributed backward substitution resolved by ONE CTA on its owner: for g = Gn-1 .. 0
//   alpha_g = inv(L_gg)' r_g,   r_g' -= L(g, g')' alpha_g  (g' < g)
// Lblk points at the block's diagonal element in the owner's local storage; r_blk / alpha_blk are its Gn*128 entries.
template <typename T>
__global__ void __launch_bounds__(256) bwd_block_solve_kernel(const T* __restrict__ Lblk, int64_t lda, const T* __restrict__ Dinv_blk,
                                                               const T* __restrict__ r_blk, T* __restrict__ alpha_blk, int Gn) {
  __shared__ T rs[8 * TB];
  __shared__ T as[TB];
  const int tid = threadIdx.x, o = tid >> 1, h = tid & 1;
  for (int q = tid; q < Gn * TB; q += 256) rs[q] = r_blk[q];
  __syncthreads();
  for (int g = Gn - 1; g >= 0; --g) {
    double acc = col_dot_half<T>(Dinv_blk + (int64_t)g * TB * TB + o * TB, rs + g * TB, h);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (h == 0) { as[o] = (T)acc; alpha_blk[g * TB + o] = (T)acc; }
    __syncthreads();
    for (int gp = 0; gp < g; ++gp) {
      const T* tile = Lblk + (int64_t)g * TB + ((int64_t)gp * TB + o) * lda;
      double a2 = col_dot_half<T>(tile, as, h);
      a2 += __shfl_xor_sync(0xffffffffu, a2, 1);
      if (h == 0) rs[gp * TB + o] -= (T)a2;
    }
    __syncthreads();
  }
}
template <typename T>
void launch_bwd_block_solve(const T* Lblk, int64_t lda, const T* Dinv_blk, const T* r_blk, T* alpha_blk, int Gn, cudaStream_t s) {
  bwd_block_solve_kernel<T><<<1, 256, 0, s>>>(Lblk, lda, Dinv_blk, r_blk, alpha_blk, Gn);
  agp_count_launch();
}
template void launch_bwd_block_solve<float>(const float*, int64_t, const float*, const float*, float*, int, cudaStream_t);
template void launch_bwd_block_solve<double>(const double*, int64_t, const double*, const double*, double*, int, cudaStream_t);

// explicit instantiations
template void launch_border_init_cols<float>(float*, int64_t, int64_t, int64_t, int64_t, int64_t, const float*, int64_t, int, int, double, const float*, cudaStream_t);
template void launch_bwd_diag<float>(const float*, const float*, float*, cudaStream_t);
template void launch_bwd_update_local<float>(const float*, int64_t, int, const float*, float*, int, int, int, int, cudaStream_t);
template void launch_border_init_cols<double>(double*, int64_t, int64_t, int64_t, int64_t, int64_t, const double*, int64_t, int, int, double, const double*, cudaStream_t);
template void launch_bwd_diag<double>(const double*, const double*, double*, cudaStream_t);
template void launch_bwd_update_local<double>(const double*, int64_t, int, const double*, double*, int, int, int, int, cudaStream_t);
template void launch_sub_mean<float>(const float*, int64_t, int, double, const float*, float*, cudaStream_t);
template void launch_sub_mean<double>(const double*, int64_t, int, double, const double*, double*, cudaStream_t);
template void launch_sub_mean_cols<float>(const float*, int64_t, int64_t, int64_t, int, double, const float*, float*, int64_t,
                                          int64_t, int64_t, cudaStream_t);
template void launch_sub_mean_cols<double>(const double*, int64_t, int64_t, int64_t, int, double, const double*, double*, int64_t,
                                           int64_t, int64_t, cudaStream_t);
template void launch_scale<float>(float*, int64_t, double, cudaStream_t);
template void launch_scale<double>(double*, int64_t, double, cudaStream_t);
template void launch_gemv_n_acc<float>(const float*, int64_t, int64_t, int64_t, const float*, float*, cudaStream_t);
template void launch_colsumsq_acc<float>(const float*, int64_t, int64_t, int64_t, double, float*, cudaStream_t);
template void launch_zero_diag_upper<float>(float*, int64_t, int64_t, cudaStream_t);
template void launch_export_upper_map<float>(const float*, int64_t, int64_t, const int64_t*, float*, int64_t, cudaStream_t);
template void launch_gemv_n_acc<double>(const double*, int64_t, int64_t, int64_t, const double*, double*, cudaStream_t);
template void launch_colsumsq_acc<double>(const double*, int64_t, int64_t, int64_t, double, double*, cudaStream_t);
template void launch_zero_diag_upper<double>(double*, int64_t, int64_t, cudaStream_t);
template void launch_export_upper_map<double>(const double*, int64_t, int64_t, const int64_t*, double*, int64_t, cudaStream_t);
template void launch_bwd_solve<float>(const float*, int64_t, const float*, int, float*, int*, cudaStream_t);
template void launch_bwd_solve<double>(const double*, int64_t, const double*, int, double*, int*, cudaStream_t);
template void launch_border_init<float>(float*, int64_t, int64_t, int64_t, const float*, int64_t, int, int, double, const float*, cudaStream_t);
template void launch_extract_v<float>(const float*, int64_t, int64_t, int, float*, double*, cudaStream_t);
template void launch_finalize_logpdf<float>(const double*, int, const double*, int, int64_t, float*, double*, cudaStream_t);
template void launch_gemv_t<float>(const float*, int64_t, int64_t, int64_t, const float*, int, double, const float*, float*, cudaStream_t);
template void launch_colsumsq_var<float>(const float*, int64_t, int64_t, int64_t, const float*, int, double, const float*, float*, cudaStream_t);
template void launch_export_upper<float>(const float*, int64_t, int64_t, float*, int64_t, cudaStream_t);
template void launch_add_mean_cols<float>(float*, int64_t, int64_t, int, int, double, const float*, cudaStream_t);
template void launch_cov_finish<float>(float*, int64_t, const float*, int64_t, cudaStream_t);
template void launch_fill<float>(float*, int64_t, double, cudaStream_t);
template void launch_copy2d<float>(const float*, int64_t, float*, int64_t, int64_t, int64_t, cudaStream_t);
template void launch_scale_cols<float>(float*, int64_t, int64_t, int64_t, const float*, cudaStream_t);
template void launch_add_diag<float>(float*, int64_t, int64_t, double, cudaStream_t);
template void launch_sumsq<float>(const float*, int64_t, double*, cudaStream_t);
template void launch_vfe_prep<float>(const float*, int64_t, int, double, const float*, int, double, const float*, const float*, float*, float*, double*, cudaStream_t);
template void launch_border_init<double>(double*, int64_t, int64_t, int64_t, const double*, int64_t, int, int, double, const double*, cudaStream_t);
template void launch_extract_v<double>(const double*, int64_t, int64_t, int, double*, double*, cudaStream_t);
template void launch_finalize_logpdf<double>(const double*, int, const double*, int, int64_t, double*, double*, cudaStream_t);
template void launch_gemv_t<double>(const double*, int64_t, int64_t, int64_t, const double*, int, double, const double*, double*, cudaStream_t);
template void launch_colsumsq_var<double>(const double*, int64_t, int64_t, int64_t, const double*, int, double, const double*, double*, cudaStream_t);
template void launch_export_upper<double>(const double*, int64_t, int64_t, double*, int64_t, cudaStream_t);
template void launch_add_mean_cols<double>(double*, int64_t, int64_t, int, int, double, const double*, cudaStream_t);
template void launch_cov_finish<double>(double*, int64_t, const double*, int64_t, cudaStream_t);
template void launch_fill<double>(double*, int64_t, double, cudaStream_t);
template void launch_copy2d<double>(const double*, int64_t, double*, int64_t, int64_t, int64_t, cudaStream_t);
template void launch_scale_cols<double>(double*, int64_t, int64_t, int64_t, const double*, cudaStream_t);
template void launch_add_diag<double>(double*, int64_t, int64_t, double, cudaStream_t);
template void launch_sumsq<double>(const double*, int64_t, double*, cudaStream_t);
template void launch_vfe_prep<double>(const double*, int64_t, int, double, const double*, int, double, const double*, const double*, double*, double*, double*, cudaStream_t);
