// gemm.cu -- K4/K5 (legacy-tensor path): the tile GEMM behind TRSM-as-GEMM (A21 <- A21 * inv(L11)'),
// the trailing SYRK (A22 -= L21 L21'), the blocked multi-RHS forward substitution of the prediction
// path, and TRMM for rand.  Replaces the LAPACK potrf trailing update / trsm inside
// cholesky(.) and `C.U' \ X` (/root/reference/src/finite_gp_projection.jl:308,
// /root/reference/src/util/common_covmat_ops.jl:54,90,101).
//
// fp64: 128x128x16 CTA tile, 3-stage cp.async pipeline, 8 warps x (64x32) warp tiles of
//       mma.sync.m8n8k4.f64 (DMMA) -- padded smem strides make every fragment load conflict-free.
// fp32: 128x128x16 CTA tile, register-prefetch double buffering, 8x8 FFMA micro-tiles.
// The int8-slice wgmma kernel (umma_ozaki.cu) replaces these on the trailing update when enabled.
#include "kernels.h"
#include "agp.h"

namespace {

constexpr int BM = 128, BN = 128, BK = 16;

// ------------------------------------------------------------------------------------------------
// fp64 DMMA kernel.  CTA tile 128 x (32*WN); WN = 2 -> 128x64 tile, 128 threads, 2 CTAs/SM so one
// CTA's read-modify-write epilogue overlaps the other's main loop; WN = 4 -> 128x128, 256 threads
// (used for the in-place panel TRSM, which needs one CTA to own all 128 columns of its rows).
// ------------------------------------------------------------------------------------------------
constexpr int D_STAGES = 3;
constexpr int D_LDK = BK + 4;  // K-major smem stride (doubles): 20 -> row shift of 8 banks
__host__ __device__ constexpr int d_opsz(int rows) { return (rows * D_LDK > BK * (rows + 4)) ? rows * D_LDK : BK * (rows + 4); }

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// element (mn, k) of a ROWS x 16 operand slab starting at (mn0, k0); MN-major smem stride ROWS+4
template <bool KMAJOR, int ROWS, int NT>
__device__ __forceinline__ void d_load_tile(double* s, const double* __restrict__ g, int64_t ld, int64_t mn0,
                                            int64_t k0, int64_t MN, int64_t K, int tid) {
  constexpr int CHUNKS = ROWS * 8;  // 16-byte chunks in the slab
#pragma unroll
  for (int it = 0; it < CHUNKS / NT; ++it) {
    const int q = tid + NT * it;
    if (!KMAJOR) {
      const int k = q / (ROWS / 2), mn = (q % (ROWS / 2)) * 2;
      const bool valid = (mn0 + mn < MN) && (k0 + k < K);
      const double* src = valid ? (g + (mn0 + mn) + (k0 + k) * ld) : g;
      cp_async16(s + k * (ROWS + 4) + mn, src, valid);
    } else {
      const int mn = q >> 3, k = (q & 7) * 2;
      const bool valid = (mn0 + mn < MN) && (k0 + k < K);
      const double* src = valid ? (g + (k0 + k) + (mn0 + mn) * ld) : g;
      cp_async16(s + mn * D_LDK + k, src, valid);
    }
  }
}

__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

template <bool AK, bool BKM, int WM, int WN>
__global__ void __launch_bounds__(32 * WM * WN, (WM * WN <= 4) ? 2 : 1) gemm_dmma_kernel(GemmArgs g) {
  constexpr int NT = 32 * WM * WN, TBM = 64 * WM, TBN = 32 * WN;
  constexpr int A_SZ = d_opsz(TBM), B_SZ = d_opsz(TBN);
  constexpr int A_LD = TBM + 4, B_LD = TBN + 4;
  const int bi = blockIdx.x, bj = blockIdx.y;
  const int64_t m0 = (int64_t)bi * TBM, n0 = (int64_t)bj * TBN;
  const int64_t bw = g.b_tile_width ? g.b_tile_width : 128;
  const int64_t n_src0 = g.b_tile_stride ? (n0 / bw) * g.b_tile_stride + (n0 % bw) + g.b_off : n0;
  if (g.lower_only && n_src0 >= m0 + TBM) return;  // tile entirely above the diagonal
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sm = reinterpret_cast<double*>(smem_raw);
  double* sA = sm;                    // [D_STAGES][A_SZ]
  double* sB = sm + D_STAGES * A_SZ;  // [D_STAGES][B_SZ]
  const double* __restrict__ A = (const double*)g.A;
  const double* __restrict__ B = (const double*)g.B + (BKM ? (n_src0 - n0) * g.ldb : (n_src0 - n0));
  double* C = (double*)g.C;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp % WM, wn = warp / WM;
  const int gq = lane >> 2, q = lane & 3;
  int64_t K = g.K;
  if (g.trmm_lower) { int64_t kl = m0 + TBM; if (kl < K) K = kl; }
  const int KT = (int)((K + BK - 1) / BK);

  double acc[8][4][2];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

#pragma unroll
  for (int s = 0; s < D_STAGES - 1; ++s) {
    if (s < KT) {
      d_load_tile<AK, TBM, NT>(sA + s * A_SZ, A, g.lda, m0, (int64_t)s * BK, g.M, K, tid);
      d_load_tile<BKM, TBN, NT>(sB + s * B_SZ, B, g.ldb, n0, (int64_t)s * BK, g.N, K, tid);
    }
    cp_async_commit();
  }
  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<D_STAGES - 2>();
    __syncthreads();
    {
      const int nk = kt + D_STAGES - 1;
      if (nk < KT) {
        const int st = nk % D_STAGES;
        d_load_tile<AK, TBM, NT>(sA + st * A_SZ, A, g.lda, m0, (int64_t)nk * BK, g.M, K, tid);
        d_load_tile<BKM, TBN, NT>(sB + st * B_SZ, B, g.ldb, n0, (int64_t)nk * BK, g.N, K, tid);
      }
      cp_async_commit();
    }
    const double* a_s = sA + (kt % D_STAGES) * A_SZ;
    const double* b_s = sB + (kt % D_STAGES) * B_SZ;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 4) {
      double af[8], bf[4];
#pragma unroll
      for (int mi = 0; mi < 8; ++mi) {
        const int m = wm * 64 + mi * 8 + gq;
        af[mi] = AK ? a_s[m * D_LDK + kk + q] : a_s[(kk + q) * A_LD + m];
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const int n = wn * 32 + ni * 8 + gq;
        bf[ni] = BKM ? b_s[n * D_LDK + kk + q] : b_s[(kk + q) * B_LD + n];
      }
#pragma unroll
      for (int mi = 0; mi < 8; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) dmma(acc[mi][ni][0], acc[mi][ni][1], af[mi], bf[ni]);
    }
  }
  cp_async_wait<0>();

  // epilogue: C(m, n); a thread holds rows gq, cols 2q, 2q+1 of each 8x8 tile.  The C reads of row
  // group mi+1 are issued before the stores of group mi so the round trips overlap.
  const int64_t mbase = m0 + wm * 64 + gq;
  const int64_t nbase = n0 + wn * 32 + 2 * q;
  const bool beta = g.beta_one != 0;
  const double sgn = g.alpha_neg ? -1.0 : 1.0;
  double cv[2][8];
  auto load_group = [&](int mi, double* dst) {
    const int64_t m = mbase + mi * 8;
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t n = nbase + ni * 8 + e;
        dst[ni * 2 + e] = (beta && m < g.M && n < g.N) ? C[m + n * g.ldc] : 0.0;
      }
  };
  load_group(0, cv[0]);
#pragma unroll
  for (int mi = 0; mi < 8; ++mi) {
    if (mi + 1 < 8) load_group(mi + 1, cv[(mi + 1) & 1]);
    const int64_t m = mbase + mi * 8;
    if (m < g.M) {
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int64_t n = nbase + ni * 8 + e;
          if (n < g.N) C[m + n * g.ldc] = fma(sgn, acc[mi][ni][e], cv[mi & 1][ni * 2 + e]);
        }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// fp32 SIMT kernel
// ------------------------------------------------------------------------------------------------
constexpr int S_LD = BM + 4;

template <bool KMAJOR>
__device__ __forceinline__ void s_fetch(float4 (&r)[2], const float* __restrict__ g, int64_t ld, int64_t mn0,
                                        int64_t k0, int64_t MN, int64_t K, int tid) {
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    int qd = tid + 256 * it;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!KMAJOR) {
      int k = qd >> 5, mn = (qd & 31) * 4;
      if (mn0 + mn < MN && k0 + k < K) v = *reinterpret_cast<const float4*>(g + (mn0 + mn) + (k0 + k) * ld);
    } else {
      int mn = qd >> 2, k = (qd & 3) * 4;
      if (mn0 + mn < MN && k0 + k < K) v = *reinterpret_cast<const float4*>(g + (k0 + k) + (mn0 + mn) * ld);
    }
    r[it] = v;
  }
}
template <bool KMAJOR>
__device__ __forceinline__ void s_stash(float* s, const float4 (&r)[2], int tid) {
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    int qd = tid + 256 * it;
    if (!KMAJOR) {
      int k = qd >> 5, mn = (qd & 31) * 4;
      *reinterpret_cast<float4*>(s + k * S_LD + mn) = r[it];
    } else {
      int mn = qd >> 2, k = (qd & 3) * 4;
      s[(k + 0) * S_LD + mn] = r[it].x;
      s[(k + 1) * S_LD + mn] = r[it].y;
      s[(k + 2) * S_LD + mn] = r[it].z;
      s[(k + 3) * S_LD + mn] = r[it].w;
    }
  }
}

template <bool AK, bool BKM>
__global__ void __launch_bounds__(256, 2) gemm_simt_kernel(GemmArgs g) {
  const int bi = blockIdx.x, bj = blockIdx.y;
  __shared__ __align__(16) float sA[2][BK * S_LD];
  __shared__ __align__(16) float sB[2][BK * S_LD];
  const float* __restrict__ A = (const float*)g.A;
  const float* B = (const float*)g.B;
  float* __restrict__ C = (float*)g.C;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)bi * BM, n0 = (int64_t)bj * BN;
  const int64_t bw = g.b_tile_width ? g.b_tile_width : 128;
  const int64_t n_src0 = g.b_tile_stride ? (n0 / bw) * g.b_tile_stride + (n0 % bw) + g.b_off : n0;
  if (g.lower_only && n_src0 >= m0 + BM) return;
  B += (BKM ? (n_src0 - n0) * g.ldb : (n_src0 - n0));
  int64_t K = g.K;
  if (g.trmm_lower) { int64_t kl = m0 + BM; if (kl < K) K = kl; }
  const int KT = (int)((K + BK - 1) / BK);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float4 ra[2], rb[2];
  if (KT > 0) {
    s_fetch<AK>(ra, A, g.lda, m0, 0, g.M, K, tid);
    s_fetch<BKM>(rb, B, g.ldb, n0, 0, g.N, K, tid);
    s_stash<AK>(sA[0], ra, tid);
    s_stash<BKM>(sB[0], rb, tid);
  }
  __syncthreads();
  for (int kt = 0; kt < KT; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < KT) {
      s_fetch<AK>(ra, A, g.lda, m0, (int64_t)(kt + 1) * BK, g.M, K, tid);
      s_fetch<BKM>(rb, B, g.ldb, n0, (int64_t)(kt + 1) * BK, g.N, K, tid);
    }
    const float* a_s = sA[cur];
    const float* b_s = sB[cur];
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 a0 = *reinterpret_cast<const float4*>(a_s + k * S_LD + tx * 4);
      float4 a1 = *reinterpret_cast<const float4*>(a_s + k * S_LD + 64 + tx * 4);
      float4 b0 = *reinterpret_cast<const float4*>(b_s + k * S_LD + ty * 4);
      float4 b1 = *reinterpret_cast<const float4*>(b_s + k * S_LD + 64 + ty * 4);
      float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < KT) {
      s_stash<AK>(sA[cur ^ 1], ra, tid);
      s_stash<BKM>(sB[cur ^ 1], rb, tid);
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int64_t n = n0 + (j < 4 ? ty * 4 + j : 64 + ty * 4 + (j - 4));
    if (n >= g.N) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t m = m0 + h * 64 + tx * 4;
      if (m >= g.M) continue;  // M is a multiple of 4
      float4* p = reinterpret_cast<float4*>(C + m + n * g.ldc);
      float4 v = make_float4(acc[h * 4 + 0][j], acc[h * 4 + 1][j], acc[h * 4 + 2][j], acc[h * 4 + 3][j]);
      if (g.alpha_neg) { v.x = -v.x; v.y = -v.y; v.z = -v.z; v.w = -v.w; }
      if (g.beta_one) { float4 c = *p; v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w; }
      *p = v;
    }
  }
}

template <typename KernelT>
void launch_cfg(KernelT kern, const GemmArgs& g, size_t smem, cudaStream_t s) {
  dim3 grid((unsigned)((g.M + BM - 1) / BM), (unsigned)((g.N + BN - 1) / BN));
  kern<<<grid, 256, smem, s>>>(g);
  agp_count_launch();
}
}  // namespace

template <bool AK, bool BKM, int WM, int WN>
static void launch_dmma(const GemmArgs& g, cudaStream_t s) {
  constexpr int TBM = 64 * WM, TBN = 32 * WN;
  const size_t smem = (size_t)D_STAGES * (d_opsz(TBM) + d_opsz(TBN)) * sizeof(double);
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  if (agp_first_use_on_device(&configured)) {
    cudaFuncSetAttribute(gemm_dmma_kernel<AK, BKM, WM, WN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  dim3 grid((unsigned)((g.M + TBM - 1) / TBM), (unsigned)((g.N + TBN - 1) / TBN));
  gemm_dmma_kernel<AK, BKM, WM, WN><<<grid, 32 * WM * WN, smem, s>>>(g);
  agp_count_launch();
}

// The operand contract of GemmArgs (kernels.h) for the instantiation a product selects; tbn is its column-tile width.
template <typename T>
static bool gemm_contract_ok(const GemmArgs& g, int64_t tbn) {
  constexpr int64_t V = 16 / sizeof(T);  // elements per 16-byte load
  auto aligned = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
  if (g.K < 0 || !aligned(g.A) || !aligned(g.B) || g.lda % V || g.ldb % V) return false;
  if (sizeof(T) == 4 && (!aligned(g.C) || g.ldc % V || g.M % V)) return false;  // float4 epilogue
  if ((g.a_kmajor || g.b_kmajor) && g.K % V) return false;  // a K-major load reads k .. k + V - 1 and checks only k
  const int64_t bw = g.b_tile_width ? g.b_tile_width : 128;
  int64_t n_hi = g.N - 1;  // highest B column read
  if (g.b_tile_stride) {
    if (g.b_tile_stride < 0 || g.b_tile_width < 0 || g.b_off < 0 || bw % tbn) return false;
    if (!g.b_kmajor && ((g.b_tile_stride - bw) % V || g.b_off % V)) return false;  // the shift keeps B's loads aligned
    const int64_t blk = n_hi / bw;
    n_hi = blk * g.b_tile_stride + n_hi % bw;
    if (blk > 0 && (blk - 1) * g.b_tile_stride + bw - 1 > n_hi) n_hi = (blk - 1) * g.b_tile_stride + bw - 1;
    n_hi += g.b_off;
  }
  if (g.lda < (g.a_kmajor ? g.K : g.M) || g.ldb < (g.b_kmajor ? g.K : n_hi + 1) || g.ldc < g.M) return false;
  // in place: one CTA owns every row (C == A) or column (C == B) it reads, and reads them all before it writes
  if (g.C == g.A && (g.a_kmajor || g.ldc != g.lda || g.N > 128)) return false;
  if (g.C == g.B && (!g.b_kmajor || g.ldc != g.ldb || g.M > 128 || g.b_tile_stride)) return false;
  return true;
}

template <>
int launch_gemm<double>(const GemmArgs& g, cudaStream_t s) {
  if (g.M <= 0 || g.N <= 0) return 0;
  if (!gemm_contract_ok<double>(g, (g.C == g.A || g.C == g.B) ? 128 : 64)) return 1;
  // in-place products (C aliases an operand) need one CTA to own every column it reads: 128-wide tile.
  // C == A (panel TRSM): 64 x 128 tiles, 2 CTAs/SM -- twice the CTAs on the latency-critical panel solve.
  // The contract leaves A MN-major when C == A and B K-major when C == B.
  if (g.C == g.A) {
    if (!g.b_kmajor) launch_dmma<false, false, 1, 4>(g, s);
    else launch_dmma<false, true, 1, 4>(g, s);
  } else if (g.C == g.B) {
    if (!g.a_kmajor) launch_dmma<false, true, 2, 4>(g, s);
    else launch_dmma<true, true, 2, 4>(g, s);
  } else {  // (64x64 tiles for the narrow next-column update were measured: 21 us vs 19 us for 128x64 -- not kept)
    if (!g.a_kmajor && !g.b_kmajor) launch_dmma<false, false, 2, 2>(g, s);
    else if (!g.a_kmajor && g.b_kmajor) launch_dmma<false, true, 2, 2>(g, s);
    else if (g.a_kmajor && !g.b_kmajor) launch_dmma<true, false, 2, 2>(g, s);
    else launch_dmma<true, true, 2, 2>(g, s);
  }
  return 0;
}

template <>
int launch_gemm<float>(const GemmArgs& g, cudaStream_t s) {
  if (g.M <= 0 || g.N <= 0) return 0;
  if (!gemm_contract_ok<float>(g, BN)) return 1;
  if (!g.a_kmajor && !g.b_kmajor) launch_cfg(gemm_simt_kernel<false, false>, g, 0, s);
  else if (!g.a_kmajor && g.b_kmajor) launch_cfg(gemm_simt_kernel<false, true>, g, 0, s);
  else if (g.a_kmajor && !g.b_kmajor) launch_cfg(gemm_simt_kernel<true, false>, g, 0, s);
  else launch_cfg(gemm_simt_kernel<true, true>, g, 0, s);
  return 0;
}
