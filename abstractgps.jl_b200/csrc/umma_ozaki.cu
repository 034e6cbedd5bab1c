// umma_ozaki.cu -- K5 on the Hopper tensor cores: the trailing update and every other large product of the path
//     C (m x n, fp64 or fp32)  +=  sign * A B'      (trailing update: B = A = the factored outer panel, lower tiles, sign -1)
// executed as EXACT int8 x int8 -> int32 products on wgmma.mma_async (s8 x s8 -> s32) with register accumulators,
// operands staged by bulk async copies into shared memory behind mbarriers, recombined exactly and rounded once in the
// epilogue (Ozaki-style error-free splitting).  Replaces the LAPACK potrf trailing update inside
// cholesky(_symmetric(C)) (reference src/finite_gp_projection.jl:308, src/exact_gpr_posterior.jl:31), the rank-512
// updates of `C.U' \ X` (src/util/common_covmat_ops.jl:54,90) and the A A' accumulation of the VFE bound
// (src/sparse_approximations.jl:296-299).
//
// Splitting.  Row i of an operand is scaled by 2^-e_i (e_i: exponent of the row maximum) to |x| < 1 and cut into
// S signed 7-bit slices  x = sum_s q_s 2^-(7s-1),  q_s in [-64, 64]  -- every step exact in fp64.
// Then  a_i . b_j = 2^(e_i+e_j) sum_d 2^(-7d-5) ACC_d[i,j],  ACC_d = sum_{s+t=d+1} q_s . q_t  (int32, exact);
// diagonals d > S are dropped (relative 2^(-7S)).  fp64: 5..8 selectable (S = 7: ~2^-49 of the row scale);
// fp32: S = 4 (28 bits >= the 24-bit significand).  fp64 default: six balanced 8-bit digits instead (ozaki8_update_kernel,
// see ozaki_slice_kernel and oz_combine), 21 MMAs per chunk for ~2^-43.4 of the row-scale products, K <= 16384.
//
// One kernel, ozaki_syrk_wgmma_kernel: persistent or bounded CTAs walking a list of 128 x BN output tiles; one producer
// warp streams the slices with bulk copies, two consumer warpgroups (64 rows each) issue the MMAs and drain their own
// accumulators.  Per 32-byte K chunk a consumer loads each A slice's 64 x 32-byte fragment into registers once
// (ldmatrix) and issues S(S+1)/2 uniform m64nBNk32 MMAs, one per slice pair (s, t), into accumulator block d = s + t;
// only B is read from shared memory.  The blocks never overlap, so ptxas pipelines the issue; wider MMAs against a
// stack of B slices would write overlapping accumulator fragments of different widths, which ptxas serialises.  The
// fragments are double-buffered so one chunk's MMAs stay in flight while the next chunk's fragments load.  The S
// accumulator blocks of 64 x BN int32 live in registers (S*BN/2 per thread), which sets BN: 64 for S <= 4, 32 above.
// The eight-bit kernel instead reads A from shared memory too (oz_chunk_ss): without fragments its six blocks of 64 x 64
// fit, and the wider tile fetches each 128-row A chunk once per 64 columns instead of once per 32 (-40 % operand bytes).
// A from registers would need two fragment buffers (48 registers) beside the 192 accumulators to keep a chunk's MMAs in
// flight while the next chunk's fragments load, more than a consumer thread has.  The producer also stages the tile's
// old C block into shared memory halfway through the tile's K loop, so the drain's read-modify-write does not wait on
// HBM (partial or unaligned tiles read C from global memory as before).
#include <cuda.h>
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "kernels.h"
#include "umma_ozaki.h"
#include "wgmma_i8.h"

namespace {

constexpr int OZ_BM = 128, OZ_KC = 32;  // rows per output tile; K bytes per chunk (one k32 MMA)
constexpr int OZ_THREADS = 384;         // warpgroups 0, 1: consumers; warpgroup 2: producer (one warp issues)

// ---------------------------------------------------------------------------------------------
// pre-pass 1: row exponents
// ---------------------------------------------------------------------------------------------
// |x| for the row maximum, with NaN mapped to +inf: fmax would drop a NaN and the row would lose it silently
__device__ __forceinline__ double oz_mag(double x) { return isnan(x) ? CUDART_INF : fabs(x); }

template <typename Tin>
__global__ void __launch_bounds__(256) ozaki_rowscale_kernel(const Tin* __restrict__ P, int64_t lda, int64_t m, int K, int kmajor,
                                                             double* __restrict__ rscale, double* __restrict__ rinv) {
  // 32 rows x 8 column groups per block: every load instruction of a warp covers 32 consecutive rows of one column
  // (row-contiguous operand) or 32 consecutive k of one row (k-major operand); the row maxima meet in shared memory
  __shared__ double part[8][33];
  double mx = 0.0;
  int64_t row;
  if (!kmajor) {
    const int x = threadIdx.x & 31, y = threadIdx.x >> 5;
    row = blockIdx.x * 32ll + x;
    if (row < m) {
      const Tin* p = P + row + (int64_t)y * lda;
#pragma unroll 4
      for (int k = y; k < K; k += 8, p += 8 * lda) mx = fmax(mx, oz_mag((double)*p));
    }
    part[y][x] = mx;
    __syncthreads();
    if (y != 0) return;
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmax(mx, part[j][x]);
  } else {  // element (row, k) at P[k + row * lda]: one warp per row, lanes along k
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int rr = w; rr < 32; rr += 8) {
      const int64_t r2 = blockIdx.x * 32ll + rr;
      double v = 0.0;
      if (r2 < m)
        for (int k = lane; k < K; k += 32) v = fmax(v, oz_mag((double)P[k + r2 * lda]));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
      if (lane == 0) part[0][rr] = v;
    }
    __syncthreads();
    if (threadIdx.x >= 32) return;
    row = blockIdx.x * 32ll + threadIdx.x;
    mx = part[0][threadIdx.x];
  }
  if (row < m) {
    int e = 0;
    if (mx > 0.0 && isfinite(mx)) frexp(mx, &e);  // mx = f * 2^e, f in [0.5, 1)
    if (e < -1022) e = -1022;  // subnormal rows: 2^1022 scales them exactly and keeps rinv finite
    // a NaN or +-Inf entry, or a maximum >= 2^1023 (2^e overflows): every output the row touches becomes NaN
    const bool bad = !(mx < 0x1p1023);
    rscale[row] = bad ? CUDART_NAN : ldexp(1.0, e);
    rinv[row] = bad ? 0.0 : ldexp(1.0, -e);
  }
}

// pre-pass 2: error-free slicing, 16 consecutive k per thread -> one 16-byte store per slice.  Rows land at
// [dst_row0, dst_row0 + m_fill) of the slice buffer (dst_row0 a multiple of 128; rscale / rinv are already offset).
// BITS = 7: S balanced 7-bit digits peeled off in fp64.  BITS = 8 (S = 6): X = rint(y 2^46) as an int64, |X| <= 2^46, cut
// into the balanced bytes q_5 .. q_1 in [-128, 127] (the low byte, sign-extended; X = (X - q) / 256 is exact) and the
// leading digit q_0 = X, |q_0| <= 64; y = sum_s q_s 2^-(6+8s) to within 2^-47.
template <int S, int BITS, typename Tin>
__global__ void ozaki_slice_kernel(const Tin* __restrict__ P, int64_t lda, int64_t m, int64_t m_fill, int64_t m_alloc,
                                   int K, int kmajor, int64_t dst_row0, const double* __restrict__ rinv, int8_t* __restrict__ SL,
                                   int bulk) {
  static_assert(BITS == 7 || (BITS == 8 && S == 6), "eight-bit digits come in six slices");
  const int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int k0 = blockIdx.y * 16;
  if (row >= m_fill) return;
  double r[16];
  const double inv = (row < m) ? rinv[row] : 0.0;
  if (!kmajor) {
#pragma unroll
    for (int i = 0; i < 16; ++i) r[i] = (row < m) ? (double)P[row + (int64_t)(k0 + i) * lda] * inv : 0.0;
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) r[i] = (row < m) ? (double)P[(k0 + i) + row * lda] * inv : 0.0;
  }
  double up = 64.0, dn = 1.0 / 64.0;  // 2^(7s-1), 2^-(7s-1)
  const int64_t drow = row + dst_row0;
  int8_t q8[BITS == 8 ? S : 1][16];
  if constexpr (BITS == 8) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const double t = r[i] * 0x1p46;
      long long X = (fabs(t) <= 0x1p46) ? __double2ll_rn(t) : 0;  // a non-finite entry (row scale NaN): no conversion
#pragma unroll
      for (int s = S - 1; s > 0; --s) {
        const int q = (int)(int8_t)(X & 0xff);
        q8[s][i] = (int8_t)q;
        X = (X - q) >> 8;
      }
      q8[0][i] = (int8_t)X;
    }
  }
#pragma unroll
  for (int s = 0; s < S; ++s) {
    union { int8_t b[16]; uint4 v; } pk;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      if constexpr (BITS == 8) {
        pk.b[i] = q8[s][i];
      } else {
        double q = rint(r[i] * up);
        if (!(fabs(q) <= 64.0)) q = 0.0;  // only a non-finite entry gets here (its row scale is NaN): no int conversion of it
        r[i] = fma(-q, dn, r[i]);
        pk.b[i] = (int8_t)(int)q;
      }
    }
    if (bulk) {
      // no-swizzle K-major layout of the wgmma descriptors, written directly: chunk (slice, 128-row block, 32-byte
      // k-block) = 4096 contiguous bytes = [16 row-groups][2 k-halves][8 rows][16 B]  (SBO 256 B, LBO 128 B)
      const int64_t rb = drow >> 7, g = (drow & 127) >> 3, r8 = drow & 7;
      const int kb = k0 >> 5, h = (k0 >> 4) & 1;
      // bulk 1: [slice][row block][k block]; bulk 2 (the MMA kernel): [row block][k block][slice] -- the S chunks one
      // (128-row tile, k block) needs are ONE contiguous S*4096-byte run
      const int64_t chunk = (bulk == 2) ? (rb * (K >> 5) + kb) * S + s : ((int64_t)s * (m_alloc >> 7) + rb) * (K >> 5) + kb;
      *reinterpret_cast<uint4*>(SL + chunk * 4096 + ((g * 2 + h) * 8 + r8) * 16) = pk.v;
    } else {
      *reinterpret_cast<uint4*>(SL + ((int64_t)s * m_alloc + drow) * K + k0) = pk.v;
    }
    up *= 128.0;
    dn *= (1.0 / 128.0);
  }
}

// ---------------------------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  uint32_t spins = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (!done && ++spins > (1u << 28)) __trap();  // turn a protocol bug into an error instead of a hang
  }
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// shared-memory matrix descriptor, no swizzle, K-major: LBO = 128 B between the two 16-byte K halves of a 32-byte chunk,
// SBO = 256 B between 8-row groups -- the layout ozaki_slice_kernel writes
__device__ __forceinline__ uint64_t desc_nosw(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(256 >> 4) << 32);
}
__device__ __forceinline__ double ld_cs(const double* p) {
  double v;
  asm volatile("ld.global.cs.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_cs(double* p, double v) { asm volatile("st.global.cs.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ double ld_cs(const float* p) {
  float v;
  asm volatile("ld.global.cs.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return (double)v;
}
__device__ __forceinline__ void st_cs(float* p, double v) { asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"((float)v) : "memory"); }

struct OzTileArgs {
  void* C; int64_t ldc;   // fp64 or fp32
  double sign;            // C += sign * (P P'); -1 for the trailing updates, +1 for accumulations
  int64_t M, N;           // extent of C (rows of P used, columns updated)
  int K;                  // bytes (= elements) per slice row
  const double* rscale;   // 2^e per P row
  int64_t b_tile_stride, b_off;  // column n of C <-> P row  (n / bw) * b_tile_stride + n % bw + b_off  (0 stride = identity + b_off)
  int64_t a_off;                 // row r of C <-> P row r + a_off
  int64_t b_tile_width;          // distribution block width bw in columns (0 -> 128)
  const int64_t* strip_start;    // table walk: first tile index of every BN-column strip (nbj + 1 entries)
  const int32_t* strip_bimin;    // table walk: first valid 128-row tile of every strip
  const int8_t* SL;              // slices in the blocked layout [128-row block][32-byte k chunk][slice][4096 B]
  int epi;                       // drain: 0 Horner-style int64 words, 1 int32 pair pre-combination (K <= 512)
  int c_bulk;                    // C and ldc 16-byte aligned: full tiles stage their C block by bulk copies
};

// per slice count, digit width and C type: output tile 128 x BN, pipeline depth, staged C block (column-major, every
// column padded by 16 bytes so the drain's shared-memory reads are free of bank conflicts).  Eight-bit digits take both
// operands from shared memory, which frees the A fragment registers for 128 x 64 tiles (four stages of 36 KB).
template <int S, int BITS, typename CT>
struct OzCfg {
  static constexpr int BN = (S <= 4 || BITS == 8) ? 64 : 32;
  static constexpr int A_BYTES = OZ_BM * OZ_KC, B_BYTES = BN * OZ_KC;
  static constexpr int STAGE_BYTES = S * (A_BYTES + B_BYTES);
  static constexpr int C_LD = OZ_BM + 16 / (int)sizeof(CT);  // elements per staged C column
  static constexpr int C_BYTES = BN * C_LD * (int)sizeof(CT);
  static constexpr int RING = 220 * 1024 - C_BYTES;
  static constexpr int STAGES = (RING / STAGE_BYTES) > 6 ? 6 : (RING / STAGE_BYTES);
  static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + C_BYTES + 1024;
};

// a tile stages its C block when it lies inside C and the bulk copies are aligned; producer and consumers decide alike
template <int BN>
__device__ __forceinline__ bool oz_c_staged(const OzTileArgs& a, int bi, int bj) {
  return a.c_bulk && (int64_t)(bi + 1) * OZ_BM <= a.M && (int64_t)(bj + 1) * BN <= a.N;
}

// slot index -> (bi, bj) for the diagonal-anchored lower triangle (R = 128 / BN column tiles per row tile), L2-BLOCKED:
// the tile grid is cut into 2048 x 2048 super-blocks (SB row tiles x R*SB column tiles); slots walk one super-block at a
// time, so the CTAs share ~15 MB of slices at any moment instead of cycling through the whole slice buffer.  Row tile bi
// owns column tiles 0 .. min(nbj, R*(bi+1))-1; slots outside the triangle are reported invalid and skipped by all roles.
constexpr int OZ_SB = 16;
template <int R>
__device__ __forceinline__ bool oz_tile(int64_t t, int nbi, int nbj, int& bi, int& bj) {
  constexpr int64_t PER = (int64_t)OZ_SB * R * OZ_SB;
  const int64_t sb = t / PER;
  const int w = (int)(t - sb * PER);
  const int64_t nJ = (nbj + R * OZ_SB - 1) / (R * OZ_SB);  // super-block columns
  const int64_t t_full = nJ * (nJ + 1) / 2;                // super-block rows I < nJ hold I+1 super-blocks
  int64_t I, Jc;
  if (sb < t_full) {
    I = (int64_t)((sqrt(8.0 * (double)sb + 1.0) - 1.0) * 0.5);
    while ((I + 1) * (I + 2) / 2 <= sb) ++I;
    while (I * (I + 1) / 2 > sb) --I;
    Jc = sb - I * (I + 1) / 2;
  } else {
    const int64_t r = sb - t_full;
    I = nJ + r / nJ;
    Jc = r % nJ;
  }
  bi = (int)(I * OZ_SB + w / (R * OZ_SB));
  bj = (int)(Jc * R * OZ_SB + w % (R * OZ_SB));
  return bi < nbi && bj < nbj && bj < R * bi + R;
}

// table-driven walk (block-cyclic column map, rectangular products): strip j owns tiles [start[j], start[j+1]) =
// row tiles bimin[j] ...
__device__ __forceinline__ void oz_tile_tab(int64_t t, int nbj, const int64_t* __restrict__ start,
                                            const int32_t* __restrict__ bimin, int& bi, int& bj) {
  int lo = 0, hi = nbj;  // find the last j with start[j] <= t
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (start[mid] <= t) lo = mid; else hi = mid;
  }
  bj = lo;
  bi = bimin[lo] + (int)(t - start[lo]);
}
template <int BN>
__device__ __forceinline__ bool oz_decode(const OzTileArgs& a, int64_t t, int nbi, int nbj, int& bi, int& bj, int64_t& brow) {
  if (a.strip_start) {
    oz_tile_tab(t, nbj, a.strip_start, a.strip_bimin, bi, bj);
    const int64_t n0 = (int64_t)bj * BN, bw = a.b_tile_width ? a.b_tile_width : 128;
    brow = (a.b_tile_stride ? (n0 / bw) * a.b_tile_stride + (n0 % bw) : n0) + a.b_off;  // stride 0 = identity column map
    return true;
  }
  const bool ok = oz_tile<OZ_BM / BN>(t, nbi, nbj, bi, bj);
  brow = (int64_t)bj * BN + a.b_off;
  return ok;
}

__device__ __forceinline__ double i64_to_f64_exact(long long x) {  // |x| < 2^51: exact, one integer add + one DADD
  return __longlong_as_double(x + 0x4338000000000000LL) - 6755399441055744.0;
}
// exact value of sum_d acc_d 128^(3-d) as two int64 words (hi: d = 0..3, lo: d = 4..S-1, scaled by 128^(S-4)), then ONE
// rounding.  Accumulator block d of element i is acc[d * BN/2 + i].  PAIR32: adjacent accumulators are first combined in
// int32 (valid for K <= 512).  BITS = 8 (six 8-bit digits): h = sum_{d<3} ACC_d 256^(2-d), l = sum_{d>=3} ACC_d 256^(5-d),
// v = h + 2^-24 l = 2^16 sum_d ACC_d 256^-d; |h|, |l| < 2^47 for K <= 16384.
template <int S, int BITS, int BN, bool PAIR32>
__device__ __forceinline__ double oz_combine(const uint32_t* acc, int i) {
  auto r = [&](int d) { return (int)acc[d * (BN / 2) + i]; };
  long long h = 0, l = 0;
  if constexpr (BITS == 8) {
    static_assert(S == 6 && !PAIR32, "eight-bit digits: six slices, int64 words only");
    h = ((long long)r(0) * 256 + r(1)) * 256 + r(2);
    l = ((long long)r(3) * 256 + r(4)) * 256 + r(5);
    return fma(i64_to_f64_exact(l), 1.0 / 16777216.0, i64_to_f64_exact(h));
  } else if constexpr (S <= 4) {  // fp32 operands (3 or 4 slices): everything fits one word, the conversion is the only rounding
    h = r(0);
#pragma unroll
    for (int d = 1; d < S; ++d) h = h * 128 + r(d);
#pragma unroll
    for (int d = S; d < 4; ++d) h *= 128;  // same 128^3 scaling as the longer splits
    return i64_to_f64_exact(h);
  } else if constexpr (PAIR32) {
    const int t01 = r(0) * 128 + r(1), t23 = r(2) * 128 + r(3);
    h = (long long)t01 * 16384 + t23;
    if constexpr (S == 5) l = r(4);
    else if constexpr (S == 6) l = r(4) * 128 + r(5);
    else if constexpr (S == 7) l = (long long)(r(4) * 128 + r(5)) * 128 + r(6);
    else l = (long long)(r(4) * 128 + r(5)) * 16384 + (r(6) * 128 + r(7));
  } else {
    h = (((long long)r(0) * 128 + r(1)) * 128 + r(2)) * 128 + r(3);
    l = r(4);
#pragma unroll
    for (int d = 5; d < S; ++d) l = l * 128 + r(d);
  }
  constexpr double LO_SCALE = (S <= 5) ? 1.0 / 128.0 : (S == 6) ? 1.0 / 16384.0 : (S == 7) ? 1.0 / 2097152.0 : 1.0 / 268435456.0;
  return fma(i64_to_f64_exact(l), LO_SCALE, i64_to_f64_exact(h));
}

__device__ __forceinline__ void ldsm_x4(uint32_t* r, uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr) : "memory");
}

// one 32-byte K chunk of one consumer warpgroup.  sa: the stage; a_lane: this lane's ldmatrix row address inside a
// 4096-byte A chunk (the four 8 x 16-byte core matrices of the warp's 16 rows are exactly the register fragment).
// Loads the S A fragments, then issues A slice s against B slice t into accumulator block s + t for every s + t < S.
// af must not belong to an MMA still in flight.
template <int S, int BN>
__device__ __forceinline__ void oz_chunk(uint32_t* acc, uint32_t (&af)[S][4], uint32_t sa, uint32_t a_lane, uint32_t acc_in) {
  constexpr int A_BYTES = OZ_BM * OZ_KC, B_BYTES = BN * OZ_KC;
#pragma unroll
  for (int s = 0; s < S; ++s) ldsm_x4(af[s], sa + s * A_BYTES + a_lane);
  const uint64_t bdesc = desc_nosw(sa + S * A_BYTES);
  wgmma_fence();
#pragma unroll
  for (int s = 0; s < S; ++s)
#pragma unroll
    for (int t = 0; t < S - s; ++t)  // s = 0 writes every block first: acc_in = 0 starts the tile
      WgmmaI8<BN>::mma(acc + (s + t) * (BN / 2), af[s], bdesc + (uint64_t)(t * (B_BYTES >> 4)), s == 0 ? acc_in : 1u);
  wgmma_commit();
}

// the same chunk with both operands in shared memory (128 x 64 tiles): a_wg = 2048 wg, the warpgroup's 8 row groups of
// each 4096-byte A chunk.  No fragments, so the stage itself is what must outlive the MMAs in flight.
template <int S>
__device__ __forceinline__ void oz_chunk_ss(uint32_t* acc, uint32_t sa, uint32_t a_wg, uint32_t acc_in) {
  constexpr int A_BYTES = OZ_BM * OZ_KC, B_BYTES = 64 * OZ_KC;
  const uint64_t adesc = desc_nosw(sa + a_wg), bdesc = desc_nosw(sa + S * A_BYTES);
  wgmma_fence();
#pragma unroll
  for (int s = 0; s < S; ++s)
#pragma unroll
    for (int t = 0; t < S - s; ++t)
      WgmmaI8SS64::mma(acc + (s + t) * 32, adesc + (uint64_t)(s * (A_BYTES >> 4)), bdesc + (uint64_t)(t * (B_BYTES >> 4)),
                       s == 0 ? acc_in : 1u);
  wgmma_commit();
}

// the drain of one consumer thread: rows r0, r0 + 8 of the tile and columns 8j + 2(lane & 3) + {0, 1} of every
// accumulator block; C += sign * (2^e_i 2^e_j 2^-33) * v with rs[h] = sign 2^e_i 2^-33 (2^-28 for 8-bit digits), streamed
// (.cs) so the int8 slices stay resident in L2.  STAGED: a full tile whose old C is in the staged block; otherwise guarded
// global loads.
template <int S, int BITS, int BN, bool PAIR32, bool STAGED, typename CT>
__device__ __forceinline__ void oz_drain(const OzTileArgs& a, const uint32_t* acc, const CT* cbuf, int bi, int bj, int64_t brow,
                                         int r0, const double* rs) {
  constexpr int C_LD = OzCfg<S, BITS, CT>::C_LD;
  CT* C = (CT*)a.C;
  const int64_t m0 = (int64_t)bi * OZ_BM + r0;
  const int cq = 2 * ((threadIdx.x & 31) & 3);
  constexpr int RND = (BITS == 8) ? 4 : 8;  // the 192 accumulators of the eight-bit tile leave room for 4 loads in flight
#pragma unroll
  for (int i0 = 0; i0 < BN / 2; i0 += RND) {  // RND elements (one or two 8-column groups) per round: loads, then stores
    double cv[RND];
#pragma unroll
    for (int i = i0; i < i0 + RND; ++i) {
      const int c = 8 * (i >> 2) + cq + (i & 1), h = (i >> 1) & 1;
      const int64_t row = m0 + 8 * h, col = (int64_t)bj * BN + c;
      if constexpr (STAGED) cv[i - i0] = (double)cbuf[c * C_LD + r0 + 8 * h];
      else cv[i - i0] = (row < a.M && col < a.N) ? ld_cs(C + row + col * a.ldc) : 0.0;
    }
#pragma unroll
    for (int i = i0; i < i0 + RND; ++i) {
      const int c = 8 * (i >> 2) + cq + (i & 1), h = (i >> 1) & 1;
      const int64_t row = m0 + 8 * h, col = (int64_t)bj * BN + c;
      const double v = oz_combine<S, BITS, BN, PAIR32>(acc, i);
      if (STAGED || (row < a.M && col < a.N)) st_cs(C + row + col * a.ldc, fma(v, rs[h] * a.rscale[brow + c], cv[i - i0]));
    }
  }
}

// the body of the update kernels; BITS is the digit width of the slices (7 or 8), which only the drain sees
template <int S, int BITS, typename CT>
__device__ __forceinline__ void oz_syrk_body(const OzTileArgs& a, int64_t ntiles, int nbi, int nbj, int tpc) {
  // tpc = 0: persistent, CTA b walks slots b, b + grid, ...   tpc > 0: BOUNDED CTAs -- CTA b owns the tpc consecutive slots
  // [b * tpc, (b + 1) * tpc) and exits; the grid is ceil(ntiles / tpc).  Bounded CTAs hand their SM back every ~0.1 ms, so
  // kernels of a higher-priority stream (the panel chain, the NCCL broadcast) are scheduled between them instead of
  // waiting for the whole update.
  using Cfg = OzCfg<S, BITS, CT>;
  constexpr int BN = Cfg::BN, STAGES = Cfg::STAGES, STAGE_BYTES = Cfg::STAGE_BYTES;
  constexpr int A_BYTES = Cfg::A_BYTES, B_BYTES = Cfg::B_BYTES, C_LD = Cfg::C_LD;
  const int64_t t_begin = tpc ? (int64_t)blockIdx.x * tpc : (int64_t)blockIdx.x;
  const int64_t t_end = tpc ? ((t_begin + tpc < ntiles) ? t_begin + tpc : ntiles) : ntiles;
  const int64_t t_step = tpc ? 1 : (int64_t)gridDim.x;
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES], c_full, c_empty;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem) + 1023) & ~(uintptr_t)1023);
  CT* cbuf = reinterpret_cast<CT*>(base + STAGES * STAGE_BYTES);  // staged C block [BN][C_LD]

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    mbar_init(&c_full, 1);
    mbar_init(&c_empty, 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int num_kb = a.K / OZ_KC;  // even: K % 64 == 0
  uint32_t cn = 0;                 // staged C blocks so far (parity of c_full / c_empty)

  if (warp >= 8) {
    // the producer warpgroup hands its registers to the consumers (128 x 40 + 256 x 232 <= 64K)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp != 8) return;
    // ---- producer: all 32 lanes walk the loop (uniform control flow), one elected lane issues the copies: the S
    // A chunks of a stage are ONE contiguous run, the B strips S pieces of BN * 32 bytes stacked behind it
    uint32_t it = 0;
    const int64_t rb_bytes = (int64_t)num_kb * S * 4096;  // bytes of one 128-row block (all k chunks, all slices)
    for (int64_t t = t_begin; t < t_end; t += t_step) {
      int bi, bj;
      int64_t brow;
      if (!oz_decode<BN>(a, t, nbi, nbj, bi, bj, brow)) continue;
      const int64_t arow = (int64_t)bi * OZ_BM + a.a_off;
      const int8_t* asrc = a.SL + (arow >> 7) * rb_bytes;
      const int8_t* bsrc = a.SL + (brow >> 7) * rb_bytes + (brow & 127) * OZ_KC;
      const bool staged = oz_c_staged<BN>(a, bi, bj);
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        if (staged && kb == num_kb / 2) {
          // the tile's C block, one bulk copy per column, half a tile ahead of the drain; by now the consumers are
          // normally past the previous tile's drain, so the wait for the buffer does not stall the ring
          mbar_wait(&c_empty, (cn & 1) ^ 1);
          if (lane == 0) mbar_expect_tx(&c_full, BN * OZ_BM * (uint32_t)sizeof(CT));
          __syncwarp();
          const CT* csrc = (const CT*)a.C + (int64_t)bi * OZ_BM + (int64_t)bj * BN * a.ldc;
          for (int c = lane; c < BN; c += 32) bulk_load(cbuf + c * C_LD, csrc + c * a.ldc, OZ_BM * sizeof(CT), &c_full);
          ++cn;
        }
        const uint32_t st = it % STAGES, ph = (it / STAGES) & 1;
        mbar_wait(&empty_bar[st], ph ^ 1);
        if (elect_one()) {
          uint8_t* dst = base + st * STAGE_BYTES;
          mbar_expect_tx(&full_bar[st], STAGE_BYTES);
          bulk_load(dst, asrc, S * A_BYTES, &full_bar[st]);
#pragma unroll
          for (int sl = 0; sl < S; ++sl) bulk_load(dst + S * A_BYTES + sl * B_BYTES, bsrc + sl * 4096, B_BYTES, &full_bar[st]);
        }
        __syncwarp();
        asrc += S * 4096;
        bsrc += S * 4096;
      }
    }
  } else {
    // ---- consumer warpgroup wg: rows 64*wg .. 64*wg+63 of the tile, all BN columns
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2;
    uint32_t acc[S * BN / 2];
    // A fragments of the even / odd K chunks, so one chunk's MMAs stay in flight while the next chunk's fragments load;
    // one buffer (and a full wait per chunk) where two would not fit next to the accumulators (S = 8)
    constexpr int NAF = (S * BN / 2 + 2 * 4 * S <= 168) ? 2 : 1;
    uint32_t af[NAF][S][4];
    uint32_t it = 0;
    const uint32_t smem0 = smem_u32(base);
    // ldmatrix.x4 row address: lanes 8j .. 8j+7 read core matrix j = (row group 8 wg + 2 (warp & 3) + (j & 1), K half j >> 1)
    const uint32_t a_lane = (((8 * wg + 2 * (warp & 3) + ((lane >> 3) & 1)) * 2 + (lane >> 4)) * 8 + (lane & 7)) * 16;
    for (int64_t t = t_begin; t < t_end; t += t_step) {
      int bi, bj;
      int64_t brow;
      if (!oz_decode<BN>(a, t, nbi, nbj, bi, bj, brow)) continue;
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const uint32_t st = it % STAGES, ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[st], ph);
        const uint32_t sa = smem0 + st * STAGE_BYTES;
        if constexpr (BITS == 8) {
          // the MMAs of chunk kb - 1 still read their stage until the wait below retires them
          oz_chunk_ss<S>(acc, sa, 2048u * wg, kb != 0 ? 1u : 0u);
          if (kb > 0) {
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
          }
        } else if constexpr (NAF == 2) {
          // the fragments of chunk kb - 2 are free: its MMAs completed at the wait below in iteration kb - 1
          if (kb & 1) oz_chunk<S, BN>(acc, af[NAF - 1], sa, a_lane, 1u);
          else oz_chunk<S, BN>(acc, af[0], sa, a_lane, kb != 0 ? 1u : 0u);
          if (kb > 0) {  // the previous chunk's MMAs are done: its stage may be refilled
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
          }
        } else {
          oz_chunk<S, BN>(acc, af[0], sa, a_lane, kb != 0 ? 1u : 0u);
          wgmma_wait<0>();
          if (lane == 0) mbar_arrive(&empty_bar[st]);
        }
      }
      if constexpr (NAF == 2 || BITS == 8) {
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }

      const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // row inside the tile
      double rs[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = (int64_t)bi * OZ_BM + r0 + 8 * h;
        // 7 bits: +-2^e_i * 2^-12 * 128^-3;  8 bits: +-2^e_i * 2^-12 * 2^-16 (v carries 2^16 sum_d ACC_d 256^-d)
        constexpr double SCALE = (BITS == 8) ? 1.0 / 268435456.0 : 1.0 / 8589934592.0;
        rs[h] = row < a.M ? a.sign * a.rscale[row + a.a_off] * SCALE : 0.0;
      }
      const bool staged = oz_c_staged<BN>(a, bi, bj);
      if (staged) mbar_wait(&c_full, cn & 1);
      if (BITS == 7 && a.epi == 1) {
        if (staged) oz_drain<S, BITS, BN, BITS == 7, true>(a, acc, cbuf, bi, bj, brow, r0, rs);
        else oz_drain<S, BITS, BN, BITS == 7, false>(a, acc, cbuf, bi, bj, brow, r0, rs);
      } else {
        if (staged) oz_drain<S, BITS, BN, false, true>(a, acc, cbuf, bi, bj, brow, r0, rs);
        else oz_drain<S, BITS, BN, false, false>(a, acc, cbuf, bi, bj, brow, r0, rs);
      }
      if (staged) {  // this warp has read its part of the staged block
        __syncwarp();
        if (lane == 0) mbar_arrive(&c_empty);
        ++cn;
      }
    }
  }
}

// seven-bit slices: fp64 C with 4..8 slices, fp32 C with 3..5
template <int S, typename CT>
__global__ void __launch_bounds__(OZ_THREADS, 1) ozaki_syrk_wgmma_kernel(OzTileArgs a, int64_t ntiles, int nbi, int nbj, int tpc) {
  oz_syrk_body<S, 7, CT>(a, ntiles, nbi, nbj, tpc);
}
// six eight-bit slices, fp64 C
__global__ void __launch_bounds__(OZ_THREADS, 1) ozaki8_update_kernel(OzTileArgs a, int64_t ntiles, int nbi, int nbj, int tpc) {
  oz_syrk_body<6, 8, double>(a, ntiles, nbi, nbj, tpc);
}

template <int S, int BITS, typename CT>
struct OzKernel {
  static_assert(BITS == 7, "eight-bit digits: six slices and fp64 C only");
  static constexpr auto fn = ozaki_syrk_wgmma_kernel<S, CT>;
};
template <>
struct OzKernel<6, 8, double> {
  static constexpr auto fn = ozaki8_update_kernel;
};

// C += sign * P_A P_B' on the slices in ws.  full = 0: lower tiles only; returns 1 if the shape needs a longer strip
// table than the workspace holds.
template <int S, int BITS, typename CT>
int launch_syrk_wgmma(const OzakiWs& ws, void* C, int64_t ldc, int64_t M, int64_t N, int64_t b_tile_stride,
                      int64_t b_tile_width, int64_t b_off, int64_t a_off, cudaStream_t s, int full, double sign) {
  using Cfg = OzCfg<S, BITS, CT>;
  constexpr int BN = Cfg::BN, R = OZ_BM / BN;
  constexpr auto kernel = OzKernel<S, BITS, CT>::fn;
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  static int nsm = 0;
  if (agp_first_use_on_device(&configured)) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
  }
  OzTileArgs a{};
  a.C = C; a.ldc = ldc; a.M = M; a.N = N; a.K = ws.K; a.rscale = ws.rscale;
  a.b_tile_stride = b_tile_stride; a.b_tile_width = b_tile_width; a.b_off = b_off; a.a_off = a_off;
  a.SL = ws.SL;
  a.sign = sign;
  a.c_bulk = ((uintptr_t)C % 16 == 0) && ((uint64_t)ldc * sizeof(CT)) % 16 == 0;
  {
    // default: the int32 pair pre-combination (S >= 5, K <= 512: bit-identical to the int64 words, fewer integer ops);
    // AGP_OZAKI_EPI=0 restores the plain int64 drain
    const char* e = getenv("AGP_OZAKI_EPI");
    a.epi = (e && atoi(e) == 0) ? 0 : 1;
    if (ws.K > 512 || BITS == 8) a.epi = 0;  // the int32 pair bound needs K <= 512 (at 8 bits 256 ACC wraps from K = 512)
  }
  const int nbi = (int)((M + OZ_BM - 1) / OZ_BM), nbj = (int)((N + BN - 1) / BN);
  int64_t ntiles = 0;
  if (!full && b_tile_stride == 0 && a_off == b_off) {  // diagonal-anchored: closed-form, L2-blocked slot enumeration
    const int64_t nJ = (nbj + R * OZ_SB - 1) / (R * OZ_SB), nI = (nbi + OZ_SB - 1) / OZ_SB;
    const int64_t nsb = (nI <= nJ) ? nI * (nI + 1) / 2 : nJ * (nJ + 1) / 2 + (nI - nJ) * nJ;
    ntiles = nsb * (int64_t)OZ_SB * R * OZ_SB;  // slots, including the skipped ones of diagonal / edge super-blocks
  } else {  // block-cyclic column map or rectangular product: per-strip table (host -> device, a few KB)
    if (nbj > ws.tab_cap) return 1;
    std::vector<int64_t> start((size_t)nbj + 1);
    std::vector<int32_t> bimin((size_t)nbj);
    const int64_t bw = b_tile_width ? b_tile_width : 128;
    for (int j = 0; j < nbj; ++j) {
      const int64_t n0 = (int64_t)j * BN;
      const int64_t nsrc = (b_tile_stride ? (n0 / bw) * b_tile_stride + (n0 % bw) : n0) + b_off;
      int64_t bm = (nsrc - a_off) >= 0 ? (nsrc - a_off) / OZ_BM : 0;  // first row tile with nsrc < a_off + bi*128 + 128
      if (full) bm = 0;  // rectangular product: every row tile of every strip
      if (bm > nbi) bm = nbi;
      bimin[j] = (int32_t)bm;
      start[j] = ntiles;
      ntiles += nbi - bm;
    }
    start[nbj] = ntiles;
    const int slot = (ws.tab_slot++) & 1;  // the main- and side-stream updates of one step are in flight together
    int64_t* d_start = ws.tab_start + (size_t)slot * (ws.tab_cap + 1);
    int32_t* d_bimin = ws.tab_bimin + (size_t)slot * (ws.tab_cap + 1);
    cudaMemcpyAsync(d_start, start.data(), ((size_t)nbj + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_bimin, bimin.data(), (size_t)nbj * sizeof(int32_t), cudaMemcpyHostToDevice, s);
    a.strip_start = d_start;
    a.strip_bimin = d_bimin;
  }
  if (ntiles <= 0) return 0;
  const int cap = (ws.max_ctas > 0 && ws.max_ctas < nsm) ? ws.max_ctas : nsm;
  int64_t grid = cap < ntiles ? cap : ntiles;
  // chunk_tiles counts 128 x 32 tiles; a 128 x 64 tile (eight-bit digits) covers two, so a bounded CTA keeps its area
  const int tpc = (BITS == 8 && ws.chunk_tiles > 1) ? ws.chunk_tiles / 2 : ws.chunk_tiles;
  if (tpc > 0) grid = (ntiles + tpc - 1) / tpc;
  kernel<<<(unsigned)grid, OZ_THREADS, Cfg::SMEM, s>>>(a, ntiles, nbi, nbj, tpc);
  agp_count_launch();
  return 0;
}

}  // namespace

int ozaki_ws_create(OzakiWs* ws, int64_t max_rows, int K, int S, cudaStream_t s, int bits) {
  memset(ws, 0, sizeof(*ws));
  if (S < 3 || S > 8 || K % 64 != 0 || (bits != 7 && bits != 8) || (bits == 8 && S != 6)) return 1;
  ws->m_alloc = (max_rows + 127) / 128 * 128;
  ws->K = K; ws->S = S; ws->bits = bits;
  if (cudaMallocAsync((void**)&ws->SL, (size_t)S * ws->m_alloc * K, s) != cudaSuccess) return 3;
  if (cudaMallocAsync((void**)&ws->rscale, (size_t)ws->m_alloc * 2 * sizeof(double), s) != cudaSuccess) return 3;
  ws->rinv = ws->rscale + ws->m_alloc;
  ws->tab_cap = (int)(ws->m_alloc / 32) + 2;  // strips of the narrowest tile (32 columns)
  if (cudaMallocAsync((void**)&ws->tab_start, (size_t)2 * (ws->tab_cap + 1) * sizeof(int64_t), s) != cudaSuccess) return 3;
  if (cudaMallocAsync((void**)&ws->tab_bimin, (size_t)2 * (ws->tab_cap + 1) * sizeof(int32_t), s) != cudaSuccess) return 3;
  ws->bulk = 2;
  { const char* ct = getenv("AGP_OZAKI_CHUNK_TEST"); ws->chunk_tiles = ct ? atoi(ct) : 0; }  // tests: bounded CTAs everywhere
  return 0;
}

void ozaki_ws_destroy(OzakiWs* ws, cudaStream_t s) {
  if (ws->SL) cudaFreeAsync(ws->SL, s);
  if (ws->rscale) cudaFreeAsync(ws->rscale, s);
  if (ws->tab_start) cudaFreeAsync(ws->tab_start, s);
  if (ws->tab_bimin) cudaFreeAsync(ws->tab_bimin, s);
  memset(ws, 0, sizeof(*ws));
}

template <typename Tin>
static void prepare_t(const OzakiWs& ws, const Tin* P, int kmajor, int64_t lda, int64_t m, int64_t dst_row0, cudaStream_t s) {
  double* rs = ws.rscale + dst_row0;
  double* ri = ws.rinv + dst_row0;
  ozaki_rowscale_kernel<Tin><<<(unsigned)((m + 31) / 32), 256, 0, s>>>(P, lda, m, ws.K, kmajor, rs, ri);
  agp_count_launch();
  const int64_t m_used = (m + 127) / 128 * 128;  // zero-fill up to the tile edge
  dim3 grid((unsigned)((m_used + 127) / 128), (unsigned)(ws.K / 16));
#define AGP_SLICE(SS, BB) ozaki_slice_kernel<SS, BB, Tin><<<grid, 128, 0, s>>>(P, lda, m, m_used, ws.m_alloc, ws.K, kmajor, dst_row0, ri, ws.SL, ws.bulk)
  if (ws.bits == 8) {
    AGP_SLICE(6, 8);
  } else {
    switch (ws.S) {
      case 3: AGP_SLICE(3, 7); break;
      case 4: AGP_SLICE(4, 7); break;
      case 5: AGP_SLICE(5, 7); break;
      case 6: AGP_SLICE(6, 7); break;
      case 7: AGP_SLICE(7, 7); break;
      default: AGP_SLICE(8, 7); break;
    }
  }
#undef AGP_SLICE
  agp_count_launch();
}

void ozaki_prepare(const OzakiWs& ws, const double* P, int64_t lda, int64_t m, cudaStream_t s) {
  if (m <= 0) return;
  prepare_t<double>(ws, P, 0, lda, m, 0, s);
}

void ozaki_prepare_ex(const OzakiWs& ws, const void* P, int p_is_float, int kmajor, int64_t lda, int64_t m, int64_t dst_row0,
                      cudaStream_t s) {
  if (m <= 0) return;
  if (p_is_float) prepare_t<float>(ws, (const float*)P, kmajor, lda, m, dst_row0, s);
  else prepare_t<double>(ws, (const double*)P, kmajor, lda, m, dst_row0, s);
}

int ozaki_update_ex(const OzakiWs& ws, void* C, int c_is_float, int64_t ldc, int64_t M, int64_t N, int full, double sign,
                    int64_t b_tile_stride, int64_t b_tile_width, int64_t b_off, int64_t a_off, cudaStream_t s) {
  if (M <= 0 || N <= 0) return 0;
  if (ws.bulk != 2 || N % 128 != 0) return 1;
  if (ws.K > 32768) return 1;  // int32 accumulators ((d+1) K 64^2 < 2^31) and the 2^51 range of the exact int64 -> fp64 drain
#define AGP_UPD(SS, CTT) return launch_syrk_wgmma<SS, 7, CTT>(ws, C, ldc, M, N, b_tile_stride, b_tile_width, b_off, a_off, s, full, sign)
  if (ws.bits == 8) {
    if (c_is_float || ws.K > OZ8_MAX_K) return 1;
    return launch_syrk_wgmma<6, 8, double>(ws, C, ldc, M, N, b_tile_stride, b_tile_width, b_off, a_off, s, full, sign);
  }
  if (c_is_float) {
    switch (ws.S) {
      case 3: AGP_UPD(3, float);
      case 4: AGP_UPD(4, float);
      case 5: AGP_UPD(5, float);
      default: return 1;
    }
  } else {
    switch (ws.S) {
      case 4: AGP_UPD(4, double);
      case 5: AGP_UPD(5, double);
      case 6: AGP_UPD(6, double);
      case 7: AGP_UPD(7, double);
      case 8: AGP_UPD(8, double);
      default: return 1;
    }
  }
#undef AGP_UPD
}

int ozaki_syrk(const OzakiWs& ws, double* C, int64_t ldc, int64_t M, int64_t N, int lower_only, int64_t b_tile_stride,
               int64_t b_tile_width, int64_t b_off, int64_t a_off, cudaStream_t s) {
  if (M <= 0 || N <= 0) return 0;
  const int full = lower_only ? 0 : 1;
  if (ws.bits == 8) {
    if (ws.K > OZ8_MAX_K) return 1;
    return launch_syrk_wgmma<6, 8, double>(ws, C, ldc, M, N, b_tile_stride, b_tile_width, b_off, a_off, s, full, -1.0);
  }
  switch (ws.S) {
    case 5: return launch_syrk_wgmma<5, 7, double>(ws, C, ldc, M, N, b_tile_stride, b_tile_width, b_off, a_off, s, full, -1.0);
    case 6: return launch_syrk_wgmma<6, 7, double>(ws, C, ldc, M, N, b_tile_stride, b_tile_width, b_off, a_off, s, full, -1.0);
    case 7: return launch_syrk_wgmma<7, 7, double>(ws, C, ldc, M, N, b_tile_stride, b_tile_width, b_off, a_off, s, full, -1.0);
    case 8: return launch_syrk_wgmma<8, 7, double>(ws, C, ldc, M, N, b_tile_stride, b_tile_width, b_off, a_off, s, full, -1.0);
    default: return 1;  // fp64 C is instantiated for 5..8 slices only (a 3- or 4-slice workspace is for fp32 panels)
  }
}
