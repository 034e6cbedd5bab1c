// potrf.cu -- K3: Cholesky of one 128x128 diagonal block, entirely in shared memory, fused with the
// inverse of the factor (used by the TRSM-as-GEMM panel solve and the blocked triangular solves).
// Replaces the diagonal-block part of LAPACK potrf inside cholesky(_symmetric(C))
// (/root/reference/src/finite_gp_projection.jl:308, /root/reference/src/exact_gpr_posterior.jl:31).
//
// Scheme: the lower triangle of the smem array holds A -> L; the STRICT UPPER triangle holds the rows
// of E = I * L^-T that a bordered elimination produces for free (E(r,c) lives at position (c,r)), its
// diagonal (1/L_jj) in dinv[].  16 micro-panels of 8 columns.  Row worker w is S row w until the
// micro-panel that finishes it, then E row w -- so all 128 workers (x2 column-parity halves) stay busy.
// Phase A: every thread factors the 8x8 diagonal block redundantly in registers (no shuffles, no
// barrier on the sqrt chain) and substitutes its own row; phase B: rank-8 trailing update of its row.
#include <stdlib.h>

#include "kernels.h"
#include "agp.h"

namespace {
constexpr int PB = AGP_TILE;  // 128
constexpr int PLD = PB + 1;   // odd leading dimension -> conflict-free column/row access

// 1/sqrt(p) on the critical path of the column chain: hardware approximation (MUFU.RSQ64H, ~20 bits)
// + two Newton steps (3 dependent DFMA-class ops each) -> full fp64 precision, ~half the dependent
// depth of rsqrt(double)'s library sequence.  p is a positive pivot.  The approximation flushes a subnormal input to
// zero (+Inf, then NaN after the Newton steps), so a subnormal p is scaled by 2^108 first and the result by 2^54; both
// scalings are exact, and a normal p takes the unscaled path unchanged.
template <typename T> __device__ __forceinline__ T dev_rsqrt_refined(T p);
template <> __device__ __forceinline__ double dev_rsqrt_refined<double>(double p) {
  const bool sub = p < 0x1p-1022;
  const double ps = sub ? p * 0x1p+108 : p;
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(ps));
  const double hp = -0.5 * ps;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const double e = fma(hp * y, y, 0.5);  // 0.5 - 0.5 p y^2
    y = fma(y, e, y);                      // y (1.5 - 0.5 p y^2)
  }
  return sub ? y * 0x1p+54 : y;
}
template <> __device__ __forceinline__ float dev_rsqrt_refined<float>(float p) {
  float r = rsqrtf(p);
  return fmaf(r * 0.5f, fmaf(-p * r, r, 1.0f), r);
}

template <typename T> __device__ __forceinline__ void load8(const T* p, T* o);
template <> __device__ __forceinline__ void load8<double>(const double* p, double* o) {
  const double2* q = reinterpret_cast<const double2*>(p);
#pragma unroll
  for (int i = 0; i < 4; ++i) { double2 v = q[i]; o[2 * i] = v.x; o[2 * i + 1] = v.y; }
}
template <> __device__ __forceinline__ void load8<float>(const float* p, float* o) {
  const float4* q = reinterpret_cast<const float4*>(p);
#pragma unroll
  for (int i = 0; i < 2; ++i) { float4 v = q[i]; o[4 * i] = v.x; o[4 * i + 1] = v.y; o[4 * i + 2] = v.z; o[4 * i + 3] = v.w; }
}

template <typename T>
__global__ void __launch_bounds__(256, 1)
potrf_diag_kernel(T* __restrict__ A, int64_t lda, T* __restrict__ Dinv, double* __restrict__ logdet_part,
                  int blk, int* __restrict__ info) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* arr = reinterpret_cast<T*>(smem_raw);  // arr[c*PLD + i]
  T* P8 = arr + PB * PLD;                   // P8[k*8 + c] : factored micro-panel, row k (16B aligned: PB*PLD even)
  T* dinv = P8 + PB * 8;
  __shared__ double red[4];
  const int tid = threadIdx.x;
  const int w = tid & (PB - 1), half = tid >> 7;  // row worker, column-parity half

  // global -> smem: 64 elements per thread, issued as 4 batches of 16 INDEPENDENT loads (a plain loop
  // serialises one DRAM round trip per element: 64 x ~0.8 us)
#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    T tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int c = idx >> 7, i = idx & 127;
      tmp[u] = (i >= c) ? __ldg(A + i + (int64_t)c * lda) : (T)0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      arr[(idx >> 7) * PLD + (idx & 127)] = tmp[u];
    }
  }
  __syncthreads();

  for (int j0 = 0; j0 < PB; j0 += 8) {
    // ---- phase A: every thread factors the 8x8 diagonal block redundantly in registers (no shuffles,
    // no barrier on the sqrt chain), then substitutes its own row against it.
    T d[8][8], rinv[8], x[8];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c <= r; ++c) d[r][c] = arr[(j0 + c) * PLD + j0 + r];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      T piv = d[c][c];
      if (!(piv > (T)0)) {
        if (tid == j0) atomicCAS(info, 0, blk * PB + j0 + c + 1);
        piv = (T)1;
      }
      const T r = dev_rsqrt_refined<T>(piv);
      rinv[c] = r;
      d[c][c] = piv * r;
#pragma unroll
      for (int r2 = c + 1; r2 < 8; ++r2) d[r2][c] *= r;
#pragma unroll
      for (int c2 = c + 1; c2 < 8; ++c2)
#pragma unroll
        for (int r2 = c2; r2 < 8; ++r2) d[r2][c2] -= d[r2][c] * d[c2][c];
    }
    const bool is_s = (w >= j0 + 8);          // still an S (factor) row; otherwise an E (inverse) row
    const bool is_diag = (w >= j0) && !is_s;  // one of the 8 diagonal rows of this micro-panel
    {
      T a[8];
      if (is_diag) {
        const int cr = w - j0;
#pragma unroll
        for (int c = 0; c < 8; ++c) a[c] = (c == cr) ? (T)1 : (T)0;
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) a[c] = arr[(j0 + c) * PLD + w];
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        T sacc = a[c];
#pragma unroll
        for (int c2 = 0; c2 < c; ++c2) sacc -= x[c2] * d[c][c2];
        x[c] = sacc * rinv[c];
      }
    }
    __syncthreads();  // every thread has read its inputs from arr before anyone overwrites them
    if (half == 0) {
      if (is_s) {
#pragma unroll
        for (int c = 0; c < 8; ++c) { arr[(j0 + c) * PLD + w] = x[c]; P8[w * 8 + c] = x[c]; }
      } else if (is_diag) {
        const int cr = w - j0;
#pragma unroll
        for (int r = 0; r < 8; ++r)
          if (r == cr) {
#pragma unroll
            for (int c = 0; c <= r; ++c) arr[(j0 + c) * PLD + w] = d[r][c];  // L row (lower part)
            dinv[w] = rinv[r];
          }
#pragma unroll
        for (int c = 0; c < 8; ++c)
          if (c > cr) arr[(j0 + c) * PLD + w] = x[c];  // E row (strict upper part)
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) arr[(j0 + c) * PLD + w] = x[c];
      }
    }
    __syncthreads();
    // ---- phase B: rank-8 trailing update of row w (S rows: columns <= w; E rows: all remaining columns).
    // 8 columns per trip, each dot product split into two 4-term chains: 16 independent DFMA chains
    // of depth 4 keep the (long-latency) fp64 pipe issue-bound instead of latency-bound.
    {
      const int kend = is_s ? w : (PB - 1);
      int k = j0 + 8 + half;
      for (; k + 14 <= kend; k += 16) {
        T lk[8][8], v0[8], v1[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) { load8<T>(P8 + (k + 2 * u) * 8, lk[u]); v0[u] = arr[(k + 2 * u) * PLD + w]; v1[u] = (T)0; }
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int u = 0; u < 8; ++u) { v0[u] -= x[c] * lk[u][c]; v1[u] -= x[c + 4] * lk[u][c + 4]; }
#pragma unroll
        for (int u = 0; u < 8; ++u) arr[(k + 2 * u) * PLD + w] = v0[u] + v1[u];
      }
      for (; k <= kend; k += 2) {
        T lk[8];
        load8<T>(P8 + k * 8, lk);
        T v0 = arr[k * PLD + w], v1 = (T)0;
#pragma unroll
        for (int c = 0; c < 4; ++c) { v0 -= x[c] * lk[c]; v1 -= x[c + 4] * lk[c + 4]; }
        arr[k * PLD + w] = v0 + v1;
      }
    }
    __syncthreads();
  }

  // ---- write back L (upper zeroed) and Dinv = inv(L) (lower, col-major)
  for (int idx = tid; idx < PB * PB; idx += 256) {
    int c = idx >> 7, i = idx & 127;  // (row i, col c)
    A[i + (int64_t)c * lda] = (i >= c) ? arr[c * PLD + i] : (T)0;
  }
  for (int idx = tid; idx < PB * PB; idx += 256) {
    int r = idx >> 7, c = idx & 127;  // Dinv(c, r) = E(r, c)
    T v = (c > r) ? arr[c * PLD + r] : ((c == r) ? dinv[r] : (T)0);
    Dinv[c + r * PB] = v;
  }
  // ---- logdet partial: sum_j log L_jj = - sum_j log dinv_j
  double part = 0.0;
  if (tid < PB) part = -log((double)dinv[tid]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (tid < PB && (tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  if (tid == 0) logdet_part[blk] = red[0] + red[1] + red[2] + red[3];
}

// ------------------------------------------------------------------------------------------------
// fp64 specialisation (v3).  Same data scheme, but (1) ONE warp factors the 8x8 diagonal block
// (lane-redundant, in registers) and publishes it through shared memory, (2) 128 row workers
// substitute their row, (3) the rank-8 trailing update runs on the DMMA tensor pipe:
// 8x8 output tiles C(rows, cols k) -= X(rows, 0:8) * X(k, 0:8)', two mma.m8n8k4 per tile, warps
// stride over the flattened tile list (E row-groups x all remaining column groups, then the lower
// triangle of S row-groups).  ~8x fewer issue slots than per-element DFMA.
// ------------------------------------------------------------------------------------------------
constexpr int XLD = 9;  // micro-panel row stride (doubles): odd -> conflict-free 64-bit stores

__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(256, 1)
potrf_diag_kernel_f64(double* __restrict__ A, int64_t lda, double* __restrict__ Dinv, double* __restrict__ logdet_part,
                      int blk, int* __restrict__ info) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* arr = reinterpret_cast<double*>(smem_raw);  // arr[c*PLD + i]
  double* XS = arr + PB * PLD;                        // XS[row*XLD + c]: substituted micro-panel, all 128 workers
  double* Ld = XS + PB * XLD;                         // Ld[r*8 + c], c <= r
  double* rinv_s = Ld + 64;                           // 8
  double* dinv = rinv_s + 8;                          // 128
  __shared__ double red[4];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, q = lane & 3;

#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int c = idx >> 7, i = idx & 127;
      tmp[u] = (i >= c) ? __ldg(A + i + (int64_t)c * lda) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      arr[(idx >> 7) * PLD + (idx & 127)] = tmp[u];
    }
  }
  __syncthreads();

  for (int j0 = 0; j0 < PB; j0 += 8) {
    const int J = j0 >> 3;
    // ---- (1) warp 0: 8x8 diagonal Cholesky in registers (every lane computes the same values)
    const int w = tid;  // row worker id for tid < 128
    double a[8];
    const bool worker = tid < PB;
    const bool is_s = worker && (w >= j0 + 8);
    const bool is_diag = worker && (w >= j0) && (w < j0 + 8);
    if (worker && !is_diag) {  // prefetch own row's micro-panel entries while warp 0 works
#pragma unroll
      for (int c = 0; c < 8; ++c) a[c] = arr[(j0 + c) * PLD + w];
    }
    if (warp == 0) {
      double d[8][8];
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c <= r; ++c) d[r][c] = arr[(j0 + c) * PLD + j0 + r];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        double piv = d[c][c];
        if (!(piv > 0.0)) {
          if (lane == 0) atomicCAS(info, 0, blk * PB + j0 + c + 1);
          piv = 1.0;
        }
        const double r = dev_rsqrt_refined<double>(piv);
        if (lane == 0) rinv_s[c] = r;
        d[c][c] = piv * r;
#pragma unroll
        for (int r2 = c + 1; r2 < 8; ++r2) d[r2][c] *= r;
#pragma unroll
        for (int c2 = c + 1; c2 < 8; ++c2)
#pragma unroll
          for (int r2 = c2; r2 < 8; ++r2) d[r2][c2] -= d[r2][c] * d[c2][c];
      }
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < 8; ++r)
#pragma unroll
          for (int c = 0; c <= r; ++c) Ld[r * 8 + c] = d[r][c];
      }
    }
    __syncthreads();
    // ---- (2) substitution by the 128 row workers
    if (worker) {
      double x[8];
      if (is_diag) {
        const int cr = w - j0;
#pragma unroll
        for (int c = 0; c < 8; ++c) a[c] = (c == cr) ? 1.0 : 0.0;
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        double sacc = a[c];
#pragma unroll
        for (int c2 = 0; c2 < c; ++c2) sacc -= x[c2] * Ld[c * 8 + c2];
        x[c] = sacc * rinv_s[c];
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) XS[w * XLD + c] = x[c];
      if (is_s) {
#pragma unroll
        for (int c = 0; c < 8; ++c) arr[(j0 + c) * PLD + w] = x[c];
      } else if (is_diag) {
        const int cr = w - j0;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          if (c <= cr) arr[(j0 + c) * PLD + w] = Ld[cr * 8 + c];  // L row (lower part of the diagonal block)
          else arr[(j0 + c) * PLD + w] = x[c];                    // E row (strict upper part)
        }
        dinv[w] = rinv_s[cr];
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) arr[(j0 + c) * PLD + w] = x[c];
      }
    }
    __syncthreads();
    // ---- (3) rank-8 trailing update on the DMMA pipe.  Warp wi owns row-groups wi and 15-wi (8 rows
    // each); an E group (rows already factored) sweeps all remaining column groups, an S group only
    // those up to its own.  Four 8x8 tiles per trip: 16 independent smem loads, then 8 DMMAs.
    // (A round-robin deal of 4-tile jobs over the warps balanced better on paper but measured 72 us
    // vs 52 us for this static map: the per-job bookkeeping costs more than the imbalance.)
    {
#pragma unroll
      for (int sel = 0; sel < 2; ++sel) {
        const int rg = sel ? (15 - warp) : warp;
        const bool isE = (rg <= J);
        const int kg_lo = J + 1, kg_hi = isE ? 15 : rg;
        if (kg_hi < kg_lo) continue;
        const int r0 = rg * 8;
        const double a0 = -XS[(r0 + gq) * XLD + q], a1 = -XS[(r0 + gq) * XLD + 4 + q];
        for (int kg = kg_lo; kg <= kg_hi; kg += 4) {
          double b0[4], b1[4], c0[4], c1[4];
          double* cp[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int kgu = min(kg + u, 15);
            b0[u] = XS[(kgu * 8 + gq) * XLD + q];
            b1[u] = XS[(kgu * 8 + gq) * XLD + 4 + q];
            cp[u] = arr + (kgu * 8 + 2 * q) * PLD + r0 + gq;
            c0[u] = cp[u][0];
            c1[u] = cp[u][PLD];
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a0, b0[u]);
#pragma unroll
          for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a1, b1[u]);
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int kgu = kg + u;
            if (kgu <= kg_hi) {
              const bool diag_tile = (!isE) && (kgu == rg);
              if (!diag_tile || 2 * q <= gq) cp[u][0] = c0[u];  // S diagonal tile: keep only k <= row
              if (!diag_tile || 2 * q + 1 <= gq) cp[u][PLD] = c1[u];
            }
          }
        }
      }
    }
    __syncthreads();
  }

  // ---- write back L (upper zeroed) and Dinv = inv(L); smem reads batched 16 deep
#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int c = idx >> 7, i = idx & 127;
      tmp[u] = (i >= c) ? arr[c * PLD + i] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      A[(idx & 127) + (int64_t)(idx >> 7) * lda] = tmp[u];
    }
  }
#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int r = idx >> 7, c = idx & 127;  // Dinv(c, r) = E(r, c)
      tmp[u] = (c > r) ? arr[c * PLD + r] : ((c == r) ? dinv[r] : 0.0);
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) Dinv[tid + 256 * (b0 + u)] = tmp[u];
  }
  double part = 0.0;
  if (tid < PB) part = -log(dinv[tid]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (tid < PB && (tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  if (tid == 0) logdet_part[blk] = red[0] + red[1] + red[2] + red[3];
}

// ------------------------------------------------------------------------------------------------
// Split variant (default for fp64): the inverse is 2/3 of the rank-8 update work and half of the
// write-back, and its rows are independent of each other -- so the factorisation kernel does the S rows
// only (one CTA, on the critical path) and the inverse is produced by 8 CTAs in parallel, CTA p owning the
// E row-groups p and 15-p (balanced: the early groups sweep many column groups, the late ones few).
// ------------------------------------------------------------------------------------------------
// 8x8 Cholesky of the diagonal block at micro-panel j0, lane-redundant in one warp; publishes Ld / rinv_s
__device__ __forceinline__ void factor_diag8(const double* arr, int j0, int lane, double* Ld, double* rinv_s, int blk, int* info) {
  double d[8][8];
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int c = 0; c <= r; ++c) d[r][c] = arr[(j0 + c) * PLD + j0 + r];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    double piv = d[c][c];
    if (!(piv > 0.0)) {
      if (lane == 0) atomicCAS(info, 0, blk * PB + j0 + c + 1);
      piv = 1.0;
    }
    const double r = dev_rsqrt_refined<double>(piv);
    if (lane == 0) rinv_s[c] = r;
    d[c][c] = piv * r;
#pragma unroll
    for (int r2 = c + 1; r2 < 8; ++r2) d[r2][c] *= r;
#pragma unroll
    for (int c2 = c + 1; c2 < 8; ++c2)
#pragma unroll
      for (int r2 = c2; r2 < 8; ++r2) d[r2][c2] -= d[r2][c] * d[c2][c];
  }
  if (lane == 0) {
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c <= r; ++c) Ld[r * 8 + c] = d[r][c];
  }
}

// rank-8 update of the S tiles of row-group rg against column groups kg_lo..kg_hi (4 tiles per trip)
__device__ __forceinline__ void s_group_update(double* arr, const double* XS, int rg, int kg_lo, int kg_hi, int gq, int q) {
  if (kg_hi < kg_lo) return;
  const int r0 = rg * 8;
  const double a0 = -XS[(r0 + gq) * XLD + q], a1 = -XS[(r0 + gq) * XLD + 4 + q];
  for (int kg = kg_lo; kg <= kg_hi; kg += 4) {
    double b0[4], b1[4], c0[4], c1[4];
    double* cp[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int kgu = min(kg + u, 15);
      b0[u] = XS[(kgu * 8 + gq) * XLD + q];
      b1[u] = XS[(kgu * 8 + gq) * XLD + 4 + q];
      cp[u] = arr + (kgu * 8 + 2 * q) * PLD + r0 + gq;
      c0[u] = cp[u][0];
      c1[u] = cp[u][PLD];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a0, b0[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a1, b1[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int kgu = kg + u;
      if (kgu <= kg_hi) {
        const bool diag_tile = (kgu == rg);
        if (!diag_tile || 2 * q <= gq) cp[u][0] = c0[u];  // diagonal tile: keep only k <= row
        if (!diag_tile || 2 * q + 1 <= gq) cp[u][PLD] = c1[u];
      }
    }
  }
}

// Factor-only kernel with INTRA-KERNEL LOOK-AHEAD: after the substitution of micro-panel J, warp 0 first
// applies the rank-8 update to the next diagonal 8x8 tile only and immediately factors it (the sqrt chain of
// micro-panel J+1) while warps 1..7 run the rest of the rank-8 update on the DMMA pipe.
__global__ void __launch_bounds__(256, 1)
potrf_factor_only_f64(double* __restrict__ A, int64_t lda, double* __restrict__ logdet_part, int blk, int* __restrict__ info) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* arr = reinterpret_cast<double*>(smem_raw);
  double* XS = arr + PB * PLD;
  double* Ld = XS + PB * XLD;
  double* rinv_s = Ld + 64;
  double* dinv = rinv_s + 8;
  __shared__ double red[4];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, q = lane & 3;
#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int c = idx >> 7, i = idx & 127;
      tmp[u] = (i >= c) ? __ldg(A + i + (int64_t)c * lda) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      arr[(idx >> 7) * PLD + (idx & 127)] = tmp[u];
    }
  }
  __syncthreads();
  if (warp == 0) factor_diag8(arr, 0, lane, Ld, rinv_s, blk, info);
  __syncthreads();
  for (int j0 = 0; j0 < PB; j0 += 8) {
    const int J = j0 >> 3;
    const int w = tid;
    const bool is_s = (tid < PB) && (w >= j0 + 8);
    const bool is_diag = (tid < PB) && (w >= j0) && (w < j0 + 8);
    // ---- substitution against the (already factored) 8x8 block of this micro-panel
    if (is_s) {
      double a[8], x[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) a[c] = arr[(j0 + c) * PLD + w];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        double sacc = a[c];
#pragma unroll
        for (int c2 = 0; c2 < c; ++c2) sacc -= x[c2] * Ld[c * 8 + c2];
        x[c] = sacc * rinv_s[c];
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) { XS[w * XLD + c] = x[c]; arr[(j0 + c) * PLD + w] = x[c]; }
    } else if (is_diag) {
      const int cr = w - j0;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c <= cr) arr[(j0 + c) * PLD + w] = Ld[cr * 8 + c];
      dinv[w] = rinv_s[cr];
    }
    __syncthreads();
    // ---- rank-8 update; warp 0 runs ahead on the next diagonal block
    if (warp == 0) {
      if (J < 15) {
        s_group_update(arr, XS, J + 1, J + 1, J + 1, gq, q);  // the next diagonal 8x8 tile only
        __syncwarp();
        factor_diag8(arr, j0 + 8, lane, Ld, rinv_s, blk, info);
        if (8 > J + 1) s_group_update(arr, XS, 8, J + 1, 8, gq, q);  // then its share of the bulk: row-group 8
      }
    } else {
#pragma unroll
      for (int sel = 0; sel < 2; ++sel) {
        const int rg = sel ? (16 - warp) : warp;  // warps 1..7 own row-groups (w, 16-w): 1..7 and 9..15
        if (rg <= J + 1) continue;                // finished groups; group J+1 is only its diagonal tile (warp 0)
        s_group_update(arr, XS, rg, J + 1, rg, gq, q);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int c = idx >> 7, i = idx & 127;
      tmp[u] = (i >= c) ? arr[c * PLD + i] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      A[(idx & 127) + (int64_t)(idx >> 7) * lda] = tmp[u];
    }
  }
  double part = 0.0;
  if (tid < PB) part = -log(dinv[tid]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (tid < PB && (tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  if (tid == 0) logdet_part[blk] = red[0] + red[1] + red[2] + red[3];
}

// inverse of a factored 128x128 lower block: CTA p (of 8) produces the rows of L^-T (= columns of L^-1) of
// the row-groups p and 15-p by the same bordered elimination, reading L from global memory.
__global__ void __launch_bounds__(256, 1)
trtri_strips_f64(const double* __restrict__ A, int64_t lda, double* __restrict__ Dinv) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* arr = reinterpret_cast<double*>(smem_raw);
  double* XS = arr + PB * PLD;
  double* dinv = XS + PB * XLD;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, q = lane & 3;
  const int p = blockIdx.x;            // owns E row-groups p and 15 - p
  const int ga = p, gb = 15 - p;
#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int c = idx >> 7, i = idx & 127;
      tmp[u] = (i >= c) ? __ldg(A + i + (int64_t)c * lda) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      arr[(idx >> 7) * PLD + (idx & 127)] = tmp[u];
    }
  }
  __syncthreads();
  if (tid < PB) dinv[tid] = 1.0 / arr[tid * PLD + tid];
  __syncthreads();
  for (int j0 = ga * 8; j0 < PB; j0 += 8) {  // group ga becomes active at its own micro-panel
    const int J = j0 >> 3;
    const int w = tid;
    if (tid < PB) {
      const int rgw = w >> 3;
      if (w >= j0 + 8) {  // S row: expose its (already final) micro-panel entries as the B operand
#pragma unroll
        for (int c = 0; c < 8; ++c) XS[w * XLD + c] = arr[(j0 + c) * PLD + w];
      } else if ((rgw == ga || rgw == gb) && rgw <= J) {  // one of my E rows, already started
        double a[8], x[8];
        if (w >= j0) {
          const int cr = w - j0;
#pragma unroll
          for (int c = 0; c < 8; ++c) a[c] = (c == cr) ? 1.0 : 0.0;
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) a[c] = arr[(j0 + c) * PLD + w];
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          double sacc = a[c];
#pragma unroll
          for (int c2 = 0; c2 < c; ++c2) sacc -= x[c2] * arr[(j0 + c2) * PLD + j0 + c];  // L_d(c, c2)
          x[c] = sacc * dinv[j0 + c];
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          XS[w * XLD + c] = x[c];
          if (j0 + c > w) arr[(j0 + c) * PLD + w] = x[c];
        }
      }
    }
    __syncthreads();
    {  // E tiles: groups ga / gb (if started) x column groups J+1..15; warp wi: group by parity, 4 tiles
      const int rg = (warp & 1) ? gb : ga;
      if (rg <= J && J < 15) {
        const int r0 = rg * 8;
        const double a0 = -XS[(r0 + gq) * XLD + q], a1 = -XS[(r0 + gq) * XLD + 4 + q];
        const int kg = J + 1 + (warp >> 1);
        double b0[4], b1[4], c0[4], c1[4];
        double* cp[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int kgu = min(kg + 4 * u, 15);
          b0[u] = XS[(kgu * 8 + gq) * XLD + q];
          b1[u] = XS[(kgu * 8 + gq) * XLD + 4 + q];
          cp[u] = arr + (kgu * 8 + 2 * q) * PLD + r0 + gq;
          c0[u] = cp[u][0];
          c1[u] = cp[u][PLD];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a0, b0[u]);
#pragma unroll
        for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a1, b1[u]);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (kg + 4 * u <= 15) { cp[u][0] = c0[u]; cp[u][PLD] = c1[u]; }
        }
      }
    }
    __syncthreads();
  }
  // my 16 columns of Dinv = L^-1 (column r <-> E row r)
  for (int idx = tid; idx < 16 * PB; idx += 256) {
    const int rr = idx >> 7, c = idx & 127;
    const int r = (rr < 8) ? (ga * 8 + rr) : (gb * 8 + rr - 8);
    const double v = (c > r) ? arr[c * PLD + r] : ((c == r) ? dinv[r] : 0.0);
    Dinv[c + r * PB] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// Panel TRSM by blocked substitution (fp64): X <- X * L11^-T for a 32-row slab of the panel per CTA,
// WITHOUT the 128x128 inverse -- only the sixteen 8x8 diagonal inverses (computed here from L11 in a few
// hundred cycles).  16 micro-steps: (a) the 8 current columns are multiplied by the 8x8 inverse,
// (b) the remaining columns receive the rank-8 update on the DMMA pipe.  Takes the strip inverse
// (trtri_strips_f64) off the critical path of the factorisation: it now runs on a side stream.
// ------------------------------------------------------------------------------------------------
constexpr int TS_R = 32;        // rows per CTA
constexpr int TS_XP = TS_R + 1; // slab column stride

__global__ void __launch_bounds__(256, 1)
trsm_sub_f64(double* __restrict__ A21, int64_t lda, int64_t M, const double* __restrict__ Lkk) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* Ls = reinterpret_cast<double*>(smem_raw);  // Ls[c*PLD + i], lower
  double* xs = Ls + PB * PLD;                        // xs[c*TS_XP + r]
  double* X8 = xs + PB * TS_XP;                      // X8[r*XLD + c]
  double* D8 = X8 + TS_R * XLD;                      // D8[J*64 + c*8 + c2] = inv(L_d(J))(c, c2)
  double* dinv = D8 + 16 * 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, q = lane & 3;
  const int64_t row0 = (int64_t)blockIdx.x * TS_R;
#pragma unroll
  for (int b0 = 0; b0 < 64; b0 += 16) {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      const int c = idx >> 7, i = idx & 127;
      tmp[u] = (i >= c) ? __ldg(Lkk + i + (int64_t)c * lda) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * (b0 + u);
      Ls[(idx >> 7) * PLD + (idx & 127)] = tmp[u];
    }
  }
  {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * u;  // 128 cols x 32 rows
      const int c = idx >> 5, r = idx & 31;
      tmp[u] = (row0 + r < M) ? A21[row0 + r + (int64_t)c * lda] : 0.0;
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * u;
      xs[(idx >> 5) * TS_XP + (idx & 31)] = tmp[u];
    }
  }
  __syncthreads();
  if (tid < PB) dinv[tid] = 1.0 / Ls[tid * PLD + tid];
  __syncthreads();
  if (tid < PB) {  // sixteen 8x8 inverses: thread (J, cr) solves L_d x = e_cr
    const int J = tid >> 3, cr = tid & 7, j0 = J * 8;
    double x[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      double sacc = (c == cr) ? 1.0 : 0.0;
#pragma unroll
      for (int c2 = 0; c2 < c; ++c2) sacc -= x[c2] * Ls[(j0 + c2) * PLD + j0 + c];
      x[c] = sacc * dinv[j0 + c];
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) D8[J * 64 + c * 8 + cr] = x[c];
  }
  __syncthreads();
  for (int J = 0; J < 16; ++J) {
    const int j0 = J * 8;
    {  // (a) 8 current columns times the 8x8 inverse (transposed): thread (r, c)
      const int r = tid & 31, c = tid >> 5;
      double acc = 0.0;
#pragma unroll
      for (int c2 = 0; c2 < 8; ++c2)
        if (c2 <= c) acc = fma(xs[(j0 + c2) * TS_XP + r], D8[J * 64 + c * 8 + c2], acc);
      __syncthreads();
      xs[(j0 + c) * TS_XP + r] = acc;
      X8[r * XLD + c] = acc;
    }
    __syncthreads();
    if (J < 15) {  // (b) rank-8 update of the remaining columns: warp -> row-group (warp & 3), column parity (warp >> 2)
      const int r0 = (warp & 3) * 8;
      const double a0 = -X8[(r0 + gq) * XLD + q], a1 = -X8[(r0 + gq) * XLD + 4 + q];
      for (int kg = J + 1 + (warp >> 2); kg <= 15; kg += 8) {
        double b0[4], b1[4], c0[4], c1[4];
        double* cp[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int kgu = min(kg + 2 * u, 15);
          b0[u] = Ls[(j0 + q) * PLD + kgu * 8 + gq];
          b1[u] = Ls[(j0 + 4 + q) * PLD + kgu * 8 + gq];
          cp[u] = xs + (kgu * 8 + 2 * q) * TS_XP + r0 + gq;
          c0[u] = cp[u][0];
          c1[u] = cp[u][TS_XP];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a0, b0[u]);
#pragma unroll
        for (int u = 0; u < 4; ++u) dmma884(c0[u], c1[u], a1, b1[u]);
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (kg + 2 * u <= 15) { cp[u][0] = c0[u]; cp[u][TS_XP] = c1[u]; }
      }
    }
    __syncthreads();
  }
  {
    double tmp[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * u;
      tmp[u] = xs[(idx >> 5) * TS_XP + (idx & 31)];
    }
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int idx = tid + 256 * u;
      const int c = idx >> 5, r = idx & 31;
      if (row0 + r < M) A21[row0 + r + (int64_t)c * lda] = tmp[u];
    }
  }
}
}  // namespace

template <typename T>
void launch_potrf_diag(T* Ablk, int64_t lda, T* Dinv, double* logdet_part, int blk, int* info, cudaStream_t s) {
  const size_t smem = (size_t)(PB * PLD + PB * 8 + PB) * sizeof(T);
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  if (agp_first_use_on_device(&configured)) {
    cudaFuncSetAttribute(potrf_diag_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  potrf_diag_kernel<T><<<1, 256, smem, s>>>(Ablk, lda, Dinv, logdet_part, blk, info);
  agp_count_launch();
}
template void launch_potrf_diag<float>(float*, int64_t, float*, double*, int, int*, cudaStream_t);
template <>
void launch_potrf_diag<double>(double* Ablk, int64_t lda, double* Dinv, double* logdet_part, int blk, int* info,
                               cudaStream_t s) {
  const size_t smem = (size_t)(PB * PLD + PB * XLD + 64 + 8 + PB) * sizeof(double);
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  if (agp_first_use_on_device(&configured)) {
    cudaFuncSetAttribute(potrf_diag_kernel_f64, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  potrf_diag_kernel_f64<<<1, 256, smem, s>>>(Ablk, lda, Dinv, logdet_part, blk, info);
  agp_count_launch();
}

// ---- split API used by the factorisation schedule (fp64): factor / strip inverse / substitution TRSM
int potrf_split_enabled() {
  static int split = -1;
  if (split < 0) { const char* v = getenv("AGP_POTRF_SPLIT"); split = v ? atoi(v) : 1; }
  return split;
}
void launch_potrf_factor_f64(double* Ablk, int64_t lda, double* logdet_part, int blk, int* info, cudaStream_t s) {
  const size_t smem = (size_t)(PB * PLD + PB * XLD + 64 + 8 + PB) * sizeof(double);
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  if (agp_first_use_on_device(&configured)) { cudaFuncSetAttribute(potrf_factor_only_f64, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); }
  potrf_factor_only_f64<<<1, 256, smem, s>>>(Ablk, lda, logdet_part, blk, info);
  agp_count_launch();
}
void launch_trtri_f64(const double* Ablk, int64_t lda, double* Dinv, cudaStream_t s) {
  const size_t smem = (size_t)(PB * PLD + PB * XLD + 64 + 8 + PB) * sizeof(double);
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  if (agp_first_use_on_device(&configured)) { cudaFuncSetAttribute(trtri_strips_f64, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); }
  trtri_strips_f64<<<8, 256, smem, s>>>(Ablk, lda, Dinv);
  agp_count_launch();
}
void launch_trsm_sub_f64(double* A21, int64_t lda, int64_t M, const double* Lkk, cudaStream_t s) {
  if (M <= 0) return;
  const size_t smem = (size_t)(PB * PLD + PB * TS_XP + TS_R * XLD + 16 * 64 + PB) * sizeof(double);
  static uint64_t configured = 0;  // per-device bit: the attribute is per device (one ctx per GPU in one process)
  if (agp_first_use_on_device(&configured)) { cudaFuncSetAttribute(trsm_sub_f64, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); }
  trsm_sub_f64<<<(unsigned)((M + TS_R - 1) / TS_R), 256, smem, s>>>(A21, lda, M, Lkk);
  agp_count_launch();
}
