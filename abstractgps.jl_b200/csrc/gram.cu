// gram.cu -- K1/K2: Gram construction fused with the diagonal-noise add.
// Replaces kernelmatrix(k,x[,z]) (KernelFunctions; call sites /root/reference/src/base_gp.jl:70,74)
// and `C + f.Sigma_y` (/root/reference/src/finite_gp_projection.jl:135).
//
// Layout: points are pre-transformed once (ScaleTransform / ARDTransform) into a point-major
// array Xt[n_pad][D].  One CTA produces a 64x64 output tile; both 64 x Dc point slabs are staged
// in shared memory and each thread keeps a 4x4 register block of squared distances computed by
// DIRECT differences (no ||x||^2+||y||^2-2xy cancellation).  Stores are column-major, 16
// consecutive rows per half-warp.  Bound: HBM write of N^2/2 elements at small D, fp64 pipe at
// large D (DESIGN.md s4).
#include <atomic>
#include "kernels.h"
#include "agp.h"
#include "composite.cuh"

static std::atomic<int64_t> g_launches{0};
int64_t agp_kernel_launches() { return g_launches.load(); }
void agp_count_launch() { g_launches.fetch_add(1); }

template <typename T>
__global__ void prep_points_kernel(const T* __restrict__ X, int layout, int64_t n, int64_t n_pad, int D,
                                   int transform, T scale, const T* __restrict__ ard, T* __restrict__ Xt) {
  int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int64_t total = n_pad * D;
  if (idx >= total) return;
  int64_t i = idx / D;
  int d = (int)(idx - i * D);
  T v = 0;
  if (i < n) {
    v = (layout == AGP_POINT_MAJOR) ? X[i * D + d] : X[(int64_t)d * n + i];
    if (transform == AGP_T_SCALE) v *= scale;
    else if (transform == AGP_T_ARD) v *= ard[d];
  }
  Xt[idx] = v;
}

template <typename T>
void launch_prep_points(const T* X, int layout, int64_t n, int64_t n_pad, int D, int transform, double scale,
                        const T* ard, T* Xt, cudaStream_t s) {
  int64_t total = n_pad * D;
  if (total == 0) return;
  int threads = 256;
  int64_t blocks = (total + threads - 1) / threads;
  prep_points_kernel<T><<<(unsigned)blocks, threads, 0, s>>>(X, layout, n, n_pad, D, transform, (T)scale, ard, Xt);
  agp_count_launch();
}
template void launch_prep_points<float>(const float*, int, int64_t, int64_t, int, int, double, const float*, float*, cudaStream_t);
template void launch_prep_points<double>(const double*, int, int64_t, int64_t, int, int, double, const double*, double*, cudaStream_t);

template <typename T> __device__ __forceinline__ T dev_exp(T x);
template <> __device__ __forceinline__ float dev_exp<float>(float x) { return expf(x); }
template <> __device__ __forceinline__ double dev_exp<double>(double x) { return exp(x); }
template <typename T> __device__ __forceinline__ T dev_sqrt(T x);
template <> __device__ __forceinline__ float dev_sqrt<float>(float x) { return sqrtf(x); }
template <> __device__ __forceinline__ double dev_sqrt<double>(double x) { return sqrt(x); }

template <typename T>
__device__ __forceinline__ T kappa(int family, T acc, T variance, T linear_c) {
  // acc = squared distance (stationary families) or dot product (linear)
  switch (family) {
    case AGP_SE: return variance * dev_exp<T>(-acc * (T)0.5);
    case AGP_MATERN12: return variance * dev_exp<T>(-dev_sqrt<T>(acc));
    case AGP_MATERN32: {
      T s = (T)1.7320508075688772935 * dev_sqrt<T>(acc);
      return variance * ((T)1 + s) * dev_exp<T>(-s);
    }
    case AGP_MATERN52: {
      T s = (T)2.2360679774997896964 * dev_sqrt<T>(acc);
      return variance * ((T)1 + s + s * s * (T)(1.0 / 3.0)) * dev_exp<T>(-s);
    }
    default: return variance * (acc + linear_c);
  }
}

constexpr int GT = 64;  // gram tile
constexpr int GDC = 32; // feature chunk

template <typename T>
__global__ void __launch_bounds__(256)
gram_kernel(const T* __restrict__ Xa, const T* __restrict__ Xb, int D, T* __restrict__ K, int64_t ldk,
            GramParams p) {
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (p.lower_only && (int64_t)tj * GT + p.diag_off > (int64_t)ti * GT + (GT - 1)) return;
  __shared__ T sa[GDC][GT + 1];
  __shared__ T sb[GDC][GT + 1];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)ti * GT, col0 = (int64_t)tj * GT;
  T acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0;
  const bool linear = (p.family == AGP_LINEAR);
  for (int d0 = 0; d0 < D; d0 += GDC) {
    const int dc = min(GDC, D - d0);
    for (int idx = tid; idx < GT * GDC; idx += 256) {
      int i = idx / GDC, d = idx - i * GDC;
      T va = 0, vb = 0;
      if (d < dc) {
        va = Xa[(row0 + i) * D + d0 + d];
        vb = Xb[(col0 + i) * D + d0 + d];
      }
      sa[d][i] = va;
      sb[d][i] = vb;
    }
    __syncthreads();
    if (linear) {
#pragma unroll 4
      for (int d = 0; d < GDC; ++d) {
        T a[4], b[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) a[r] = sa[d][tx + 16 * r];
#pragma unroll
        for (int c = 0; c < 4; ++c) b[c] = sb[d][ty + 16 * c];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[r][c] += a[r] * b[c];
      }
    } else {
#pragma unroll 4
      for (int d = 0; d < GDC; ++d) {
        T a[4], b[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) a[r] = sa[d][tx + 16 * r];
#pragma unroll
        for (int c = 0; c < 4; ++c) b[c] = sb[d][ty + 16 * c];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            T df = a[r] - b[c];
            acc[r][c] += df * df;
          }
      }
    }
    __syncthreads();
  }
  const T variance = (T)p.variance, lc = (T)p.linear_c;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int64_t gj = col0 + ty + 16 * c;
    const int64_t gjg = gj + p.diag_off;  // global column index
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int64_t gi = row0 + tx + 16 * r;
      T v;
      const bool pad_a = p.mask_a ? (p.mask_a[gi] == 0) : (gi >= p.valid_a);
      const bool pad_b = p.mask_b ? (p.mask_b[gj] == 0) : (gjg >= p.valid_b);
      if (pad_a || pad_b) {
        v = (p.symmetric && gi == gjg) ? (T)1 : (T)0;  // identity padding
      } else {
        T a = acc[r][c];
        if (p.symmetric && gi == gjg && !linear) a = 0;  // exactly-zero self distance
        v = kappa<T>(p.family, a, variance, lc);
        if (p.symmetric && gi == gjg && p.noise_kind >= 0)
          v += (p.noise_kind == 0) ? (T)p.noise_s : ((const T*)p.noise_v)[gi - p.noise_off];
      }
      K[gi + gj * ldk] = v;
    }
  }
}

// ---- composite kernels: sum of product terms over UNTRANSFORMED points (each factor applies its own transform) ---------
// Same contract as gram_kernel (lower_only, identity padding, valid/mask, diag_off, noise, exact-zero self distance), but
// each thread keeps NA accumulator blocks, one per distinct distance the descriptor needs (CompositeDesc::acc_kind).  The
// per-dimension weights of every accumulator (1 for the shared raw sums, ARD v, Periodic transform weight and 1/r) are
// staged in shared memory per feature chunk beside the point slabs.  The tile is 64 x 16*CB with a 4 x CB block per
// thread: CB shrinks as NA grows so that 4 * CB * NA accumulators stay in registers.
template <int NA> struct CompCB { static constexpr int v = NA <= 2 ? 4 : (NA <= 4 ? 2 : 1); };

template <typename T, int NA, int CB>
__global__ void __launch_bounds__(256, 1)
composite_gram_kernel(const T* __restrict__ Xa, const T* __restrict__ Xb, int D, T* __restrict__ K, int64_t ldk,
                      GramParams p, const __grid_constant__ CompositeDesc cd) {
  constexpr int TC = 16 * CB;
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (p.lower_only && (int64_t)tj * TC + p.diag_off > (int64_t)ti * GT + (GT - 1)) return;
  __shared__ T sa[GDC][GT + 1];
  __shared__ T sb[GDC][TC + 1];
  __shared__ T sw[NA][GDC];
  __shared__ T sr[NA][GDC];
  const T* __restrict__ W = (const T*)cd.w;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)ti * GT, col0 = (int64_t)tj * TC;
  T acc[NA][4][CB];
#pragma unroll
  for (int a = 0; a < NA; ++a)
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < CB; ++c) acc[a][r][c] = 0;
  for (int d0 = 0; d0 < D; d0 += GDC) {
    const int dc = min(GDC, D - d0);
    for (int idx = tid; idx < GT * GDC; idx += 256) {
      const int i = idx / GDC, d = idx - i * GDC;
      sa[d][i] = (d < dc) ? Xa[(row0 + i) * D + d0 + d] : (T)0;
    }
    for (int idx = tid; idx < TC * GDC; idx += 256) {
      const int i = idx / GDC, d = idx - i * GDC;
      sb[d][i] = (d < dc) ? Xb[(col0 + i) * D + d0 + d] : (T)0;
    }
    for (int idx = tid; idx < NA * GDC; idx += 256) {
      const int a = idx / GDC, d = idx - a * GDC;
      sw[a][d] = (d < dc) ? W[(int64_t)(2 * a) * D + d0 + d] : (T)0;
      sr[a][d] = (d < dc) ? W[(int64_t)(2 * a + 1) * D + d0 + d] : (T)0;
    }
    __syncthreads();
#pragma unroll 1
    for (int d = 0; d < dc; ++d) {
      T xa[4], xb[CB];
#pragma unroll
      for (int r = 0; r < 4; ++r) xa[r] = sa[d][tx + 16 * r];
#pragma unroll
      for (int c = 0; c < CB; ++c) xb[c] = sb[d][ty + 16 * c];
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        const int kind = cd.acc_kind[a];
        const T w = sw[a][d];
        if (kind == COMP_ACC_SQ) {
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < CB; ++c) {
              const T df = w * (xa[r] - xb[c]);
              acc[a][r][c] += df * df;
            }
        } else if (kind == COMP_ACC_DOT) {
          const T ww = w * w;
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < CB; ++c) acc[a][r][c] += ww * xa[r] * xb[c];
        } else {  // COMP_ACC_PER
          const T ri = sr[a][d];
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < CB; ++c) {
              const T sn = comp_sinpi<T>(w * (xa[r] - xb[c])) * ri;
              acc[a][r][c] += sn * sn;
            }
        }
      }
    }
    __syncthreads();
  }
  // one element at a time: the factor evaluation is inlined once, not 4 * CB times (register pressure)
#pragma unroll 1
  for (int e = 0; e < 4 * CB; ++e) {
    const int r = e & 3, c = e >> 2;
    const int64_t gj = col0 + ty + 16 * c;
    const int64_t gjg = gj + p.diag_off;
    {
      const int64_t gi = row0 + tx + 16 * r;
      T v;
      const bool pad_a = p.mask_a ? (p.mask_a[gi] == 0) : (gi >= p.valid_a);
      const bool pad_b = p.mask_b ? (p.mask_b[gj] == 0) : (gjg >= p.valid_b);
      if (pad_a || pad_b) {
        v = (p.symmetric && gi == gjg) ? (T)1 : (T)0;
      } else {
        const bool self = p.symmetric && gi == gjg;
        T x[NA];
#pragma unroll
        for (int a = 0; a < NA; ++a) {
          T y = acc[a][0][0];
#pragma unroll
          for (int q = 1; q < 4 * CB; ++q)
            if (q == e) y = acc[a][q & 3][q >> 2];
          x[a] = (self && cd.acc_kind[a] != COMP_ACC_DOT) ? (T)0 : y;
        }
        v = comp_eval<T, NA>(cd, x);
        if (self && p.noise_kind >= 0)
          v += (p.noise_kind == 0) ? (T)p.noise_s : ((const T*)p.noise_v)[gi - p.noise_off];
      }
      K[gi + gj * ldk] = v;
    }
  }
}

template <typename T, int NA>
static void launch_composite_gram_na(const T* Xa, const T* Xb, int64_t na_pad, int64_t nb_pad, int D, T* K, int64_t ldk,
                                     const GramParams& p, cudaStream_t s) {
  constexpr int CB = CompCB<NA>::v;
  dim3 grid((unsigned)(na_pad / GT), (unsigned)(nb_pad / (16 * CB)));
  composite_gram_kernel<T, NA, CB><<<grid, 256, 0, s>>>(Xa, Xb, D, K, ldk, p, *p.comp);
  agp_count_launch();
}

template <typename T>
static void launch_composite_gram(const T* Xa, const T* Xb, int64_t na_pad, int64_t nb_pad, int D, T* K, int64_t ldk,
                                  const GramParams& p, cudaStream_t s) {
  switch (p.comp->nacc) {
    case 1: launch_composite_gram_na<T, 1>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
    case 2: launch_composite_gram_na<T, 2>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
    case 3: launch_composite_gram_na<T, 3>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
    case 4: launch_composite_gram_na<T, 4>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
    case 5: launch_composite_gram_na<T, 5>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
    case 6: launch_composite_gram_na<T, 6>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
    case 7: launch_composite_gram_na<T, 7>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
    default: launch_composite_gram_na<T, 8>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); break;
  }
}

template <typename T>
void launch_gram(const T* Xa, const T* Xb, int64_t na_pad, int64_t nb_pad, int D, T* K, int64_t ldk,
                 const GramParams& p, cudaStream_t s) {
  if (na_pad == 0 || nb_pad == 0) return;
  if (p.family == AGP_COMPOSITE) { launch_composite_gram<T>(Xa, Xb, na_pad, nb_pad, D, K, ldk, p, s); return; }
  dim3 grid((unsigned)(na_pad / GT), (unsigned)(nb_pad / GT));
  gram_kernel<T><<<grid, 256, 0, s>>>(Xa, Xb, D, K, ldk, p);
  agp_count_launch();
}
template void launch_gram<float>(const float*, const float*, int64_t, int64_t, int, float*, int64_t, const GramParams&, cudaStream_t);
template void launch_gram<double>(const double*, const double*, int64_t, int64_t, int, double*, int64_t, const GramParams&, cudaStream_t);

// kernelmatrix_diag (/root/reference/src/base_gp.jl:72)
template <typename T>
__global__ void kdiag_kernel(const T* __restrict__ Xt, int64_t n, int D, int family, T variance, T linear_c,
                             T* __restrict__ out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (family != AGP_LINEAR) { out[i] = variance; return; }
  T acc = 0;
  for (int d = 0; d < D; ++d) { T v = Xt[i * D + d]; acc += v * v; }
  out[i] = variance * (acc + linear_c);
}
// composite diagonal sum_t v_t prod_f kappa_f(x, x): stationary, RQ, Periodic and White factors give 1, Constant c, Linear
// |x~|^2 + c -- only the DOT accumulators are non-zero
template <typename T>
__global__ void composite_kdiag_kernel(const T* __restrict__ Xt, int64_t n, int D, const __grid_constant__ CompositeDesc cd,
                                       T* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T* __restrict__ W = (const T*)cd.w;
  T v[AGP_COMP_MAX];
#pragma unroll
  for (int a = 0; a < AGP_COMP_MAX; ++a) {
    v[a] = 0;
    if (a < cd.nacc && cd.acc_kind[a] == COMP_ACC_DOT)
      for (int d = 0; d < D; ++d) {
        const T w = W[(int64_t)(2 * a) * D + d], x = Xt[i * D + d];
        v[a] += w * w * x * x;
      }
  }
  out[i] = comp_eval<T, AGP_COMP_MAX>(cd, v);
}

template <typename T>
void launch_kdiag(const T* Xt, int64_t n, int D, int family, double variance, double linear_c, T* out,
                  cudaStream_t s, const CompositeDesc* comp) {
  if (n == 0) return;
  if (family == AGP_COMPOSITE) {
    composite_kdiag_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(Xt, n, D, *comp, out);
    agp_count_launch();
    return;
  }
  kdiag_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(Xt, n, D, family, (T)variance, (T)linear_c, out);
  agp_count_launch();
}
template void launch_kdiag<float>(const float*, int64_t, int, int, double, double, float*, cudaStream_t,
                                  const CompositeDesc*);
template void launch_kdiag<double>(const double*, int64_t, int, int, double, double, double*, cudaStream_t,
                                   const CompositeDesc*);
