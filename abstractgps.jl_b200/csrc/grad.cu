// grad.cu -- EXPERIMENTAL (compiles, NOT yet run on a device): the fused reduction of the logpdf gradient,
//   dL/dtheta = 1/2 sum_ij W_ij dC_ij/dtheta,   W = alpha alpha' - C^-1,
// what Zygote produces through the reference for `logpdf(f(x, s2), y)` (/root/reference/test/finite_gp_projection.jl:152-178,
// /root/reference/examples/1-mauna-loa/script.jl:200-242; SURVEY s8f rank 1).
//
// One CTA per 64x64 tile of the LOWER triangle (same tiling and the same direct-difference distances as gram_kernel):
// the tile's kappa and kappa'(r) r are recomputed from the transformed points, W_ij is read once from the C^-1 buffer
// (N^2/2 elements -- the kernel is bound by that read at small D and by the fp64 pipe at D = 64), off-diagonal elements
// count twice.  All sums are accumulated in fp64 whatever T is.  Scalars leave the CTA through one atomicAdd each;
// the ARD pass re-stages the point slabs and reduces one feature at a time.
//
// sums[0] = sum w kappa                (-> d/d variance  = 1/2 sums[0])
// sums[1] = sum w kappa'(r) r  |  sum w <tx, tx'>  (linear)   (-> d/d scale)
// sums[2] = sum w                      (linear only: d/d c)
// sums[3] = sum_i W_ii                 (-> d/d sigma^2 = 1/2 sums[3]; per-point: noise_diag[i] = 1/2 W_ii)
// sums[4] = sum_i alpha_i              (-> d/d mean constant)
// sums[5 + d] = sum w q tdiff_d^2  |  sum w tx_d tx'_d  (linear)        (-> d/d ard_d)
#include "kernels.h"
#include "agp.h"
#include "composite.cuh"

namespace {

constexpr int RT = 64;   // tile
constexpr int RDC = 32;  // feature chunk

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// kappa(d2) and kappa'(r) r without the variance, fp64
__device__ __forceinline__ void kappa_pair(int family, double d2, double& kap, double& kr) {
  switch (family) {
    case AGP_SE: {
      const double e = exp(-0.5 * d2);
      kap = e; kr = -d2 * e;
      break;
    }
    case AGP_MATERN12: {
      const double d = sqrt(d2), e = exp(-d);
      kap = e; kr = -d * e;
      break;
    }
    case AGP_MATERN32: {
      const double s = 1.7320508075688772935 * sqrt(d2), e = exp(-s);
      kap = (1.0 + s) * e; kr = -3.0 * d2 * e;
      break;
    }
    default: {  // AGP_MATERN52
      const double s = 2.2360679774997896964 * sqrt(d2), e = exp(-s);
      kap = (1.0 + s + s * s * (1.0 / 3.0)) * e; kr = -(5.0 / 3.0) * d2 * (1.0 + s) * e;
      break;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
grad_reduce_kernel(const T* __restrict__ Xt, int D, int64_t n, const T* __restrict__ Cinv, int64_t ldc,
                   const T* __restrict__ alpha, int family, double linear_c, int want_ard,
                   double* __restrict__ sums, T* __restrict__ noise_diag) {
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (tj > ti) return;
  __shared__ T sa[RDC][RT + 1];
  __shared__ T sb[RDC][RT + 1];
  __shared__ double red[8][5];
  __shared__ double sard[RDC];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)ti * RT, col0 = (int64_t)tj * RT;
  const bool linear = (family == AGP_LINEAR);
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
  for (int d0 = 0; d0 < D; d0 += RDC) {
    const int dc = min(RDC, D - d0);
    for (int idx = tid; idx < RT * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      T va = 0, vb = 0;
      if (d < dc) {
        va = Xt[(row0 + i) * D + d0 + d];
        vb = Xt[(col0 + i) * D + d0 + d];
      }
      sa[d][i] = va;
      sb[d][i] = vb;
    }
    __syncthreads();
#pragma unroll 4
    for (int d = 0; d < RDC; ++d) {
      double a[4], b[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = (double)sa[d][tx + 16 * r];
#pragma unroll
      for (int c = 0; c < 4; ++c) b[c] = (double)sb[d][ty + 16 * c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if (linear) acc[r][c] += a[r] * b[c];
          else { const double df = a[r] - b[c]; acc[r][c] += df * df; }
        }
    }
    __syncthreads();
  }
  // per-element weights; wq = weight of the element in the ARD sums
  double wq[4][4];
  double s_var = 0.0, s_scale = 0.0, s_c = 0.0, s_noise = 0.0, s_alpha = 0.0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int64_t gj = col0 + ty + 16 * c;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int64_t gi = row0 + tx + 16 * r;
      wq[r][c] = 0.0;
      if (gi >= n || gj >= n || gj > gi) continue;
      const double ai = (double)alpha[gi], aj = (double)alpha[gj];
      const double w = ai * aj - (double)Cinv[gi + gj * ldc];
      const double mult = (gi == gj) ? 1.0 : 2.0;
      if (gi == gj) {
        s_noise += w;
        s_alpha += ai;
        if (noise_diag) noise_diag[gi] = (T)(0.5 * w);
      }
      if (linear) {
        s_var += mult * w * (acc[r][c] + linear_c);
        s_scale += mult * w * acc[r][c];
        s_c += mult * w;
        wq[r][c] = mult * w;
      } else {
        const double d2 = (gi == gj) ? 0.0 : acc[r][c];
        double kap, kr;
        kappa_pair(family, d2, kap, kr);
        s_var += mult * w * kap;
        s_scale += mult * w * kr;
        wq[r][c] = (d2 > 0.0) ? mult * w * kr / d2 : 0.0;
      }
    }
  }
  // block reduction of the five scalars
  {
    double v[5] = {s_var, s_scale, s_c, s_noise, s_alpha};
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const double t = warp_sum_d(v[q]);
      if (lane == 0) red[wid][q] = t;
    }
    __syncthreads();
    if (tid < 5) {
      double t = 0.0;
      for (int w8 = 0; w8 < 8; ++w8) t += red[w8][tid];
      atomicAdd(&sums[tid], t);
    }
  }
  if (!want_ard) return;
  // ARD pass: one feature at a time, sum_ij wq_ij * (tdiff_d)^2   (linear: wq_ij * tx_d * tx'_d)
  for (int d0 = 0; d0 < D; d0 += RDC) {
    const int dc = min(RDC, D - d0);
    __syncthreads();
    for (int idx = tid; idx < RT * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      T va = 0, vb = 0;
      if (d < dc) {
        va = Xt[(row0 + i) * D + d0 + d];
        vb = Xt[(col0 + i) * D + d0 + d];
      }
      sa[d][i] = va;
      sb[d][i] = vb;
    }
    if (tid < RDC) sard[tid] = 0.0;
    __syncthreads();
    for (int d = 0; d < dc; ++d) {
      double a[4], b[4], part = 0.0;
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = (double)sa[d][tx + 16 * r];
#pragma unroll
      for (int c = 0; c < 4; ++c) b[c] = (double)sb[d][ty + 16 * c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          if (linear) part += wq[r][c] * a[r] * b[c];
          else { const double df = a[r] - b[c]; part += wq[r][c] * df * df; }
        }
      part = warp_sum_d(part);
      if (lane == 0) atomicAdd(&sard[d], part);
    }
    __syncthreads();
    if (tid < dc) atomicAdd(&sums[5 + d0 + tid], sard[tid]);
  }
}

// ---- composite kernels ---------------------------------------------------------------------------------------------
// (comp_factor_grad, comp_all_kappa and comp_other, the factor evaluation in fp64, are in composite.cuh)

// does factor F have per-dimension parameters (ARD v of a distance / Linear factor, or Periodic r)?
__device__ __forceinline__ bool comp_perdim(const CompFactor& F) {
  if (F.family == AGP_PERIODIC) return true;
  return F.transform == AGP_T_ARD && F.family != AGP_WHITE && F.family != AGP_CONSTANT;
}

// The tiling of composite_gram_kernel over the lower triangle: a 64 x 16*CB tile, 4 x CB elements per thread, fp64
// accumulators.  Per element: every factor's kappa and derivative pieces, the term products and, by the product rule
// without dividing by any kappa, v_t prod_{g != f} kappa_g for each factor.  Scalar partials (8 variances, 8 scale and
// 8 parameter slots, the noise trace and sum alpha) leave the CTA through one atomic each; each factor with
// per-dimension parameters then takes its own pass over the feature chunks, like grad_reduce_kernel's ARD pass.
template <int NA> struct CompGradCB { static constexpr int v = NA <= 2 ? 2 : 1; };

template <typename T, int NA, int CB>
__global__ void __launch_bounds__(256, 1)
composite_grad_reduce_kernel(const T* __restrict__ Xt, int D, int64_t n, const T* __restrict__ Cinv, int64_t ldc,
                             const T* __restrict__ alpha, const __grid_constant__ CompositeDesc cd,
                             double* __restrict__ sums, T* __restrict__ noise_diag) {
  constexpr int TC = 16 * CB;
  constexpr int NS = 3 * AGP_COMP_MAX + 2;  // variances, scale slots, parameter slots, noise, alpha
  const int ti = blockIdx.x, tj = blockIdx.y;
  const int64_t row0 = (int64_t)ti * RT, col0 = (int64_t)tj * TC;
  if (col0 > row0 + RT - 1) return;
  __shared__ T sa[RDC][RT + 1];
  __shared__ T sb[RDC][TC + 1];
  __shared__ double sw[NA][RDC];
  __shared__ double sr[NA][RDC];
  __shared__ double red[8][NS];
  __shared__ double sard[2][RDC];
  const T* __restrict__ Wt = (const T*)cd.w;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  double acc[NA][4][CB];
#pragma unroll
  for (int a = 0; a < NA; ++a)
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < CB; ++c) acc[a][r][c] = 0.0;
  for (int d0 = 0; d0 < D; d0 += RDC) {
    const int dc = min(RDC, D - d0);
    for (int idx = tid; idx < RT * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      sa[d][i] = (d < dc) ? Xt[(row0 + i) * D + d0 + d] : (T)0;
    }
    for (int idx = tid; idx < TC * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      sb[d][i] = (d < dc) ? Xt[(col0 + i) * D + d0 + d] : (T)0;
    }
    for (int idx = tid; idx < NA * RDC; idx += 256) {
      const int a = idx / RDC, d = idx - a * RDC;
      sw[a][d] = (d < dc) ? (double)Wt[(int64_t)(2 * a) * D + d0 + d] : 0.0;
      sr[a][d] = (d < dc) ? (double)Wt[(int64_t)(2 * a + 1) * D + d0 + d] : 0.0;
    }
    __syncthreads();
#pragma unroll 1
    for (int d = 0; d < dc; ++d) {
      double xa[4], xb[CB];
#pragma unroll
      for (int r = 0; r < 4; ++r) xa[r] = (double)sa[d][tx + 16 * r];
#pragma unroll
      for (int c = 0; c < CB; ++c) xb[c] = (double)sb[d][ty + 16 * c];
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        const int kind = cd.acc_kind[a];
        const double w = sw[a][d];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < CB; ++c) {
            double t;
            if (kind == COMP_ACC_SQ) t = w * (xa[r] - xb[c]);
            else if (kind == COMP_ACC_DOT) t = w * w * xa[r] * xb[c];
            else t = sinpi(w * (xa[r] - xb[c])) * sr[a][d];
            acc[a][r][c] += (kind == COMP_ACC_DOT) ? t : t * t;
          }
      }
    }
    __syncthreads();
  }
  // element weights w = mult * (alpha_i alpha_j - Cinv_ij), 0 outside the lower triangle / padding
  double wq[4][CB];
  double part[NS];
#pragma unroll
  for (int q = 0; q < NS; ++q) part[q] = 0.0;
#pragma unroll 1
  for (int e = 0; e < 4 * CB; ++e) {
    const int r = e & 3, c = e >> 2;
    const int64_t gi = row0 + tx + 16 * r, gj = col0 + ty + 16 * c;
    double w = 0.0;
    if (gi < n && gj < n && gj <= gi) {
      const double ai = (double)alpha[gi], aj = (double)alpha[gj];
      w = ai * aj - (double)Cinv[gi + gj * ldc];
      if (gi == gj) {
        part[NS - 2] += w;
        part[NS - 1] += ai;
        if (noise_diag) noise_diag[gi] = (T)(0.5 * w);
      } else {
        w *= 2.0;
      }
    }
#pragma unroll
    for (int q = 0; q < 4 * CB; ++q)
      if (q == e) wq[q & 3][q >> 2] = w;
    if (w == 0.0) continue;
    double x[NA];
#pragma unroll
    for (int a = 0; a < NA; ++a) {
      double y = acc[a][0][0];
#pragma unroll
      for (int q = 1; q < 4 * CB; ++q)
        if (q == e) y = acc[a][q & 3][q >> 2];
      x[a] = (gi == gj && cd.acc_kind[a] != COMP_ACC_DOT) ? 0.0 : y;
    }
    double kap[AGP_COMP_MAX];
    comp_all_kappa<NA>(cd, x, kap);
#pragma unroll
    for (int t = 0; t < AGP_COMP_MAX; ++t) {
      double pt = 1.0;
#pragma unroll
      for (int g = 0; g < AGP_COMP_MAX; ++g)
        if (g < cd.nfactors && cd.f[g].term == t) pt *= kap[g];
      part[t] += w * pt;
    }
#pragma unroll
    for (int f = 0; f < AGP_COMP_MAX; ++f) {
      if (f >= cd.nfactors) continue;
      double k_, ds, dp, q;  // the derivative pieces are recomputed here rather than kept for every factor (registers)
      comp_factor_grad(cd.f[f], comp_pick<double, NA>(x, cd.f[f].acc), k_, ds, dp, q);
      const double o = w * comp_other(cd, kap, f);
      part[AGP_COMP_MAX + f] += o * ds;
      part[2 * AGP_COMP_MAX + f] += o * dp;
    }
  }
#pragma unroll
  for (int q = 0; q < NS; ++q) {
    const double t = warp_sum_d(part[q]);
    if (lane == 0) red[wid][q] = t;
  }
  __syncthreads();
  if (tid < NS) {
    double t = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) t += red[w8][tid];
    int slot = -1;
    if (tid < AGP_COMP_MAX) slot = tid < cd.nterms ? cd.g_var[tid] : -1;
    else if (tid < 2 * AGP_COMP_MAX) slot = tid - AGP_COMP_MAX < cd.nfactors ? cd.f[tid - AGP_COMP_MAX].g_s : -1;
    else if (tid < 3 * AGP_COMP_MAX) slot = tid - 2 * AGP_COMP_MAX < cd.nfactors ? cd.f[tid - 2 * AGP_COMP_MAX].g_p : -1;
    else slot = tid == NS - 2 ? 3 : 4;
    if (slot >= 0) atomicAdd(&sums[slot], t);
  }
  // per-dimension passes, one per factor with ARD v or Periodic r
#pragma unroll 1
  for (int f = 0; f < cd.nfactors; ++f) {
    const CompFactor& F = cd.f[f];
    if (!comp_perdim(F)) continue;
    const bool per = F.family == AGP_PERIODIC, lin = F.family == AGP_LINEAR;
    // coefficient of the element: w v_t prod_{g != f} kappa_g times q (distance ARD) / kappa (Periodic) / 1 (Linear)
    double coef[4][CB];
#pragma unroll 1
    for (int e = 0; e < 4 * CB; ++e) {
      const int r = e & 3, c = e >> 2;
      const int64_t gi = row0 + tx + 16 * r;
      double w = wq[0][0];
#pragma unroll
      for (int q = 1; q < 4 * CB; ++q)
        if (q == e) w = wq[q & 3][q >> 2];
      double cf = 0.0;
      if (w != 0.0) {
        const int64_t gj = col0 + ty + 16 * c;
        double x[NA];
#pragma unroll
        for (int a = 0; a < NA; ++a) {
          double y = acc[a][0][0];
#pragma unroll
          for (int q = 1; q < 4 * CB; ++q)
            if (q == e) y = acc[a][q & 3][q >> 2];
          x[a] = (gi == gj && cd.acc_kind[a] != COMP_ACC_DOT) ? 0.0 : y;
        }
        double kap[AGP_COMP_MAX];
        comp_all_kappa<NA>(cd, x, kap);
        double k_, ds, dp, qf;
        comp_factor_grad(F, comp_pick<double, NA>(x, F.acc), k_, ds, dp, qf);
        cf = w * comp_other(cd, kap, f) * (lin ? 1.0 : qf);
      }
#pragma unroll
      for (int q = 0; q < 4 * CB; ++q)
        if (q == e) coef[q & 3][q >> 2] = cf;
    }
    const int a = F.acc;
    for (int d0 = 0; d0 < D; d0 += RDC) {
      const int dc = min(RDC, D - d0);
      __syncthreads();
      for (int idx = tid; idx < RT * RDC; idx += 256) {
        const int i = idx / RDC, d = idx - i * RDC;
        sa[d][i] = (d < dc) ? Xt[(row0 + i) * D + d0 + d] : (T)0;
      }
      for (int idx = tid; idx < TC * RDC; idx += 256) {
        const int i = idx / RDC, d = idx - i * RDC;
        sb[d][i] = (d < dc) ? Xt[(col0 + i) * D + d0 + d] : (T)0;
      }
      if (tid < RDC) {
        sw[0][tid] = (tid < dc) ? (double)Wt[(int64_t)(2 * a) * D + d0 + tid] : 0.0;
        sr[0][tid] = (tid < dc) ? (double)Wt[(int64_t)(2 * a + 1) * D + d0 + tid] : 0.0;
        sard[0][tid] = 0.0;
        sard[1][tid] = 0.0;
      }
      __syncthreads();
      for (int d = 0; d < dc; ++d) {
        const double wd = sw[0][d], ri = sr[0][d];
        double p0 = 0.0, p1 = 0.0;  // p0: d/d transform weight, p1: d/d r (Periodic)
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < CB; ++c) {
            const double xa = (double)sa[d][tx + 16 * r], xb = (double)sb[d][ty + 16 * c], df = xa - xb;
            if (per) {
              double sn, cs;
              sincospi(wd * df, &sn, &cs);
              const double sr_ = sn * ri;
              p1 += coef[r][c] * sr_ * sr_ * ri;
              p0 -= coef[r][c] * 3.14159265358979323846 * df * sn * cs * ri * ri;
            } else if (lin) {
              p0 += coef[r][c] * 2.0 * wd * xa * xb;
            } else {
              p0 += coef[r][c] * wd * df * df;
            }
          }
        p0 = warp_sum_d(p0);
        p1 = warp_sum_d(p1);
        if (lane == 0) { atomicAdd(&sard[0][d], p0); atomicAdd(&sard[1][d], p1); }
      }
      __syncthreads();
      if (tid < dc) {
        if (F.transform == AGP_T_ARD) atomicAdd(&sums[F.g_w + d0 + tid], sard[0][tid]);
        else if (F.transform == AGP_T_SCALE && per) atomicAdd(&sums[F.g_s], sard[0][tid]);
        if (per) atomicAdd(&sums[F.g_r + d0 + tid], sard[1][tid]);
      }
    }
  }
}

template <typename T, int NA>
void launch_composite_grad_na(const T* Xt, int D, int64_t n, int64_t n_pad, const T* Cinv, int64_t ldc, const T* alpha,
                              const CompositeDesc& cd, double* sums, T* noise_diag, cudaStream_t s) {
  constexpr int CB = CompGradCB<NA>::v;
  dim3 grid((unsigned)(n_pad / RT), (unsigned)(n_pad / (16 * CB)));
  composite_grad_reduce_kernel<T, NA, CB><<<grid, 256, 0, s>>>(Xt, D, n, Cinv, ldc, alpha, cd, sums, noise_diag);
  agp_count_launch();
}

}  // namespace

template <typename T>
void launch_composite_grad_reduce(const T* Xt, int D, int64_t n, int64_t n_pad, const T* Cinv, int64_t ldc, const T* alpha,
                                  const CompositeDesc& cd, double* sums, T* noise_diag, cudaStream_t s) {
  if (n_pad <= 0) return;
  switch (cd.nacc) {
    case 1: launch_composite_grad_na<T, 1>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
    case 2: launch_composite_grad_na<T, 2>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
    case 3: launch_composite_grad_na<T, 3>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
    case 4: launch_composite_grad_na<T, 4>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
    case 5: launch_composite_grad_na<T, 5>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
    case 6: launch_composite_grad_na<T, 6>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
    case 7: launch_composite_grad_na<T, 7>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
    default: launch_composite_grad_na<T, 8>(Xt, D, n, n_pad, Cinv, ldc, alpha, cd, sums, noise_diag, s); break;
  }
}
template void launch_composite_grad_reduce<float>(const float*, int, int64_t, int64_t, const float*, int64_t, const float*,
                                                  const CompositeDesc&, double*, float*, cudaStream_t);
template void launch_composite_grad_reduce<double>(const double*, int, int64_t, int64_t, const double*, int64_t, const double*,
                                                   const CompositeDesc&, double*, double*, cudaStream_t);

template <typename T>
void launch_grad_reduce(const T* Xt, int D, int64_t n, int64_t n_pad, const T* Cinv, int64_t ldc, const T* alpha,
                        int family, double linear_c, int want_ard, double* sums, T* noise_diag, cudaStream_t s) {
  if (n_pad <= 0) return;
  const unsigned nt = (unsigned)(n_pad / RT);
  dim3 grid(nt, nt);
  grad_reduce_kernel<T><<<grid, 256, 0, s>>>(Xt, D, n, Cinv, ldc, alpha, family, linear_c, want_ard, sums, noise_diag);
  agp_count_launch();
}
template void launch_grad_reduce<float>(const float*, int, int64_t, int64_t, const float*, int64_t, const float*, int, double,
                                        int, double*, float*, cudaStream_t);
template void launch_grad_reduce<double>(const double*, int, int64_t, int64_t, const double*, int64_t, const double*, int,
                                         double, int, double*, double*, cudaStream_t);
