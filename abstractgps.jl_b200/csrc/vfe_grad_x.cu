// vfe_grad_x.cu -- the gradient of the VFE objectives with respect to the training inputs (agp.h agp_vfe_elbo_grad_x).
// With W = Kbar_zx[m, n] = G / s_n + r_m delta_n s_n^-1/2 (vfe_grad.cu), t the Scale s, the ARD v or 1 and x~ = t x:
//   stationary  xbar[n, d] = -sigma^2 t_d (sum_m cz z~_md - x~_nd sum_m cz),   cz = W kappa'(r) r / d2  (0 where d2 == 0)
//   Linear      xbar[n, d] =  sigma^2 t_d (sum_m W z~_md - c x~_nd / s_n)      (the second term is the kdiag term)
// with c = 1 for the elbo and 0 for DTC (kdiagbar_n = -c / (2 s_n)).
// That is a sum over the inducing points of each data column, the transpose of the reduction vfe_cross_grad_kernel does
// per row block, so it runs in its own pass over the chunk while G = R K_zx,c is still in its buffer:
//   vfe_x_grad_kernel   a CTA owns 64 data points of the chunk and sweeps a fixed range of 64-row tiles of inducing
//                       points; per element it recomputes W and the distance (dot product) from the transformed points
//                       and accumulates, in fp64, sum_m cz z~_md and sum_m cz (sum_m W z~_md for Linear) into its own
//                       slot of the workspace (row range x (D + 1) x points; no atomics);
//   vfe_x_finish_kernel adds the row ranges in a fixed order, applies sigma^2, the chain factor t_d and the kdiag term, and
//                       writes the caller's layout at the chunk's offset.
// Two calls give the same bits; a different chunking changes only the rounding.
#include "kernels.h"
#include "agp.h"

namespace {

constexpr int XR = 64;           // rows (inducing points) per tile
constexpr int XC = 64;           // columns (data points) per CTA
constexpr int XDC = 16;          // feature chunk
constexpr int X_CTA_TARGET = 264;  // column blocks x row ranges aimed at (two CTAs per SM of a 132-SM H100)
constexpr int X_MAX_SPLIT = 64;

// kappa'(r) r / d2 without the variance (d2 > 0); vfe_grad.cu's kappa_pair with kr divided by d2
__device__ __forceinline__ double kr_over_d2(int family, double d2) {
  switch (family) {
    case AGP_SE: return -exp(-0.5 * d2);
    case AGP_MATERN12: { const double d = sqrt(d2); return -exp(-d) / d; }
    case AGP_MATERN32: return -3.0 * exp(-1.7320508075688772935 * sqrt(d2));
    default: { const double s = 2.2360679774997896964 * sqrt(d2); return -(5.0 / 3.0) * (1.0 + s) * exp(-s); }
  }
}

template <typename T, bool LIN>
__global__ void __launch_bounds__(256)
vfe_x_grad_kernel(const T* __restrict__ Zt, int64_t M, const T* __restrict__ Xc, int64_t nc, int D,
                  const T* __restrict__ G, int64_t ldg, const T* __restrict__ r, const T* __restrict__ delta,
                  const T* __restrict__ isn, int family, int ntiles, int nsplit, double* __restrict__ xpart, int64_t ldx) {
  const int cb = blockIdx.x, sp = blockIdx.y;
  const int t0 = (int)((int64_t)ntiles * sp / nsplit), t1 = (int)((int64_t)ntiles * (sp + 1) / nsplit);
  const int64_t col0 = (int64_t)cb * XC;
  __shared__ T sa[XDC][XR];
  // the column features during the distance pass, the per-element coefficients after it
  __shared__ double sbuf[XR * (XC + 1)];
  T(*sb)[XC + 1] = reinterpret_cast<T(*)[XC + 1]>(sbuf);
  double(*sc)[XC + 1] = reinterpret_cast<double(*)[XC + 1]>(sbuf);
  __shared__ double srow[XR];
  __shared__ double scol[2][XC];  // delta s^-1/2 and 1/s of the columns
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int ci = tid & 63, cg = tid >> 6;  // per-dimension pass: column, dimension group
  if (tid < XC) {
    const int64_t gj = col0 + tid;
    const double is = gj < nc ? (double)isn[gj] : 0.0;
    scol[0][tid] = gj < nc ? (double)delta[gj] * is : 0.0;
    scol[1][tid] = is * is;
  }
  // slot (sp, d) of column col0 + ci; the first tile of the range writes it, the others add to it
  auto slot = [&](int d) -> double& { return xpart[((int64_t)sp * (D + 1) + d) * ldx + col0 + ci]; };

#pragma unroll 1
  for (int tile = t0; tile < t1; ++tile) {
    const int64_t row0 = (int64_t)tile * XR;
    double acc[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) acc[q][p] = 0.0;
    for (int d0 = 0; d0 < D; d0 += XDC) {
      const int dc = min(XDC, D - d0);
      __syncthreads();
      for (int idx = tid; idx < XR * XDC; idx += 256) {
        const int i = idx / XDC, d = idx - i * XDC;
        sa[d][i] = (d < dc && row0 + i < M) ? Zt[(row0 + i) * D + d0 + d] : (T)0;
        sb[d][i] = (d < dc && col0 + i < nc) ? Xc[(col0 + i) * D + d0 + d] : (T)0;
      }
      __syncthreads();
#pragma unroll 1
      for (int d = 0; d < dc; ++d) {
        double a[4], b[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) { a[q] = (double)sa[d][tx + 16 * q]; b[q] = (double)sb[d][ty + 16 * q]; }
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            if (LIN) acc[q][p] += a[q] * b[p];
            else { const double df = a[q] - b[p]; acc[q][p] += df * df; }
          }
      }
    }
    if (tid < XR) srow[tid] = row0 + tid < M ? (double)r[row0 + tid] : 0.0;
    __syncthreads();  // sb is dead from here: sc takes its place
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int i = tx + 16 * q, j = ty + 16 * p;
        const int64_t gi = row0 + i, gj = col0 + j;
        double cz = 0.0;
        if (gi < M && gj < nc) {
          const double W = (double)G[gi + gj * ldg] * scol[1][j] + srow[i] * scol[0][j];
          if (LIN) cz = W;
          else if (acc[q][p] > 0.0) cz = W * kr_over_d2(family, acc[q][p]);
        }
        sc[i][j] = cz;
      }
    __syncthreads();
    const bool first = tile == t0, own = col0 + ci < nc;
    if (!LIN && cg == 0 && own) {  // sum_m cz, in a fixed order
      double t = 0.0;
      for (int i = 0; i < XR; ++i) t += sc[i][ci];
      double& o = slot(D);
      o = first ? t : o + t;
    }
    // per-dimension pass: thread (column ci, group cg) owns dimensions cg, cg + 4, ... of each chunk
    for (int d0 = 0; d0 < D; d0 += XDC) {
      const int dc = min(XDC, D - d0);
      if (d0 > 0) __syncthreads();
      for (int idx = tid; idx < XR * XDC; idx += 256) {
        const int i = idx / XDC, d = idx - i * XDC;
        sa[d][i] = (d < dc && row0 + i < M) ? Zt[(row0 + i) * D + d0 + d] : (T)0;
      }
      __syncthreads();
      double res[XDC / 4];
#pragma unroll
      for (int k = 0; k < XDC / 4; ++k) res[k] = 0.0;
#pragma unroll 4
      for (int i = 0; i < XR; ++i) {
        const double c = sc[i][ci];
#pragma unroll
        for (int k = 0; k < XDC / 4; ++k) res[k] += c * (double)sa[cg + 4 * k][i];
      }
      if (own) {
#pragma unroll
        for (int k = 0; k < XDC / 4; ++k)
          if (cg + 4 * k < dc) {
            double& o = slot(d0 + cg + 4 * k);
            o = first ? res[k] : o + res[k];
          }
      }
    }
    __syncthreads();
  }
}

// out[(c0 + n, d) in `layout`] = sigma^2 t_d (...) from the row ranges summed in a fixed order (see the top of the file)
template <typename T>
__global__ void vfe_x_finish_kernel(const double* __restrict__ xpart, int nsplit, int64_t ldx, int64_t nc, int D,
                                    const T* __restrict__ Xc, const T* __restrict__ isn, int linear, double variance,
                                    double c, double mult, const T* __restrict__ ard, int layout, int64_t N,
                                    int64_t c0, T* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nc * D) return;
  const int64_t n = idx / D;
  const int d = (int)(idx - n * D);
  double s = 0.0, sz = 0.0;
  for (int q = 0; q < nsplit; ++q) s += xpart[((int64_t)q * (D + 1) + d) * ldx + n];
  const double x = (double)Xc[n * D + d];
  double v;
  if (linear) {
    const double is = (double)isn[n];
    v = s - c * x * (is * is);
  } else {
    for (int q = 0; q < nsplit; ++q) sz += xpart[((int64_t)q * (D + 1) + D) * ldx + n];
    v = -(s - x * sz);
  }
  v *= variance * mult;
  if (ard) v *= (double)ard[d];
  const int64_t gn = c0 + n;
  out[layout == AGP_POINT_MAJOR ? gn * D + d : (int64_t)d * N + gn] = (T)v;
}

}  // namespace

void vfe_x_shape(int64_t m_pad, int64_t cap, int* nsplit) {
  const int ncb = (int)((cap + XC - 1) / XC), ntiles = (int)(m_pad / XR);
  int s = (X_CTA_TARGET + ncb - 1) / ncb;
  s = s < 1 ? 1 : (s > X_MAX_SPLIT ? X_MAX_SPLIT : s);
  *nsplit = s < ntiles ? s : ntiles;
}

template <typename T>
void launch_vfe_x_grad(const T* Zt, int64_t M, int64_t m_pad, const T* Xc, int64_t nc, int D, const T* G, int64_t ldg,
                       const T* r, const T* delta, const T* isn, int family, int nsplit, double* xpart, int64_t ldx,
                       cudaStream_t s) {
  if (nc <= 0) return;
  const int ncb = (int)((nc + XC - 1) / XC), ntiles = (int)(m_pad / XR);
  dim3 grid((unsigned)ncb, (unsigned)nsplit);
  if (family == AGP_LINEAR)
    vfe_x_grad_kernel<T, true><<<grid, 256, 0, s>>>(Zt, M, Xc, nc, D, G, ldg, r, delta, isn, family, ntiles, nsplit, xpart, ldx);
  else
    vfe_x_grad_kernel<T, false><<<grid, 256, 0, s>>>(Zt, M, Xc, nc, D, G, ldg, r, delta, isn, family, ntiles, nsplit, xpart, ldx);
  agp_count_launch();
}

template <typename T>
void launch_vfe_x_finish(const double* xpart, int nsplit, int64_t ldx, int64_t nc, int D, const T* Xc, const T* isn,
                         int linear, double variance, double c, double mult, const T* ard, int layout, int64_t N,
                         int64_t c0, T* out, cudaStream_t s) {
  const int64_t tot = nc * D;
  if (tot <= 0) return;
  vfe_x_finish_kernel<T><<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(xpart, nsplit, ldx, nc, D, Xc, isn, linear, variance,
                                                                       c, mult, ard, layout, N, c0, out);
  agp_count_launch();
}

template void launch_vfe_x_grad<double>(const double*, int64_t, int64_t, const double*, int64_t, int, const double*, int64_t,
                                        const double*, const double*, const double*, int, int, double*, int64_t,
                                        cudaStream_t);
template void launch_vfe_x_finish<double>(const double*, int, int64_t, int64_t, int, const double*, const double*, int,
                                          double, double, double, const double*, int, int64_t, int64_t, double*,
                                          cudaStream_t);
