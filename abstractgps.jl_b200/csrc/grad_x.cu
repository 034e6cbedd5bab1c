// grad_x.cu -- gradient of logpdf(fx, y) with respect to the input points,
//   dL/dx_{i,d} = sum_j W_ij d1k(x_i, x_j)_d,   W = alpha alpha' - C^-1   (j over all points, j == i included),
// d1 the derivative in the first argument.  Every kernel is handled as a sum of product terms (composite.cuh): a single
// kernel is a one-factor descriptor over the handle's transformed points, and its Scale / ARD chain factor is applied by
// the finishing kernel.  Per element (i, j) and accumulator a (kernels.h COMP_ACC_*) the product rule gives one
// coefficient c_a = W_ij sum_{f on a} v_t prod_{g != f} kappa_g * (q_f s2_f | s2_f for Linear), q_f = 2 dkappa_f/dd2
// (kappa_f itself for Periodic), never dividing by a factor's value; then
//   SQ   dL/dx_{i,d} += c_a w_d^2 (x_i - x_j)_d                            (direct differences, as gram_kernel)
//   DOT  dL/dx_{i,d} += c_a w_d^2 x_{j,d}
//   PER  dL/dx_{i,d} += c_a (-pi/2) w_d / r_d^2 sinpi(2 w_d (x_i - x_j)_d)
// Coincident points have an exactly zero difference, so they add 0 for every stationary factor (Matern 1/2: q = 0 at
// d2 = 0, its zero subgradient).
//
// C^-1 holds its lower tiles only: a CTA owns a 64-row block of outputs and sweeps a fixed range of column tiles, reading
// tiles above the diagonal transposed through shared memory.  Each CTA writes fp64 partials it alone owns (no atomics);
// grad_x_finish_kernel sums the column ranges in a fixed order, so two calls give the same bits.
#include "kernels.h"
#include "agp.h"
#include "composite.cuh"

namespace {

constexpr int RT = 64;            // output rows per CTA
constexpr int RDC = 16;           // feature chunk
constexpr int CTA_TARGET = 264;   // row blocks x column ranges aimed at (two CTAs per SM of a 132-SM H100)
constexpr int MAX_SPLIT = 64;

template <int NA> struct GxCB { static constexpr int v = NA <= 2 ? 2 : 1; };  // column tile 16 * CB (registers)

template <typename T, int NA, int CB>
__global__ void __launch_bounds__(256, 1)
grad_x_kernel(const T* __restrict__ X, int D, int64_t n, const T* __restrict__ Cinv, int64_t ldc,
              const T* __restrict__ alpha, const __grid_constant__ CompositeDesc cd, int ntiles, int nsplit,
              double* __restrict__ part, int64_t ldp) {
  constexpr int TC = 16 * CB;
  const int rb = blockIdx.x, sp = blockIdx.y;
  const int t0 = (int)((int64_t)ntiles * sp / nsplit), t1 = (int)((int64_t)ntiles * (sp + 1) / nsplit);
  const int64_t row0 = (int64_t)rb * RT;
  __shared__ T sa[RDC][RT];
  __shared__ T sb[RDC][TC + 1];
  __shared__ double sw[NA][RDC];
  __shared__ double sr[NA][RDC];
  __shared__ double sc[RT][TC + 1];  // the C^-1 tile, then one accumulator's coefficients
  __shared__ double sal[RT + TC];    // alpha of the rows, then of the columns
  const T* __restrict__ Wt = (const T*)cd.w;  // null: unit weights (a single kernel on transformed points)
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int ci = tid & 63, cg = tid >> 6;  // per-dimension pass: output row, dimension group
  double* __restrict__ out = part + (int64_t)sp * D * ldp;
  if (tid < RT) sal[tid] = row0 + tid < n ? (double)alpha[row0 + tid] : 0.0;

  // stage feature chunk [d0, d0 + dc) of the row block, the column tile and accumulators [a0, a0 + na)'s weights
  auto stage = [&](int64_t col0, int d0, int dc, int a0, int na) {
    for (int idx = tid; idx < RT * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      sa[d][i] = (d < dc && row0 + i < n) ? X[(row0 + i) * D + d0 + d] : (T)0;
    }
    for (int idx = tid; idx < TC * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      sb[d][i] = (d < dc && col0 + i < n) ? X[(col0 + i) * D + d0 + d] : (T)0;
    }
    for (int idx = tid; idx < na * RDC; idx += 256) {
      const int a = idx / RDC, d = idx - a * RDC, ag = a0 + a;
      sw[a][d] = (d < dc && Wt) ? (double)Wt[(int64_t)(2 * ag) * D + d0 + d] : 1.0;
      sr[a][d] = (d < dc && Wt) ? (double)Wt[(int64_t)(2 * ag + 1) * D + d0 + d] : 1.0;
    }
  };

#pragma unroll 1
  for (int tcol = t0; tcol < t1; ++tcol) {
    const int64_t col0 = (int64_t)tcol * TC;
    // distances of the 64 x TC tile, the accumulation of composite_gram_kernel
    double acc[NA][4][CB];
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < CB; ++c) acc[a][r][c] = 0.0;
    for (int d0 = 0; d0 < D; d0 += RDC) {
      const int dc = min(RDC, D - d0);
      __syncthreads();
      stage(col0, d0, dc, 0, NA);
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
    }
    // C^-1 tile: lower storage below the diagonal (coalesced along rows), transposed above it (coalesced along columns),
    // element by element where the tile straddles the diagonal
    __syncthreads();
    if (tid < TC) sal[RT + tid] = col0 + tid < n ? (double)alpha[col0 + tid] : 0.0;
    const bool below = col0 + TC <= row0, above = col0 >= row0 + RT;
    for (int idx = tid; idx < RT * TC; idx += 256) {
      int i, j;
      if (above) { i = idx / TC; j = idx - i * TC; } else { j = idx / RT; i = idx - j * RT; }
      const int64_t gi = row0 + i, gj = col0 + j;
      double v = 0.0;
      if (gi < n && gj < n) v = (double)((below || (!above && gi >= gj)) ? Cinv[gi + gj * ldc] : Cinv[gj + gi * ldc]);
      sc[i][j] = v;
    }
    __syncthreads();
    double wq[4][CB];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < CB; ++c) {
        const int i = tx + 16 * r, j = ty + 16 * c;
        wq[r][c] = (row0 + i < n && col0 + j < n) ? sal[i] * sal[RT + j] - sc[i][j] : 0.0;
      }
#pragma unroll 1
    for (int a = 0; a < NA; ++a) {
      const int kind = cd.acc_kind[a];
      __syncthreads();
      // coefficient of accumulator a for every element of the tile
#pragma unroll 1
      for (int e = 0; e < 4 * CB; ++e) {
        const int r = e & 3, c = e >> 2;
        const int64_t gi = row0 + tx + 16 * r, gj = col0 + ty + 16 * c;
        double w = wq[0][0];
#pragma unroll
        for (int q = 1; q < 4 * CB; ++q)
          if (q == e) w = wq[q & 3][q >> 2];
        double cf = 0.0;
        if (w != 0.0) {
          double x[NA];
#pragma unroll
          for (int b = 0; b < NA; ++b) {
            double y = acc[b][0][0];
#pragma unroll
            for (int q = 1; q < 4 * CB; ++q)
              if (q == e) y = acc[b][q & 3][q >> 2];
            x[b] = (gi == gj && cd.acc_kind[b] != COMP_ACC_DOT) ? 0.0 : y;
          }
          double kap[AGP_COMP_MAX];
          comp_all_kappa<NA>(cd, x, kap);
#pragma unroll 1
          for (int f = 0; f < cd.nfactors; ++f) {
            const CompFactor& F = cd.f[f];
            if (F.acc != a) continue;
            double k_, ds, dp, qf;
            comp_factor_grad(F, comp_pick<double, NA>(x, a), k_, ds, dp, qf);
            cf += comp_other(cd, kap, f) * (kind == COMP_ACC_DOT ? F.s2 : qf * F.s2);
          }
          cf *= w;
        }
        sc[tx + 16 * r][ty + 16 * c] = cf;
      }
      // per-dimension pass: thread (row ci, group cg) owns dimensions cg, cg + 4, ... of each chunk
      for (int d0 = 0; d0 < D; d0 += RDC) {
        const int dc = min(RDC, D - d0);
        __syncthreads();
        stage(col0, d0, dc, a, 1);
        __syncthreads();
        double xi[RDC / 4], res[RDC / 4];
#pragma unroll
        for (int k = 0; k < RDC / 4; ++k) { xi[k] = (double)sa[cg + 4 * k][ci]; res[k] = 0.0; }
        if (kind == COMP_ACC_SQ) {
#pragma unroll 4
          for (int j = 0; j < TC; ++j) {
            const double c = sc[ci][j];
#pragma unroll
            for (int k = 0; k < RDC / 4; ++k) res[k] += c * (xi[k] - (double)sb[cg + 4 * k][j]);
          }
        } else if (kind == COMP_ACC_DOT) {
#pragma unroll 4
          for (int j = 0; j < TC; ++j) {
            const double c = sc[ci][j];
#pragma unroll
            for (int k = 0; k < RDC / 4; ++k) res[k] += c * (double)sb[cg + 4 * k][j];
          }
        } else {
#pragma unroll 1
          for (int j = 0; j < TC; ++j) {
            const double c = sc[ci][j];
#pragma unroll
            for (int k = 0; k < RDC / 4; ++k)
              res[k] += c * sinpi(2.0 * sw[0][cg + 4 * k] * (xi[k] - (double)sb[cg + 4 * k][j]));
          }
        }
        if (row0 + ci < n) {
#pragma unroll
          for (int k = 0; k < RDC / 4; ++k) {
            const int d = cg + 4 * k;
            if (d >= dc) continue;
            const double wd = sw[0][d];
            const double m = kind == COMP_ACC_PER ? -1.5707963267948966192 * wd * sr[0][d] * sr[0][d] : wd * wd;
            out[(int64_t)(d0 + d) * ldp + row0 + ci] += m * res[k];
          }
        }
      }
    }
    __syncthreads();
  }
}

// out = mult * chain_d * sum over column ranges (fixed order), in the caller's layout
template <typename T>
__global__ void grad_x_finish_kernel(const double* __restrict__ part, int nsplit, int64_t ldp, int64_t n, int D,
                                     double mult, const T* __restrict__ ard, int layout, T* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * D) return;
  int64_t i;
  int d;
  if (layout == AGP_POINT_MAJOR) { i = idx / D; d = (int)(idx - i * D); }
  else { d = (int)(idx / n); i = idx - (int64_t)d * n; }
  double s = 0.0;
  for (int q = 0; q < nsplit; ++q) s += part[((int64_t)q * D + d) * ldp + i];
  s *= mult;
  if (ard) s *= (double)ard[d];
  out[idx] = (T)s;
}

int gx_cb(int nacc) { return nacc <= 2 ? 2 : 1; }

void gx_shape(int64_t n, int nacc, int* ntiles, int* nrb, int* nsplit) {
  const int tc = 16 * gx_cb(nacc);
  *ntiles = (int)((n + tc - 1) / tc);
  *nrb = (int)((n + RT - 1) / RT);
  int s = (CTA_TARGET + *nrb - 1) / *nrb;
  s = s < 1 ? 1 : (s > MAX_SPLIT ? MAX_SPLIT : s);
  *nsplit = s < *ntiles ? s : *ntiles;
}

template <typename T, int NA>
void launch_na(const T* X, int D, int64_t n, const T* Cinv, int64_t ldc, const T* alpha, const CompositeDesc& cd,
               double* part, cudaStream_t s) {
  int ntiles, nrb, nsplit;
  gx_shape(n, NA, &ntiles, &nrb, &nsplit);
  dim3 grid((unsigned)nrb, (unsigned)nsplit);
  grad_x_kernel<T, NA, GxCB<NA>::v><<<grid, 256, 0, s>>>(X, D, n, Cinv, ldc, alpha, cd, ntiles, nsplit, part,
                                                         (int64_t)nrb * RT);
  agp_count_launch();
}

}  // namespace

int64_t grad_x_part_len(int64_t n, int D, int nacc) {
  int ntiles, nrb, nsplit;
  gx_shape(n, nacc, &ntiles, &nrb, &nsplit);
  return (int64_t)nsplit * D * nrb * RT;
}

template <typename T>
void launch_grad_x(const T* X, int D, int64_t n, const T* Cinv, int64_t ldc, const T* alpha, const CompositeDesc& cd,
                   double mult, const T* ard, int layout, double* part, T* out, cudaStream_t s) {
  if (n <= 0) return;
  cudaMemsetAsync(part, 0, (size_t)grad_x_part_len(n, D, cd.nacc) * sizeof(double), s);
  switch (cd.nacc) {
    case 1: launch_na<T, 1>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
    case 2: launch_na<T, 2>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
    case 3: launch_na<T, 3>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
    case 4: launch_na<T, 4>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
    case 5: launch_na<T, 5>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
    case 6: launch_na<T, 6>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
    case 7: launch_na<T, 7>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
    default: launch_na<T, 8>(X, D, n, Cinv, ldc, alpha, cd, part, s); break;
  }
  int ntiles, nrb, nsplit;
  gx_shape(n, cd.nacc, &ntiles, &nrb, &nsplit);
  const int64_t tot = n * D;
  grad_x_finish_kernel<T><<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(part, nsplit, (int64_t)nrb * RT, n, D, mult, ard,
                                                                         layout, out);
  agp_count_launch();
}
template void launch_grad_x<float>(const float*, int, int64_t, const float*, int64_t, const float*, const CompositeDesc&,
                                   double, const float*, int, double*, float*, cudaStream_t);
template void launch_grad_x<double>(const double*, int, int64_t, const double*, int64_t, const double*,
                                    const CompositeDesc&, double, const double*, int, double*, double*, cudaStream_t);
