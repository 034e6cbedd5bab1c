// post_xs_grad.cu -- the test-point gradient of mean_and_var over an exact posterior (agp_post_mean_var_grad, agp.h).
// With P = C^-1 K_xs (n_pad x m_pad, column-major), alpha = C^-1 (y - m) and the cotangents mbar, vbar of the means and
// variances,
//   xs_grad[j] = sum_n Kbar_sx[j, n] d1k(x*_j, x_n) + 2 vbar_j d1k(x*_j, x*_j),   Kbar_sx[j, n] = mbar_j alpha_n - 2 vbar_j P[n, j]
// over the N x M cross pairs only: no N x N or (N + M)^2 buffer, and the weight Kbar_sx is formed on the fly from one tile
// of P and three vectors, never stored.  Every kernel is a sum of product terms (composite.cuh); a single kernel is a
// one-factor descriptor over the handle's transformed points and its Scale / ARD chain factor is applied by the finishing
// kernel, as in grad_x.cu.  Per pair (j, n) and accumulator a the product rule gives one coefficient
// c_a = Kbar_sx[j, n] sum_{f on a} v_t prod_{g != f} kappa_g * (q_f s2_f | s2_f for Linear) from comp_factor_grad and
// comp_other, and the per-dimension pass adds
//   SQ   c_a w_d^2 (x*_j - x_n)_d,   DOT  c_a w_d^2 x_{n,d},   PER  c_a (-pi/2) w_d / r_d^2 sinpi(2 w_d (x*_j - x_n)_d).
// A test point on a training point has an exactly zero difference, so the pair adds 0 for every stationary factor
// (Matern 1/2: q = 0 at d2 = 0, its zero subgradient).
//
// The second term is the derivative of k(x*_j, x*_j), which only dot-product accumulators carry: the finishing kernel
// adds 2 vbar_j sum_{f on a DOT accumulator} v_t prod_{g != f} kappa_g s2_f w_d^2 x*_{j,d} with every factor evaluated on
// the diagonal (SQ and PER accumulators 0).
//
// A CTA owns 64 test points and sweeps a fixed range of training-point tiles; the ranges are chosen so that the grid
// fills the GPU even for one test point.  Each CTA writes fp64 partials it alone owns (no atomics), and
// cross_grad_x_finish_kernel sums the ranges in a fixed order, so two calls give the same bits.
#include "kernels.h"
#include "agp.h"
#include "composite.cuh"

namespace {

constexpr int RT = 64;            // test points per CTA
constexpr int RDC = 16;           // feature chunk
constexpr int CTA_TARGET = 264;   // row blocks x column ranges aimed at (two CTAs per SM of a 132-SM H100)
constexpr int MAX_SPLIT = 264;    // one row block (M <= 64) is split over up to 264 column ranges

template <int NA> struct CxCB { static constexpr int v = NA <= 2 ? 2 : 1; };  // column tile 16 * CB (registers)

template <typename T, int NA, int CB>
__global__ void __launch_bounds__(256, 1)
cross_grad_x_kernel(const T* __restrict__ Xs, const T* __restrict__ X, int D, int64_t m, int64_t n,
                    const T* __restrict__ P, int64_t ldp, const T* __restrict__ alpha, const T* __restrict__ mbar,
                    const T* __restrict__ vbar, const __grid_constant__ CompositeDesc cd, int ntiles, int nsplit,
                    double* __restrict__ part, int64_t ldq) {
  constexpr int TC = 16 * CB;
  const int rb = blockIdx.x, sp = blockIdx.y;
  const int t0 = (int)((int64_t)ntiles * sp / nsplit), t1 = (int)((int64_t)ntiles * (sp + 1) / nsplit);
  const int64_t row0 = (int64_t)rb * RT;
  __shared__ T sa[RDC][RT];
  __shared__ T sb[RDC][TC + 1];
  __shared__ double sw[NA][RDC];
  __shared__ double sr[NA][RDC];
  __shared__ double sc[RT][TC + 1];      // the P tile, then one accumulator's coefficients
  __shared__ double sv[2 * RT + TC];     // mbar and -2 vbar of the rows, alpha of the columns
  const T* __restrict__ Wt = (const T*)cd.w;  // null: unit weights (a single kernel on transformed points)
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int ci = tid & 63, cg = tid >> 6;  // per-dimension pass: output row, dimension group
  double* __restrict__ out = part + (int64_t)sp * D * ldq;
  if (tid < RT) {
    const bool ok = row0 + tid < m;
    sv[tid] = ok ? (double)mbar[row0 + tid] : 0.0;
    sv[RT + tid] = ok ? -2.0 * (double)vbar[row0 + tid] : 0.0;
  }

  // stage feature chunk [d0, d0 + dc) of the test points, the training tile and accumulators [a0, a0 + na)'s weights
  auto stage = [&](int64_t col0, int d0, int dc, int a0, int na) {
    for (int idx = tid; idx < RT * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      sa[d][i] = (d < dc && row0 + i < m) ? Xs[(row0 + i) * D + d0 + d] : (T)0;
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
    // the P tile (coalesced along the training points) and alpha of the columns
    __syncthreads();
    if (tid < TC) sv[2 * RT + tid] = col0 + tid < n ? (double)alpha[col0 + tid] : 0.0;
    for (int idx = tid; idx < RT * TC; idx += 256) {
      const int i = idx / TC, j = idx - i * TC;
      const int64_t gi = row0 + i, gj = col0 + j;
      sc[i][j] = (gi < m && gj < n) ? (double)P[gj + gi * ldp] : 0.0;
    }
    __syncthreads();
    double wq[4][CB];  // Kbar_sx = mbar_j alpha_n - 2 vbar_j P[n, j]
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < CB; ++c) {
        const int i = tx + 16 * r, j = ty + 16 * c;
        wq[r][c] = sv[i] * sv[2 * RT + j] + sv[RT + i] * sc[i][j];
      }
#pragma unroll 1
    for (int a = 0; a < NA; ++a) {
      const int kind = cd.acc_kind[a];
      __syncthreads();
      // coefficient of accumulator a for every element of the tile
#pragma unroll 1
      for (int e = 0; e < 4 * CB; ++e) {
        const int r = e & 3, c = e >> 2;
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
            x[b] = y;
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
        if (row0 + ci < m) {
#pragma unroll
          for (int k = 0; k < RDC / 4; ++k) {
            const int d = cg + 4 * k;
            if (d >= dc) continue;
            const double wd = sw[0][d];
            const double mu = kind == COMP_ACC_PER ? -1.5707963267948966192 * wd * sr[0][d] * sr[0][d] : wd * wd;
            out[(int64_t)(d0 + d) * ldq + row0 + ci] += mu * res[k];
          }
        }
      }
    }
    __syncthreads();
  }
}

// out = mult * chain_d * (sum over column ranges in a fixed order + the kdiag term), in the caller's layout.  kdiag: the
// descriptor has a DOT accumulator (a Linear factor), so d k(x*_j, x*_j) / d x*_j is not zero.
template <typename T>
__global__ void cross_grad_x_finish_kernel(const double* __restrict__ part, int nsplit, int64_t ldq, const T* __restrict__ Xs,
                                           int64_t m, int D, const T* __restrict__ vbar,
                                           const __grid_constant__ CompositeDesc cd, int kdiag, double mult,
                                           const T* __restrict__ ard, int layout, T* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * D) return;
  int64_t i;
  int d;
  if (layout == AGP_POINT_MAJOR) { i = idx / D; d = (int)(idx - i * D); }
  else { d = (int)(idx / m); i = idx - (int64_t)d * m; }
  double s = 0.0;
  for (int q = 0; q < nsplit; ++q) s += part[((int64_t)q * D + d) * ldq + i];
  const double vb = (double)vbar[i];
  if (kdiag && vb != 0.0) {
    const T* __restrict__ Wt = (const T*)cd.w;
    double x[AGP_COMP_MAX];
#pragma unroll
    for (int a = 0; a < AGP_COMP_MAX; ++a) {
      x[a] = 0.0;
      if (a < cd.nacc && cd.acc_kind[a] == COMP_ACC_DOT)
        for (int e = 0; e < D; ++e) {
          const double w = Wt ? (double)Wt[(int64_t)(2 * a) * D + e] : 1.0, v = (double)Xs[i * D + e];
          x[a] += w * w * v * v;
        }
    }
    double kap[AGP_COMP_MAX];
    comp_all_kappa<AGP_COMP_MAX>(cd, x, kap);
    double t = 0.0;
    for (int f = 0; f < cd.nfactors; ++f) {
      const CompFactor& F = cd.f[f];
      if (F.acc < 0 || cd.acc_kind[F.acc] != COMP_ACC_DOT) continue;
      const double w = Wt ? (double)Wt[(int64_t)(2 * F.acc) * D + d] : 1.0;
      t += comp_other(cd, kap, f) * F.s2 * w * w;
    }
    s += 2.0 * vb * t * (double)Xs[i * D + d];
  }
  s *= mult;
  if (ard) s *= (double)ard[d];
  out[idx] = (T)s;
}

int cx_cb(int nacc) { return nacc <= 2 ? 2 : 1; }

void cx_shape(int64_t m, int64_t n, int nacc, int* ntiles, int* nrb, int* nsplit) {
  const int tc = 16 * cx_cb(nacc);
  *ntiles = (int)((n + tc - 1) / tc);
  *nrb = (int)((m + RT - 1) / RT);
  int s = (CTA_TARGET + *nrb - 1) / *nrb;
  s = s < 1 ? 1 : (s > MAX_SPLIT ? MAX_SPLIT : s);
  *nsplit = s < *ntiles ? s : *ntiles;
}

template <typename T, int NA>
void launch_na(const T* Xs, int64_t m, const T* X, int64_t n, int D, const T* P, int64_t ldp, const T* alpha,
               const T* mbar, const T* vbar, const CompositeDesc& cd, double* part, cudaStream_t s) {
  int ntiles, nrb, nsplit;
  cx_shape(m, n, NA, &ntiles, &nrb, &nsplit);
  dim3 grid((unsigned)nrb, (unsigned)nsplit);
  cross_grad_x_kernel<T, NA, CxCB<NA>::v><<<grid, 256, 0, s>>>(Xs, X, D, m, n, P, ldp, alpha, mbar, vbar, cd, ntiles,
                                                               nsplit, part, (int64_t)nrb * RT);
  agp_count_launch();
}

}  // namespace

int64_t cross_grad_x_part_len(int64_t m, int64_t n, int D, int nacc) {
  int ntiles, nrb, nsplit;
  cx_shape(m, n, nacc, &ntiles, &nrb, &nsplit);
  return (int64_t)nsplit * D * nrb * RT;
}

template <typename T>
void launch_cross_grad_x(const T* Xs, int64_t m, const T* X, int64_t n, int D, const T* P, int64_t ldp, const T* alpha,
                         const T* mbar, const T* vbar, const CompositeDesc& cd, double mult, const T* ard, int layout,
                         double* part, T* out, cudaStream_t s) {
  if (m <= 0 || n <= 0 || D <= 0) return;
  cudaMemsetAsync(part, 0, (size_t)cross_grad_x_part_len(m, n, D, cd.nacc) * sizeof(double), s);
  switch (cd.nacc) {
    case 1: launch_na<T, 1>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
    case 2: launch_na<T, 2>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
    case 3: launch_na<T, 3>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
    case 4: launch_na<T, 4>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
    case 5: launch_na<T, 5>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
    case 6: launch_na<T, 6>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
    case 7: launch_na<T, 7>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
    default: launch_na<T, 8>(Xs, m, X, n, D, P, ldp, alpha, mbar, vbar, cd, part, s); break;
  }
  int kdiag = 0;
  for (int a = 0; a < cd.nacc; ++a) kdiag |= cd.acc_kind[a] == COMP_ACC_DOT;
  int ntiles, nrb, nsplit;
  cx_shape(m, n, cd.nacc, &ntiles, &nrb, &nsplit);
  const int64_t tot = m * D;
  cross_grad_x_finish_kernel<T><<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(part, nsplit, (int64_t)nrb * RT, Xs, m, D,
                                                                               vbar, cd, kdiag, mult, ard, layout, out);
  agp_count_launch();
}
template void launch_cross_grad_x<float>(const float*, int64_t, const float*, int64_t, int, const float*, int64_t,
                                         const float*, const float*, const float*, const CompositeDesc&, double,
                                         const float*, int, double*, float*, cudaStream_t);
template void launch_cross_grad_x<double>(const double*, int64_t, const double*, int64_t, int, const double*, int64_t,
                                          const double*, const double*, const double*, const CompositeDesc&, double,
                                          const double*, int, double*, double*, cudaStream_t);
