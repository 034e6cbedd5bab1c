// vfe_grad.cu -- the streamed part of the gradient of the VFE objectives (agp.h agp_vfe_elbo_grad).  With A = L_z^-1 K_zx
// S^-1/2, Lam = I + A A', m_e = Lam^-1 A delta, V_z = L_z^-1, H = c I - Lam^-1 - m_e m_e' and c = 1 (elbo) | 0 (DTC):
//   Kbar_zx = R K_zx S^-1 + r (delta o s^-1/2)',   R = V_z' H V_z,  r = V_z' m_e
//   Kbar_zz = -1/2 V_z' E V_z,                      E = c (Lam - I) - I + Lam^-1 + m_e m_e'
// The engine forms R, r and V_z' E V_z once (O(M^3)); vfe_cross_grad_kernel then takes one chunk of the data at a time
// with G = R K_zx,c already formed by the GEMM, and per element W = Kbar_zx[m, n] = G / s_n + r_m delta_n s_n^-1/2
// recomputes kappa and kappa'(r) r from direct differences of the transformed points (as grad_reduce_kernel does).  It
// accumulates in fp64:
//   - the hyper-parameter sums in grad_reduce_kernel's units (w = 2 W, so the engine maps both with one formula);
//   - per row block, the column sums q_n = sum_m W K and u_n = sum_m K r_m (vfe_point_grad_kernel adds the blocks in a
//     fixed order);
//   - per column range, the row partials sum_n W q(d2) (z~_m - x~_n) (stationary, q = kappa'(r) / r) or sum_n W x~_n
//     (Linear) of the inducing-point gradient (vfe_z_finish_kernel adds the ranges in a fixed order).
// Column sums and inducing-point partials are written by the one CTA that owns them (no atomics: two calls give the same
// bits).  The scalar sums leave each CTA through one atomic per slot; the ARD sums through one atomic per tile and
// feature.
#include "kernels.h"
#include "agp.h"

namespace {

constexpr int RT = 64;           // rows (inducing points) per CTA
constexpr int TC = 32;           // columns (data points) per tile
constexpr int RDC = 16;          // feature chunk
constexpr int CTA_TARGET = 264;  // row blocks x column ranges aimed at (two CTAs per SM of a 132-SM H100)
constexpr int MAX_SPLIT = 64;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// kappa(d2) and kappa'(r) r without the variance (grad.cu's kappa_pair)
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

// H and E (m_pad x m_pad, full) from Lam^-1 (full), D = Lam - I (lower storage, ldd) and m_e; 0 outside M x M
template <typename T>
__global__ void vfe_hz_kernel(const T* __restrict__ Laminv, const T* __restrict__ Dl, int64_t ldd, const T* __restrict__ me,
                              int64_t M, int64_t m_pad, double c, T* __restrict__ H, T* __restrict__ E) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m_pad * m_pad) return;
  const int64_t j = idx / m_pad, i = idx - j * m_pad;
  double h = 0.0, e = 0.0;
  if (i < M && j < M) {
    const double li = (double)Laminv[idx], mm = (double)me[i] * (double)me[j], id = i == j ? 1.0 : 0.0;
    const double d = (double)(i >= j ? Dl[i + j * ldd] : Dl[j + i * ldd]);
    h = c * id - li - mm;
    e = c * d - id + li + mm;
  }
  H[idx] = (T)h;
  E[idx] = (T)e;
}

template <typename T, bool LIN>
__global__ void __launch_bounds__(256)
vfe_cross_grad_kernel(const T* __restrict__ Zt, int64_t M, const T* __restrict__ Xc, int64_t nc, int D,
                      const T* __restrict__ G, int64_t ldg, const T* __restrict__ r, const T* __restrict__ delta,
                      const T* __restrict__ isn, int family, double variance, double linear_c, int want_ard, int ntiles,
                      int nsplit, double* __restrict__ sums, double* __restrict__ qpart, double* __restrict__ upart,
                      int64_t ldq, double* __restrict__ zpart, int64_t ldz) {
  const int rb = blockIdx.x, sp = blockIdx.y;
  const int t0 = (int)((int64_t)ntiles * sp / nsplit), t1 = (int)((int64_t)ntiles * (sp + 1) / nsplit);
  const int64_t row0 = (int64_t)rb * RT;
  __shared__ T sa[RDC][RT];
  __shared__ T sb[RDC][TC + 1];
  __shared__ double sc[RT][TC + 1];
  __shared__ double srow[RT];
  __shared__ double scol[2][TC];  // delta s^-1/2 and 1/s of the columns
  __shared__ double red[8][3];
  __shared__ double sard[RDC];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, tx = tid & 15, ty = tid >> 4;
  const int ci = tid & 63, cg = tid >> 6;  // per-dimension pass: row, dimension group
  if (tid < RT) srow[tid] = row0 + tid < M ? (double)r[row0 + tid] : 0.0;
  double s_var = 0.0, s_scale = 0.0, s_c = 0.0;

  auto stage = [&](int64_t col0, int d0, int dc) {
    for (int idx = tid; idx < RT * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      sa[d][i] = (d < dc && row0 + i < M) ? Zt[(row0 + i) * D + d0 + d] : (T)0;
    }
    for (int idx = tid; idx < TC * RDC; idx += 256) {
      const int i = idx / RDC, d = idx - i * RDC;
      sb[d][i] = (d < dc && col0 + i < nc) ? Xc[(col0 + i) * D + d0 + d] : (T)0;
    }
  };

#pragma unroll 1
  for (int tcol = t0; tcol < t1; ++tcol) {
    const int64_t col0 = (int64_t)tcol * TC;
    double acc[4][2];
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q][0] = acc[q][1] = 0.0;
    for (int d0 = 0; d0 < D; d0 += RDC) {
      const int dc = min(RDC, D - d0);
      __syncthreads();
      stage(col0, d0, dc);
      __syncthreads();
#pragma unroll 1
      for (int d = 0; d < dc; ++d) {
        double a[4], b[2];
#pragma unroll
        for (int q = 0; q < 4; ++q) a[q] = (double)sa[d][tx + 16 * q];
#pragma unroll
        for (int q = 0; q < 2; ++q) b[q] = (double)sb[d][ty + 16 * q];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int p = 0; p < 2; ++p) {
            if (LIN) acc[q][p] += a[q] * b[p];
            else { const double df = a[q] - b[p]; acc[q][p] += df * df; }
          }
      }
    }
    if (tid < TC) {
      const int64_t gj = col0 + tid;
      const double is = gj < nc ? (double)isn[gj] : 0.0;
      scol[0][tid] = gj < nc ? (double)delta[gj] * is : 0.0;
      scol[1][tid] = is * is;
    }
    __syncthreads();
    // per element: W, the scalar sums, and (q_n, u_n, the z coefficient) staged one at a time through sc
    double wk[4][2], kr_[4][2], cz[4][2];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int i = tx + 16 * q, j = ty + 16 * p;
        const int64_t gi = row0 + i, gj = col0 + j;
        wk[q][p] = kr_[q][p] = cz[q][p] = 0.0;
        if (gi >= M || gj >= nc) continue;
        const double W = (double)G[gi + gj * ldg] * scol[1][j] + srow[i] * scol[0][j];
        const double w = 2.0 * W;
        double K;
        if (LIN) {
          K = variance * (acc[q][p] + linear_c);
          s_var += w * (acc[q][p] + linear_c);
          s_scale += w * acc[q][p];
          s_c += w;
          cz[q][p] = W;
        } else {
          const double d2 = acc[q][p];
          double kap, kr;
          kappa_pair(family, d2, kap, kr);
          K = variance * kap;
          s_var += w * kap;
          s_scale += w * kr;
          cz[q][p] = d2 > 0.0 ? W * kr / d2 : 0.0;
        }
        wk[q][p] = W * K;
        kr_[q][p] = K * srow[i];
      }
    // column sums q_n (then u_n) over the 64 rows, in a fixed order
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int p = 0; p < 2; ++p) sc[tx + 16 * q][ty + 16 * p] = pass == 0 ? wk[q][p] : kr_[q][p];
      __syncthreads();
      if (tid < TC && col0 + tid < nc) {
        double t = 0.0;
        for (int i = 0; i < RT; ++i) t += sc[i][tid];
        (pass == 0 ? qpart : upart)[(int64_t)rb * ldq + col0 + tid] = t;
      }
      __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 2; ++p) sc[tx + 16 * q][ty + 16 * p] = cz[q][p];
    // per-dimension pass: thread (row ci, group cg) owns dimensions cg, cg + 4, ... of each chunk
    for (int d0 = 0; d0 < D; d0 += RDC) {
      const int dc = min(RDC, D - d0);
      __syncthreads();
      stage(col0, d0, dc);
      if (tid < RDC) sard[tid] = 0.0;
      __syncthreads();
      double xi[RDC / 4], res[RDC / 4], ard[RDC / 4];
#pragma unroll
      for (int k = 0; k < RDC / 4; ++k) { xi[k] = (double)sa[cg + 4 * k][ci]; res[k] = 0.0; ard[k] = 0.0; }
#pragma unroll 4
      for (int j = 0; j < TC; ++j) {
        const double c = sc[ci][j];
#pragma unroll
        for (int k = 0; k < RDC / 4; ++k) {
          const double xj = (double)sb[cg + 4 * k][j];
          if (LIN) {
            res[k] += c * xj;
          } else {
            const double df = xi[k] - xj;
            res[k] += c * df;
            ard[k] += c * df * df;
          }
        }
      }
      if (row0 + ci < M) {
#pragma unroll
        for (int k = 0; k < RDC / 4; ++k)
          if (cg + 4 * k < dc) zpart[((int64_t)sp * D + d0 + cg + 4 * k) * ldz + row0 + ci] += res[k];
      }
      if (want_ard) {  // sum w q tdiff_d^2 = 2 sum cz tdiff_d^2  |  sum w z~_d x~_d = 2 z~_d sum cz x~_d  (Linear)
#pragma unroll
        for (int k = 0; k < RDC / 4; ++k) {
          const double v = warp_sum_d(2.0 * (LIN ? xi[k] * res[k] : ard[k]));
          if (lane == 0 && cg + 4 * k < dc) atomicAdd(&sard[cg + 4 * k], v);
        }
        __syncthreads();
        if (tid < dc) atomicAdd(&sums[5 + d0 + tid], sard[tid]);
      }
    }
    __syncthreads();
  }
  double v[3] = {s_var, s_scale, s_c};
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const double t = warp_sum_d(v[q]);
    if (lane == 0) red[wid][q] = t;
  }
  __syncthreads();
  if (tid < 3) {
    double t = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) t += red[w8][tid];
    if (t != 0.0) atomicAdd(&sums[tid], t);
  }
}

// per data point of a chunk: deltabar, sbar, mbar from q_n, u_n (row blocks summed in order), the kdiag term of the
// hyper-parameter sums (kdiagbar = -c / (2 s), in the units w = -c / s), and the scalar noise / mean sums nm[0], nm[1]
template <typename T>
__global__ void __launch_bounds__(256)
vfe_point_grad_kernel(const double* __restrict__ qpart, const double* __restrict__ upart, int64_t ldq, int nrb, int64_t nc,
                      const T* __restrict__ delta, const T* __restrict__ isn, const T* __restrict__ kd, int noise_kind,
                      double noise_s, const T* __restrict__ noise_v, double c, const T* __restrict__ Xc, int D, int linear,
                      double linear_c, int want_ard, double* __restrict__ sums, double* __restrict__ nm,
                      T* __restrict__ noise_diag, T* __restrict__ mean_diag) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  __shared__ double red[8][5];
  double sbar = 0.0, mbar = 0.0, w = 0.0, n2 = 0.0;
  const bool ok = j < nc;
  if (ok) {
    double q = 0.0, u = 0.0;
    for (int b = 0; b < nrb; ++b) { q += qpart[(int64_t)b * ldq + j]; u += upart[(int64_t)b * ldq + j]; }
    const double dl = (double)delta[j], is = (double)isn[j];
    const double hs = 0.5 / (noise_kind == 1 ? (double)noise_v[j] : noise_s);  // 1 / (2 s)
    const double dbar = -dl + is * u;
    sbar = hs * (-1.0 + 2.0 * hs * c * (double)kd[j] - q - dbar * dl);
    mbar = -is * dbar;
    if (noise_diag) noise_diag[j] = (T)sbar;
    if (mean_diag) mean_diag[j] = (T)mbar;
    w = -2.0 * c * hs;
    if (linear)
      for (int d = 0; d < D; ++d) { const double x = (double)Xc[j * D + d]; n2 += x * x; }
  }
  {
    const double t0 = warp_sum_d(sbar), t1 = warp_sum_d(mbar), t2 = warp_sum_d(linear ? w * (n2 + linear_c) : w);
    const double t3 = warp_sum_d(linear ? w * n2 : 0.0), t4 = warp_sum_d(linear ? w : 0.0);
    if (lane == 0) { red[wid][0] = t0; red[wid][1] = t1; red[wid][2] = t2; red[wid][3] = t3; red[wid][4] = t4; }
  }
  __syncthreads();
  if (tid < 5) {
    double t = 0.0;
    for (int w8 = 0; w8 < 8; ++w8) t += red[w8][tid];
    if (tid < 2) atomicAdd(&nm[tid], t);
    else if (t != 0.0) atomicAdd(&sums[tid - 2], t);
  }
  if (!(linear && want_ard)) return;
  for (int d = 0; d < D; ++d) {  // Linear ARD: sum w x~_d^2
    __syncthreads();
    const double x = ok ? (double)Xc[j * D + d] : 0.0;
    const double t = warp_sum_d(w * x * x);
    if (lane == 0) red[wid][0] = t;
    __syncthreads();
    if (tid == 0) {
      double s = 0.0;
      for (int w8 = 0; w8 < 8; ++w8) s += red[w8][0];
      atomicAdd(&sums[5 + d], s);
    }
  }
}

// out = zz + mult * chain_d * sum over column ranges (fixed order), in the caller's layout; zz already holds the K_zz part
template <typename T>
__global__ void vfe_z_finish_kernel(const double* __restrict__ zpart, int nsplit, int64_t ldz, int64_t M, int D,
                                    double mult, const T* __restrict__ ard, int layout, const T* __restrict__ zz,
                                    T* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * D) return;
  int64_t i;
  int d;
  if (layout == AGP_POINT_MAJOR) { i = idx / D; d = (int)(idx - i * D); }
  else { d = (int)(idx / M); i = idx - (int64_t)d * M; }
  double s = 0.0;
  for (int q = 0; q < nsplit; ++q) s += zpart[((int64_t)q * D + d) * ldz + i];
  s *= mult;
  if (ard) s *= (double)ard[d];
  out[idx] = (T)((double)zz[idx] + s);
}

template <typename S, typename D>
__global__ void cast_kernel(const S* __restrict__ in, D* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (D)in[i];
}

}  // namespace

template <typename S, typename D>
void launch_cast(const S* in, D* out, int64_t n, cudaStream_t s) {
  if (n <= 0) return;
  cast_kernel<S, D><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(in, out, n);
  agp_count_launch();
}
template void launch_cast<float, double>(const float*, double*, int64_t, cudaStream_t);
template void launch_cast<double, float>(const double*, float*, int64_t, cudaStream_t);

void vfe_cross_shape(int64_t m_pad, int64_t cap, int* nrb, int* nsplit) {
  *nrb = (int)(m_pad / RT);
  const int ntiles = (int)((cap + TC - 1) / TC);
  int s = (CTA_TARGET + *nrb - 1) / *nrb;
  s = s < 1 ? 1 : (s > MAX_SPLIT ? MAX_SPLIT : s);
  *nsplit = s < ntiles ? s : ntiles;
}

template <typename T>
void launch_vfe_hz(const T* Laminv, const T* Dl, int64_t ldd, const T* me, int64_t M, int64_t m_pad, double c, T* H, T* E,
                   cudaStream_t s) {
  const int64_t tot = m_pad * m_pad;
  vfe_hz_kernel<T><<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(Laminv, Dl, ldd, me, M, m_pad, c, H, E);
  agp_count_launch();
}

template <typename T>
void launch_vfe_cross_grad(const T* Zt, int64_t M, int64_t m_pad, const T* Xc, int64_t nc, int D, const T* G, int64_t ldg,
                           const T* r, const T* delta, const T* isn, int family, double variance, double linear_c,
                           int want_ard, int nsplit, double* sums, double* qpart, double* upart, int64_t ldq,
                           double* zpart, cudaStream_t s) {
  const int nrb = (int)(m_pad / RT);
  const int ntiles = (int)((nc + TC - 1) / TC);
  const int ns = nsplit < ntiles ? nsplit : ntiles;
  dim3 grid((unsigned)nrb, (unsigned)ns);
  if (family == AGP_LINEAR)
    vfe_cross_grad_kernel<T, true><<<grid, 256, 0, s>>>(Zt, M, Xc, nc, D, G, ldg, r, delta, isn, family, variance, linear_c,
                                                        want_ard, ntiles, ns, sums, qpart, upart, ldq, zpart, m_pad);
  else
    vfe_cross_grad_kernel<T, false><<<grid, 256, 0, s>>>(Zt, M, Xc, nc, D, G, ldg, r, delta, isn, family, variance, linear_c,
                                                         want_ard, ntiles, ns, sums, qpart, upart, ldq, zpart, m_pad);
  agp_count_launch();
}

template <typename T>
void launch_vfe_point_grad(const double* qpart, const double* upart, int64_t ldq, int nrb, int64_t nc, const T* delta,
                           const T* isn, const T* kd, int noise_kind, double noise_s, const T* noise_v, double c, const T* Xc,
                           int D, int linear, double linear_c, int want_ard, double* sums, double* nm, T* noise_diag,
                           T* mean_diag, cudaStream_t s) {
  if (nc <= 0) return;
  vfe_point_grad_kernel<T><<<(unsigned)((nc + 255) / 256), 256, 0, s>>>(qpart, upart, ldq, nrb, nc, delta, isn, kd, noise_kind,
                                                                         noise_s, noise_v, c, Xc, D, linear, linear_c,
                                                                         want_ard, sums, nm, noise_diag, mean_diag);
  agp_count_launch();
}

template <typename T>
void launch_vfe_z_finish(const double* zpart, int nsplit, int64_t ldz, int64_t M, int D, double mult, const T* ard,
                         int layout, const T* zz, T* out, cudaStream_t s) {
  const int64_t tot = M * D;
  if (tot <= 0) return;
  vfe_z_finish_kernel<T><<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(zpart, nsplit, ldz, M, D, mult, ard, layout, zz, out);
  agp_count_launch();
}

#define AGP_VFE_GRAD_INST(T)                                                                                                 \
  template void launch_vfe_hz<T>(const T*, const T*, int64_t, const T*, int64_t, int64_t, double, T*, T*, cudaStream_t);   \
  template void launch_vfe_cross_grad<T>(const T*, int64_t, int64_t, const T*, int64_t, int, const T*, int64_t, const T*,  \
                                         const T*, const T*, int, double, double, int, int, double*, double*, double*,      \
                                         int64_t, double*, cudaStream_t);                                                   \
  template void launch_vfe_point_grad<T>(const double*, const double*, int64_t, int, int64_t, const T*, const T*, const T*, \
                                         int, double, const T*, double, const T*, int, int, double, int, double*, double*,  \
                                         T*, T*, cudaStream_t);                                                             \
  template void launch_vfe_z_finish<T>(const double*, int, int64_t, int64_t, int, double, const T*, int, const T*, T*,     \
                                       cudaStream_t);
AGP_VFE_GRAD_INST(double)
