// composite.cuh -- device helpers shared by the composite Gram (gram.cu) and gradient (grad.cu) kernels.
// A composite kernel is K(x, y) = sum_t v_t prod_{f in t} kappa_f(T_f x, T_f y) (agp.h agp_kernel_composite).  The
// kernels accumulate one distance per accumulator slot (CompositeDesc::acc_kind) and evaluate the factors from those.
#pragma once
#include <cuda_runtime.h>
#include "agp.h"
#include "kernels.h"

template <typename T> __device__ __forceinline__ T comp_exp(T x);
template <> __device__ __forceinline__ float comp_exp<float>(float x) { return expf(x); }
template <> __device__ __forceinline__ double comp_exp<double>(double x) { return exp(x); }
template <typename T> __device__ __forceinline__ T comp_sqrt(T x);
template <> __device__ __forceinline__ float comp_sqrt<float>(float x) { return sqrtf(x); }
template <> __device__ __forceinline__ double comp_sqrt<double>(double x) { return sqrt(x); }
template <typename T> __device__ __forceinline__ T comp_sinpi(T x);
template <> __device__ __forceinline__ float comp_sinpi<float>(float x) { return sinpif(x); }
template <> __device__ __forceinline__ double comp_sinpi<double>(double x) { return sinpi(x); }
template <typename T> __device__ __forceinline__ T comp_pow(T x, T y);
template <> __device__ __forceinline__ float comp_pow<float>(float x, float y) { return powf(x, y); }
template <> __device__ __forceinline__ double comp_pow<double>(double x, double y) { return pow(x, y); }

// v[a] for a runtime slot a without dynamic register indexing (which would put v on the stack)
template <typename T, int NA>
__device__ __forceinline__ T comp_pick(const T (&v)[NA], int a) {
  T x = v[0];
#pragma unroll
  for (int i = 1; i < NA; ++i)
    if (a == i) x = v[i];
  return x;
}

// kappa_f from its accumulator value x (the symmetric diagonal has SQ / PER accumulators already zeroed).  A factor on a
// shared raw accumulator scales it by s^2 (F.s2 is 1 for ARD and Periodic factors, whose weights are in the sum).
template <typename T>
__device__ __forceinline__ T comp_factor(const CompFactor& F, T x) {
  const T d2 = x * (T)F.s2;
  switch (F.family) {
    case AGP_SE: return comp_exp<T>(-d2 * (T)0.5);
    case AGP_MATERN12: return comp_exp<T>(-comp_sqrt<T>(d2));
    case AGP_MATERN32: {
      const T s = (T)1.7320508075688772935 * comp_sqrt<T>(d2);
      return ((T)1 + s) * comp_exp<T>(-s);
    }
    case AGP_MATERN52: {
      const T s = (T)2.2360679774997896964 * comp_sqrt<T>(d2);
      return ((T)1 + s + s * s * (T)(1.0 / 3.0)) * comp_exp<T>(-s);
    }
    case AGP_RQ: {
      const T a = (T)F.param;
      return comp_pow<T>((T)1 + d2 / ((T)2 * a), -a);
    }
    case AGP_PERIODIC: return comp_exp<T>(-(T)0.5 * x);
    case AGP_WHITE: return x == (T)0 ? (T)1 : (T)0;
    case AGP_CONSTANT: return (T)F.param;
    default: return d2 + (T)F.param;  // AGP_LINEAR
  }
}

// The same factors in fp64 for the gradient kernels (grad.cu, grad_x.cu): kappa_f from its accumulator value x and
// ds = d kappa / d s (Scale transform on a shared raw accumulator), dp = d kappa / d param (RQ alpha, Linear / Constant
// c), q = 2 d kappa / d d2 (stationary / RQ: the ARD pass uses q v_d diff_d^2), or kappa itself for a Periodic factor
// (its pass needs kappa sin_d^2 / r_d^3 and the sinpi cospi terms).  q is 0 for Linear, White and Constant, and for
// Matern 1/2 at d2 == 0 (its zero subgradient there).
__device__ __forceinline__ void comp_factor_grad(const CompFactor& F, double x, double& kap, double& ds, double& dp,
                                                 double& q) {
  const double d2 = x * F.s2;
  ds = 0.0; dp = 0.0; q = 0.0;
  switch (F.family) {
    case AGP_SE: { const double e = exp(-0.5 * d2); kap = e; q = -e; break; }
    case AGP_MATERN12: { const double d = sqrt(d2), e = exp(-d); kap = e; q = d > 0.0 ? -e / d : 0.0; break; }
    case AGP_MATERN32: {
      const double s = 1.7320508075688772935 * sqrt(d2), e = exp(-s);
      kap = (1.0 + s) * e; q = -3.0 * e;
      break;
    }
    case AGP_MATERN52: {
      const double s = 2.2360679774997896964 * sqrt(d2), e = exp(-s);
      kap = (1.0 + s + s * s * (1.0 / 3.0)) * e; q = -(5.0 / 3.0) * (1.0 + s) * e;
      break;
    }
    case AGP_RQ: {
      const double a = F.param, u = d2 / (2.0 * a);
      kap = pow(1.0 + u, -a);
      q = -kap / (1.0 + u);
      dp = kap * (u / (1.0 + u) - log1p(u));
      break;
    }
    case AGP_PERIODIC: kap = exp(-0.5 * x); q = kap; break;
    case AGP_WHITE: kap = (x == 0.0) ? 1.0 : 0.0; break;
    case AGP_CONSTANT: kap = F.param; dp = 1.0; break;
    default: kap = d2 + F.param; dp = 1.0; break;  // AGP_LINEAR
  }
  if (F.transform == AGP_T_SCALE) {
    if (F.family == AGP_LINEAR) ds = 2.0 * F.s * x;
    else if (F.family <= AGP_RQ && F.family != AGP_LINEAR) ds = q * F.s * x;  // d d2 / d s = 2 s x
  }
}

template <int NA>
__device__ __forceinline__ void comp_all_kappa(const CompositeDesc& cd, const double (&x)[NA], double (&kap)[AGP_COMP_MAX]) {
#pragma unroll
  for (int f = 0; f < AGP_COMP_MAX; ++f) {
    double ds, dp, q;
    kap[f] = 1.0;
    if (f < cd.nfactors) comp_factor_grad(cd.f[f], comp_pick<double, NA>(x, cd.f[f].acc), kap[f], ds, dp, q);
  }
}

// v_t prod_{g in t, g != f} kappa_g
__device__ __forceinline__ double comp_other(const CompositeDesc& cd, const double (&kap)[AGP_COMP_MAX], int f) {
  const int t = cd.f[f].term;
  double o = cd.variance[t];
#pragma unroll
  for (int g = 0; g < AGP_COMP_MAX; ++g)
    if (g < cd.nfactors && g != f && cd.f[g].term == t) o *= kap[g];
  return o;
}

// sum_t v_t prod_{f in t} kappa_f; factors are stored term by term
template <typename T, int NA>
__device__ __forceinline__ T comp_eval(const CompositeDesc& cd, const T (&v)[NA]) {
  T sum = 0;
  int f = 0;
  for (int t = 0; t < cd.nterms; ++t) {
    T prod = (T)cd.variance[t];
    for (; f < cd.nfactors && cd.f[f].term == t; ++f) prod *= comp_factor<T>(cd.f[f], comp_pick<T, NA>(v, cd.f[f].acc));
    sum += prod;
  }
  return sum;
}
