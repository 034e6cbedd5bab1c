/* Minimal C client of the drop-in boundary (include/agp.h): logpdf + posterior weights from ONE call, then a
 * predictive mean/variance at the training points.  Build (the library itself needs an H100 to run):
 *   gcc -std=c99 -Iinclude examples/c_abi_demo.c -o c_abi_demo -Labstractgps.jl_b200 -l:libagp.so -lm
 * This is what the reference-side binding (julia/AGPBlackwell.jl, `ccall`) does, in C. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "agp.h"

int main(void) {
  enum { N = 512, D = 2 };
  static double X[N * D], y[N], alpha[N], mu[N], var[N];
  for (int i = 0; i < N; ++i) {
    X[i * D + 0] = (double)rand() / RAND_MAX;  /* point-major: x_i = X[i*D .. i*D+D) */
    X[i * D + 1] = (double)rand() / RAND_MAX;
    y[i] = sin(6.0 * X[i * D]) + 0.1 * ((double)rand() / RAND_MAX - 0.5);
  }
  agp_ctx* ctx = NULL;
  int32_t rc = agp_init(&ctx, 0, NULL);
  if (rc != AGP_OK) { fprintf(stderr, "agp_init: status %d (no CUDA device?)\n", rc); return 2; }
  agp_kernel k = {AGP_MATERN32, AGP_T_SCALE, 1.0, 4.0, 0.0, NULL}; /* Matern32 o ScaleTransform(4) */
  agp_mean m = {0, 0.0, NULL};                                      /* ZeroMean */
  agp_noise s2 = {0, 1e-2, NULL};                                   /* f(x, 0.01) */
  double lp = 0.0;
  agp_post* post = NULL;
  rc = agp_fit(ctx, AGP_F64, &k, &m, &s2, AGP_POINT_MAJOR, X, N, D, y, 1, &lp, alpha, &post);
  if (rc == AGP_ERR_NOT_POSDEF) { fprintf(stderr, "PosDefException(%lld)\n", (long long)agp_last_info(ctx)); return 1; }
  if (rc != AGP_OK) { fprintf(stderr, "agp_fit: %s\n", agp_last_error(ctx)); return 1; }
  rc = agp_post_mean_var(post, AGP_POINT_MAJOR, X, N, NULL, &s2, mu, var);
  if (rc != AGP_OK) { fprintf(stderr, "agp_post_mean_var: %s\n", agp_last_error(ctx)); return 1; }
  printf("logpdf = %.9f   mean[0] = %.6f (y[0] = %.6f)   var[0] = %.3e\n", lp, mu[0], y[0], var[0]);
  agp_post_free(post);
  agp_destroy(ctx);
  return 0;
}
