// rand_grad.cu -- the two small kernels of the pullback of rand(fx, S) (agp_rand_grad and agp_post_rand_grad, agp.h).  The N^3 work of that
// pullback runs on the tile GEMM and the forward substitution; what is left is
//   - Q: the symmetric matrix whose lower triangle (diagonal included) is that of Zbar Z'.  The lower-only GEMM writes
//     the lower tiles; symmetrize_lower copies the strict lower triangle onto the upper one.
//   - the mean cotangent mbar_i = sum_s Obar_is, summed in fp64 in column order (two calls give the same bits).
#include "kernels.h"

namespace {

constexpr int ST = 32;  // transpose tile

// A[i + j*lda] = A[j + i*lda] for i < j < n: one CTA per 32 x 32 tile on or above the diagonal, staged through shared
// memory so that both the read (a tile of the lower triangle) and the write (its mirror) are coalesced.  The elements read
// (strictly lower) and written (strictly upper) are disjoint, also on the diagonal tiles.
template <typename T>
__global__ void symmetrize_lower_kernel(T* __restrict__ A, int64_t lda, int64_t n) {
  const int bi = blockIdx.x, bj = blockIdx.y;  // destination tile (rows bi, columns bj), bj >= bi
  if (bj < bi) return;
  __shared__ T tile[ST][ST + 1];
  const int64_t r0 = (int64_t)bi * ST, c0 = (int64_t)bj * ST;
  const int tx = threadIdx.x;
  // source: rows c0.., columns r0.. (the lower tile), tile[c][r] = A(c0 + c, r0 + r)
  for (int y = threadIdx.y; y < ST; y += blockDim.y) {
    const int64_t gi = c0 + tx, gj = r0 + y;
    if (gi < n && gj < n && gi > gj) tile[tx][y] = A[gi + gj * lda];
  }
  __syncthreads();
  for (int y = threadIdx.y; y < ST; y += blockDim.y) {
    const int64_t gi = r0 + tx, gj = c0 + y;  // A(gi, gj) = A(gj, gi) = tile[y][tx]
    if (gi < n && gj < n && gi < gj) A[gi + gj * lda] = tile[y][tx];
  }
}

template <typename T>
__global__ void rowsum_kernel(const T* __restrict__ A, int64_t lda, int64_t n, int S, double* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = 0.0;
  for (int s = 0; s < S; ++s) acc += (double)A[i + (int64_t)s * lda];
  out[i] = acc;
}

}  // namespace

template <typename T>
void launch_symmetrize_lower(T* A, int64_t lda, int64_t n, cudaStream_t s) {
  if (n <= 0) return;
  const unsigned nt = (unsigned)((n + ST - 1) / ST);
  symmetrize_lower_kernel<T><<<dim3(nt, nt), dim3(ST, 8), 0, s>>>(A, lda, n);
  agp_count_launch();
}

template <typename T>
void launch_rowsum(const T* A, int64_t lda, int64_t n, int S, double* out, cudaStream_t s) {
  if (n <= 0) return;
  rowsum_kernel<T><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(A, lda, n, S, out);
  agp_count_launch();
}

template void launch_symmetrize_lower<double>(double*, int64_t, int64_t, cudaStream_t);
template void launch_rowsum<double>(const double*, int64_t, int64_t, int, double*, cudaStream_t);
// agp_post_rand_grad runs fp32 handles in fp32
template void launch_symmetrize_lower<float>(float*, int64_t, int64_t, cudaStream_t);
template void launch_rowsum<float>(const float*, int64_t, int64_t, int, double*, cudaStream_t);
