// umma_ozaki.h -- host interface of the int8-sliced (Ozaki) trailing update on the Hopper tensor cores (wgmma)
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

struct OzakiWs {
  int8_t* SL;       // S slices, each m_alloc rows x K bytes (K-major), slice s at row s*m_alloc
  double* rscale;   // 2^e_i per panel row
  double* rinv;     // 2^-e_i
  int64_t m_alloc;  // rows per slice (multiple of 128)
  int K;            // panel width (bytes per slice row), multiple of 64
  int S;            // number of slices (3..8; 6 for 8-bit digits)
  int bits;         // digit width, fixed at creation: 7 (balanced 7-bit slices) or 8 (six balanced 8-bit slices, K <= OZ8_MAX_K)
  int bulk;   // 2: slices in the blocked no-swizzle K-major layout [row block][k block][slice] fetched with 1-D bulk copies
  int64_t* tab_start;  // device tables of the block-cyclic tile enumeration  of tab_cap+1 entries:
  int32_t* tab_bimin;  // consecutive calls (main / side stream) alternate slots
  int tab_cap;
  mutable int tab_slot;
  mutable int chunk_tiles;  // > 0 -> bounded CTAs of this many consecutive tiles (see the kernel), 0 -> persistent
  mutable int max_ctas;  // persistent kernel: cap on the grid, 0 = one CTA per SM.  The distributed schedule leaves
                         // a few SMs to the NCCL broadcast that overlaps the update.
};

// eight-bit digits keep the int32 accumulators exact (|ACC_d| <= 5 2^14 K < 2^31) up to this K
constexpr int OZ8_MAX_K = 16384;
int ozaki_ws_create(OzakiWs* ws, int64_t max_rows, int K, int S, cudaStream_t s, int bits = 7);  // 0 = ok
void ozaki_ws_destroy(OzakiWs* ws, cudaStream_t s);
// slice the panel P (m x K fp64, column-major, lda) into ws
void ozaki_prepare(const OzakiWs& ws, const double* P, int64_t lda, int64_t m, cudaStream_t s);
// C (M x N, ldc) -= P P'  using the slices in ws; column n of C pairs with panel row
// (n/128)*b_tile_stride + n%128 + b_off  (b_tile_stride = 0: n + b_off), row r of C with panel row r + a_off;
// lower_only skips tiles above the diagonal.  Returns 0 once launched, 1 (nothing launched) if ws.S is not 5..8, an 8-bit
// workspace has K > OZ8_MAX_K, or the strip table of the shape does not fit the workspace; the caller must then run the
// update another way.
int ozaki_syrk(const OzakiWs& ws, double* C, int64_t ldc, int64_t M, int64_t N, int lower_only, int64_t b_tile_stride,
               int64_t b_tile_width, int64_t b_off, int64_t a_off, cudaStream_t s);

// generalised entry points:
//  * operands may be fp32 or fp64, row-contiguous (element (row, k) at P[row + k*lda]) or k-major (P[k + row*lda]); the
//    rows land at [dst_row0, dst_row0 + m) of the slice buffer (dst_row0 a multiple of 128), so the two operands of a general
//    product C += sign * A B' are sliced into ONE workspace and addressed with a_off / b_off;
//  * C may be fp32 or fp64; full = 1: every row tile of every 64-column strip (rectangular product), 0: lower tiles only.
// returns 0 on success, 1 if the workspace / shape is not supported (an 8-bit workspace takes fp64 C and K <= OZ8_MAX_K).
void ozaki_prepare_ex(const OzakiWs& ws, const void* P, int p_is_float, int kmajor, int64_t lda, int64_t m, int64_t dst_row0,
                      cudaStream_t s);
int ozaki_update_ex(const OzakiWs& ws, void* C, int c_is_float, int64_t ldc, int64_t M, int64_t N, int full, double sign,
                    int64_t b_tile_stride, int64_t b_tile_width, int64_t b_off, int64_t a_off, cudaStream_t s);
