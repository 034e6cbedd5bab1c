// wgmma_i8.h -- wgmma.mma_async m64nNk32 s32 <- s8 x s8 wrappers for the tile widths the int8-slice kernel issues.
// WgmmaI8<N>: A comes from registers, 4 x b32 per thread in the mma.m16n8k32 layout of each warp's 16 rows (reg 0: row
// lane/4, k bytes 4 (lane%4) .. +3; reg 1: row + 8; regs 2, 3: the same at k + 16).  B is K-major in shared memory, described by
// a 64-bit matrix descriptor.  One accumulator fragment of N/2 registers per thread; scale_d = 0 overwrites the
// accumulators, 1 adds to them.
#pragma once
#include <stdint.h>

// operand lists: 8 accumulator registers starting at d[b] (constraint)
#define AGP_D8(b) "+r"(d[b]), "+r"(d[b + 1]), "+r"(d[b + 2]), "+r"(d[b + 3]), "+r"(d[b + 4]), "+r"(d[b + 5]), "+r"(d[b + 6]), "+r"(d[b + 7])
#define AGP_D16(b) AGP_D8(b), AGP_D8(b + 8)
#define AGP_D32(b) AGP_D16(b), AGP_D16(b + 16)

template <int N> struct WgmmaI8;
#define AGP_WGMMA_I8(N, A, B, SC, REGS, ...)                                                                       \
  template <> struct WgmmaI8<N> {                                                                                  \
    __device__ __forceinline__ static void mma(uint32_t* d, const uint32_t* a, uint64_t b, uint32_t scale_d) {     \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #SC ", 0;\n\t"                                          \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k32.s32.s8.s8 {" REGS "}, {" A "}, %" #B ", p;\n\t}"     \
                   : __VA_ARGS__                                                                                   \
                   : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));                           \
    }                                                                                                              \
  };
AGP_WGMMA_I8(32, "%16,%17,%18,%19", 20, 21, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15",
             AGP_D16(0))
AGP_WGMMA_I8(64, "%32,%33,%34,%35", 36, 37, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31",
             AGP_D32(0))
#undef AGP_WGMMA_I8

// the same MMA with A read from shared memory too: A is the warpgroup's 64 rows in the K-major layout of B, described
// by its own matrix descriptor
struct WgmmaI8SS64 {
  __device__ __forceinline__ static void mma(uint32_t* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
                 "%32, %33, p;\n\t}"
                 : AGP_D32(0)
                 : "l"(a), "l"(b), "r"(scale_d));
  }
};
#undef AGP_D32
#undef AGP_D16
#undef AGP_D8
