// Hopper (sm_90a) warpgroup MMA helpers: wgmma.mma_async with both operands in shared memory, fp32 accumulators in registers.
// Operand tiles are K-major in the 128-byte swizzle layout: row r of a tile (128 B = 64 16-bit or 32 tf32 elements) at
// (r >> 3) * 1024 + (r & 7) * 128, 16-byte chunks XOR-ed with (r & 7) - what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B.
// The MMAs here are m64 n64 (n32 for narrow 16-bit tiles): a 128-row tile is two m-blocks 8 KB apart, a wider N is several
// n-chunks 8 KB apart.
//
// Accumulator fragment of one m64 n64 MMA (thread t of the warpgroup, w = t / 32, l = t % 32), j = 0..7:
//   d[4j + 0], d[4j + 1]: row 16 w + l / 4,     columns 8 j + 2 (l % 4) + {0, 1}
//   d[4j + 2], d[4j + 3]: row 16 w + l / 4 + 8, same columns
#pragma once
#include <stdint.h>

namespace serl {

// start address >> 4 | leading byte offset (unused by this layout: 1) | stride byte offset 1024 B >> 4 | layout type 1 (128B swizzle)
__device__ inline uint64_t wg_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// The 32-byte swizzle (CU_TENSOR_MAP_SWIZZLE_32B) for tiles whose rows are 32 B (one k16 step of 16-bit elements): row r at
// r * 32, the two 16-byte chunks of a row XOR-ed with bit 2 of r; an m64 operand is 8 atoms of 8 rows, 256 B apart.
// start address >> 4 | leading byte offset (unused: 1) | stride byte offset 256 B >> 4 | layout type 3 (32B swizzle)
__device__ inline uint64_t wg_desc_sw32(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (16ull << 32) | (3ull << 62);
}
__device__ inline void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ inline void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ inline void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

#define SERL_WG_D32(d)                                                                                                     \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),  \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), \
      "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), \
      "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define SERL_WG_REGS                                                                                                       \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}"

#define SERL_WG_D16(d)                                                                                                     \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),  \
      "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define SERL_WG_REGS16 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}"

// D (+)= A (64 x 16) B^T (64 x 16), 16-bit operands: kBf16 selects bf16, else fp16.  accumulate == 0 overwrites D.
template <bool kBf16>
__device__ inline void wg_mma_h16(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (kBf16)
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " SERL_WG_REGS ", %32, %33, p, 1, 1, 0, 0;\n}"
                 : SERL_WG_D32(d) : "l"(a), "l"(b), "r"(accumulate));
  else
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " SERL_WG_REGS ", %32, %33, p, 1, 1, 0, 0;\n}"
                 : SERL_WG_D32(d) : "l"(a), "l"(b), "r"(accumulate));
}
// D (+)= A (64 x 8) B^T (64 x 8), tf32 operands (fp32 bit patterns; the tensor core ignores the low 13 mantissa bits)
__device__ inline void wg_mma_tf32(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
  asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
               " wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " SERL_WG_REGS ", %32, %33, p, 1, 1;\n}"
               : SERL_WG_D32(d) : "l"(a), "l"(b), "r"(accumulate));
}
// m64 n32 k16, 16-bit operands: d[4j + .] as above for j = 0..3
template <bool kBf16>
__device__ inline void wg_mma_h16_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (kBf16)
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 " SERL_WG_REGS16 ", %16, %17, p, 1, 1, 0, 0;\n}"
                 : SERL_WG_D16(d) : "l"(a), "l"(b), "r"(accumulate));
  else
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 " SERL_WG_REGS16 ", %16, %17, p, 1, 1, 0, 0;\n}"
                 : SERL_WG_D16(d) : "l"(a), "l"(b), "r"(accumulate));
}
// n64 or n32 by the accumulator's size
template <bool kBf16, int W>
__device__ inline void wg_mma_h16_n(float (&d)[W], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (W == 32) wg_mma_h16<kBf16>(d, a, b, accumulate);
  else wg_mma_h16_n32<kBf16>(d, a, b, accumulate);
}
#undef SERL_WG_REGS
#undef SERL_WG_D32
#undef SERL_WG_REGS16
#undef SERL_WG_D16

}  // namespace serl
