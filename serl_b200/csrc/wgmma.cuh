// Hopper (sm_90a) warpgroup MMA helpers: wgmma.mma_async with both operands in shared memory, fp32 accumulators in registers.
// Operand tiles are K-major in the 128-byte swizzle layout: row r of a tile (128 B = 64 16-bit or 32 tf32 elements) at
// (r >> 3) * 1024 + (r & 7) * 128, 16-byte chunks XOR-ed with (r & 7) - what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B.
// The MMAs here are m64 n64 (n32 for narrow 16-bit tiles): a 128-row tile is two m-blocks 8 KB apart, a wider N is several
// n-chunks 8 KB apart; m64 n256 (wg_mma_h16_n256) takes a 256-row B tile as one descriptor (32 row groups 1024 B apart).
//
// Accumulator fragment of one m64 n64 MMA (thread t of the warpgroup, w = t / 32, l = t % 32), j = 0..7:
//   d[4j + 0], d[4j + 1]: row 16 w + l / 4,     columns 8 j + 2 (l % 4) + {0, 1}
//   d[4j + 2], d[4j + 3]: row 16 w + l / 4 + 8, same columns
// m64 n256: the same with j = 0..31 (128 accumulators per thread).
#pragma once
#include <stdint.h>

namespace serl {

// start address >> 4 | leading byte offset (unused by this layout: 1) | stride byte offset 1024 B >> 4 | layout type 1 (128B swizzle)
__device__ inline uint64_t wg_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
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
#define SERL_WG_D128(d)                                                                                               \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),                     \
  "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),               \
  "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),             \
  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),             \
  "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),             \
  "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),             \
  "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),             \
  "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),             \
  "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),             \
  "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),             \
  "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),             \
  "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),             \
  "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),         \
  "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),     \
  "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),     \
  "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
#define SERL_WG_REGS128                                                                                               \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31," \
  "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63," \
  "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95," \
  "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}"

// m64 n256 k16, 16-bit operands: d[4j + .] as in the header comment for j = 0..31 (the fragment of m64 n64 extended to 256 columns)
template <bool kBf16>
__device__ inline void wg_mma_h16_n256(float (&d)[128], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (kBf16)
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %130, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " SERL_WG_REGS128 ", %128, %129, p, 1, 1, 0, 0;\n}"
                 : SERL_WG_D128(d) : "l"(a), "l"(b), "r"(accumulate));
  else
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %130, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " SERL_WG_REGS128 ", %128, %129, p, 1, 1, 0, 0;\n}"
                 : SERL_WG_D128(d) : "l"(a), "l"(b), "r"(accumulate));
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
#undef SERL_WG_REGS128
#undef SERL_WG_D128

}  // namespace serl
