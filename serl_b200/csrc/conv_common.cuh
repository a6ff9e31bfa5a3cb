// Helpers shared by the tensor-core convolutions (conv_tcgen05.cu, conv3x3_res.cu, stem_pool.cu): mbarrier waits, TMA loads,
// the 16-bit operand formats, the named barriers of the warp-specialised kernels, and where a consumer gets its GroupNorm
// affine from.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "common.cuh"

namespace serl {

__device__ inline uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ inline void tc_mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ inline void tc_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must not hang the GPU box.  Returns false (and flags) on timeout.
__device__ inline bool tc_mbar_wait(uint64_t* bar, uint32_t parity, int32_t* error) {
  const uint32_t addr = smem_u32(bar);
  const long long t0 = clock64();
#pragma unroll 1
  for (;;) {
    uint32_t done;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    if (done) return true;
    if (clock64() - t0 > 4000000000ll) break;               // ~2 s: flag and bail out instead of hanging the box
  }
  atomicOr(error, 2);
  return false;
}
// The same bounded wait with acquire semantics at cluster scope: the phase was completed by other CTAs' st.async writes.
__device__ inline bool tc_mbar_wait_cluster(uint64_t* bar, uint32_t parity, int32_t* error) {
  const uint32_t addr = smem_u32(bar);
  const long long t0 = clock64();
#pragma unroll 1
  for (;;) {
    uint32_t done;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    if (done) return true;
    if (clock64() - t0 > 4000000000ll) break;
  }
  atomicOr(error, 2);
  return false;
}

// 16-bit MMA operand formats: bf16 (8-bit mantissa) or fp16 (11-bit mantissa, same tensor throughput).
struct Bf16 {
  static constexpr bool kBf16 = true;
  __device__ static inline uint32_t pack(float lo, float hi) { __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi); return *reinterpret_cast<uint32_t*>(&v); }
  __device__ static inline float2 unpack(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u)); }
  __device__ static inline uint32_t max2(uint32_t a, uint32_t b) {
    __nv_bfloat162 r = __hmax2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b)); return *reinterpret_cast<uint32_t*>(&r);
  }
};
struct Fp16 {
  static constexpr bool kBf16 = false;
  __device__ static inline uint32_t pack(float lo, float hi) {            // saturating: fp16 max is 65504
    __half2 v = __floats2half2_rn(fminf(fmaxf(lo, -65504.f), 65504.f), fminf(fmaxf(hi, -65504.f), 65504.f));
    return *reinterpret_cast<uint32_t*>(&v);
  }
  __device__ static inline float2 unpack(uint32_t u) { return __half22float2(*reinterpret_cast<__half2*>(&u)); }
  __device__ static inline uint32_t max2(uint32_t a, uint32_t b) {
    __half2 r = __hmax2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b)); return *reinterpret_cast<uint32_t*>(&r);
  }
};
template <class F>
__device__ inline uint32_t affine_relu_x2(uint32_t u, float a0, float b0, float a1, float b1) {
  float2 f = F::unpack(u);
  return F::pack(fmaxf(fmaf(f.x, a0, b0), 0.f), fmaxf(fmaf(f.y, a1, b1), 0.f));
}

__device__ inline void tc_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ inline void tc_tma_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// 4-D tile load; coordinates outside the tensor (negative included) read as zeros
__device__ inline void tc_tma_4d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// ---- the warp-specialised kernels (conv3x3_res.cu, stem_pool.cu): two consumer warpgroups + one producer warpgroup ----
constexpr int CONV_THREADS = 384;

// named barrier over the 256 MMA threads that also ANDs a flag across them
__device__ inline bool mma_bar_and(bool v) {
  uint32_t r;
  asm volatile("{\n .reg .pred p, q;\n setp.ne.u32 p, %1, 0;\n barrier.red.and.pred q, 1, 256, p;\n selp.u32 %0, 1, 0, q;\n}"
               : "=r"(r) : "r"((uint32_t)v) : "memory");
  return r != 0;
}
__device__ inline void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;\n barrier.cluster.wait.acquire;" ::: "memory");
}
__device__ inline void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ inline void named_bar_arrive(int id, int threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
// four 8x8 b16 tiles between shared memory (one 16-byte row per address, rows = pixels) and the accumulator layout (rows =
// channels), transposed on the way
__device__ inline void ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ inline void stsm_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]) : "memory");
}

// ---- where a consumer gets its GroupNorm affine from: a precomputed (N, C) table (serl_gn_finalize), or straight from the
// conv epilogue's sums + the frozen scale / bias (same arithmetic as gn_finalize_kernel, bit for bit) - the "_gn" entry
// points, which take the 12 finalize launches out of the trunk's dependency chain.
struct GnSrc {
  const float* a; const float* b;
  const float* stats; const float* gamma; const float* beta;
  float count, eps; int Cg;
};
__device__ inline void gn_load8(const GnSrc& g, int n, int C, int c0, float (&a)[8], float (&b)[8]) {
  if (g.stats) {
    const int grp = c0 / g.Cg;                                 // 8 consecutive channels never straddle a group (Cg >= 16)
    const float s = g.stats[((size_t)n * 4 + grp) * 2], ss = g.stats[((size_t)n * 4 + grp) * 2 + 1];
    const float mean = s / g.count;
    const float var = fmaxf(ss / g.count - mean * mean, 0.f);
    const float rstd = rsqrtf(var + g.eps);
    const float4 g0 = *reinterpret_cast<const float4*>(g.gamma + c0), g1 = *reinterpret_cast<const float4*>(g.gamma + c0 + 4);
    const float4 e0 = *reinterpret_cast<const float4*>(g.beta + c0), e1 = *reinterpret_cast<const float4*>(g.beta + c0 + 4);
    const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, bt[8] = {e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) { a[j] = rstd * gm[j]; b[j] = bt[j] - mean * a[j]; }
  } else {
    const size_t co = (size_t)n * C + c0;
    const float4 a0 = *reinterpret_cast<const float4*>(g.a + co), a1 = *reinterpret_cast<const float4*>(g.a + co + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(g.b + co), b1 = *reinterpret_cast<const float4*>(g.b + co + 4);
    a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
    b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
  }
}

typedef CUresult (*TcEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline TcEncodeTiledFn tc_get_encode() {
  static TcEncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<TcEncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace serl
