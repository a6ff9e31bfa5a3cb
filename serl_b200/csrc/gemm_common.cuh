// Shared by the CUDA-core SGEMM (gemm_fp32.cu) and the tensor-core 3xTF32 GEMM (gemm_tf32x3.cu): kernel arguments and
// the deterministic split-K / batch-reduce pass (fixed summation order, no atomics).
#pragma once
#include "common.cuh"

namespace serl {

struct GemmArgs {
  const float* A; const float* B; float* C; const float* bias; float* ws;
  int M, N, K, Z, S;                 // S = k-splits
  long long sAz, sAm, sAk, sBz, sBk, sBn, sCz, sBiasZ;
  int ldc;
  int accumulate, to_ws;
  int kchunk, a_mode, b_mode;                       // tensor-core path only: staging mode of each operand (see gemm_tf32x3.cu)
};

// C[zc](m,n) = sum_{parts} ws[part](m,n) + bias + (accumulate ? C : 0); parts of zc: reduce_z ? all Z*S : S.
static __global__ void gemm_reduce_kernel(const GemmArgs g, int reduce_z) {
  pdl_prologue();
  const int ZC = reduce_z ? 1 : g.Z;
  const size_t MN = (size_t)g.M * g.N, total = MN * ZC;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int zc = (int)(e / MN); const size_t mn = e - (size_t)zc * MN;
    const int m = (int)(mn / g.N), n = (int)(mn - (size_t)m * g.N);
    const int p0 = reduce_z ? 0 : zc * g.S, np = reduce_z ? g.Z * g.S : g.S;
    float v = 0.f;
    for (int p = 0; p < np; ++p) v += g.ws[(size_t)(p0 + p) * MN + mn];
    if (g.bias) v += (g.bias + zc * g.sBiasZ)[n];
    float* c = g.C + zc * g.sCz + (size_t)m * g.ldc + n;
    *c = g.accumulate ? (*c + v) : v;
  }
}


// ---- fp32 operand staging of the tensor-core GEMMs (gemm_tf32x3.cu, tgemm.cu): cp.async into a raw ring, then all threads
// split / round the raw tile into K-major, 128B-swizzled tf32 operand tiles for wgmma (which takes tf32 operands K-major only).
constexpr int T_THREADS = 256;

__device__ inline uint32_t t_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ inline void t_cp16(uint32_t dst, const float* src, int nbytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(nbytes) : "memory");
}
__device__ inline void t_cp4(uint32_t dst, const float* src, int nbytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(nbytes) : "memory");
}

// Staging modes of one operand, seen as a (ROWS x 32) tile indexed (r, k) with global strides (sR, sK):
//   0: sK == 1, 16-byte copies, raw layout [r][32]        2: any strides, 4-byte copies, raw layout [r][32]
//   1: sR == 1, 16-byte copies, raw layout [k][ROWS]      3: any strides, 4-byte copies, raw layout [k][ROWS]
template <int ROWS>
__device__ inline void t_issue_raw(uint32_t dst, const float* P, int rows_total, int r0, long long sR, long long sK, int k0, int kend,
                                   int mode, int tid) {
  if (mode == 0) {
#pragma unroll
    for (int i = 0; i < ROWS * 8 / T_THREADS; ++i) {
      const int it = tid + T_THREADS * i, r = it >> 3, c = it & 7, gr = r0 + r, gk = k0 + 4 * c;
      const int nb = gr < rows_total ? min(16, max(0, (kend - gk) * 4)) : 0;
      t_cp16(dst + it * 16, nb ? P + gr * sR + gk : P, nb);
    }
  } else if (mode == 1) {
    constexpr int CPR = ROWS / 4;
#pragma unroll
    for (int i = 0; i < ROWS * 8 / T_THREADS; ++i) {
      const int it = tid + T_THREADS * i, k = it / CPR, c = it % CPR, gk = k0 + k, gr = r0 + 4 * c;
      const int nb = gk < kend ? min(16, max(0, (rows_total - gr) * 4)) : 0;
      t_cp16(dst + it * 16, nb ? P + gk * sK + gr : P, nb);
    }
  } else if (mode == 2) {
#pragma unroll 4
    for (int i = 0; i < ROWS * 32 / T_THREADS; ++i) {
      const int it = tid + T_THREADS * i, r = it >> 5, k = it & 31, gr = r0 + r, gk = k0 + k;
      const bool v = gr < rows_total && gk < kend;
      t_cp4(dst + it * 4, v ? P + gr * sR + gk * sK : P, v ? 4 : 0);
    }
  } else {
#pragma unroll 4
    for (int i = 0; i < ROWS * 32 / T_THREADS; ++i) {
      const int it = tid + T_THREADS * i, k = it / ROWS, r = it % ROWS, gr = r0 + r, gk = k0 + k;
      const bool v = gr < rows_total && gk < kend;
      t_cp4(dst + it * 4, v ? P + gr * sR + gk * sK : P, v ? 4 : 0);
    }
  }
}

__device__ inline void t_split(float x, float& hi, float& lo) {
  uint32_t h;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  hi = __uint_as_float(h);
  lo = x - hi;
}

// raw fp32 tile -> K-major SWIZZLE_128B hi / lo tiles: element (r, k) at r*128 + (((k>>2) ^ (r&7)) << 4) + (k&3)*4
template <int ROWS>
__device__ inline void t_convert(const float* raw, uint8_t* hi, uint8_t* lo, bool layout_kr, int tid) {   // lo == nullptr: hi only
#pragma unroll
  for (int i = 0; i < ROWS * 8 / T_THREADS; ++i) {
    const int it = tid + T_THREADS * i;
    int r, c;
    float4 v;
    if (!layout_kr) {
      r = it >> 3; c = it & 7;
      v = reinterpret_cast<const float4*>(raw)[it];
    } else {                                               // consecutive lanes take consecutive rows: conflict-free both ways
      r = it % ROWS; c = it / ROWS;
      const float* p = raw + (4 * c) * ROWS + r;
      v = make_float4(p[0], p[ROWS], p[2 * ROWS], p[3 * ROWS]);
    }
    float4 h, l;
    t_split(v.x, h.x, l.x); t_split(v.y, h.y, l.y); t_split(v.z, h.z, l.z); t_split(v.w, h.w, l.w);
    const int off = r * 128 + ((c ^ (r & 7)) << 4);
    *reinterpret_cast<float4*>(hi + off) = h;
    if (lo) *reinterpret_cast<float4*>(lo + off) = l;
  }
}

// operand staging mode from its strides/alignment (see t_issue_raw)
static inline int pick_mode(const float* base, long long sZ, long long sR, long long sK, int Z) {
  const bool base_ok = (reinterpret_cast<uintptr_t>(base) & 15) == 0 && (Z == 1 || sZ % 4 == 0);
  if (sK == 1 && base_ok && sR % 4 == 0) return 0;
  if (sR == 1 && base_ok && sK % 4 == 0) return 1;
  const long long ar = sR < 0 ? -sR : sR, ak = sK < 0 ? -sK : sK;
  return ak <= ar ? 2 : 3;
}


// host side: launch the reduce pass for a descriptor whose partials sit in g.ws
inline int launch_gemm_reduce(const GemmArgs& g, int reduce_z, cudaStream_t st) {
  size_t total = (size_t)g.M * g.N * (reduce_z ? 1 : g.Z);
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 8) blocks = 132 * 8;
  launch_k(gemm_reduce_kernel, blocks, 256, 0, st, g, reduce_z);
  return check_launch("gemm_reduce_kernel");
}

}  // namespace serl
