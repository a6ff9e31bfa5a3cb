// Batched, strided fp32 GEMM on the Hopper tensor cores (wgmma) with fp32-class accuracy ("3xTF32"): the speed build's carrier
// of every dense contraction of the trainable heads (same call sites as gemm_fp32.cu: networks/mlp.py:22-31,
// networks/actor_critic_nets.py:64-72,187-192, vision/resnet_v1.py:371, common/encoding.py:65-67 and their jax.grad
// transposes, common/common.py:204).  Same descriptor and semantics as serl_gemm_f32:
//   C[z](m, n) = sum_k A[z](m, k) * B[z](k, n) (+ bias[z](n)) (+ C[z](m, n) if accumulate);  reduce_z: C = sum_z (...)
//
// Each fp32 operand x is split into hi = rna_tf32(x) and lo = x - hi (exact); the product is accumulated as
// a_lo*b_hi + a_hi*b_lo + a_hi*b_hi in fp32 register accumulators (wgmma m64n64k8 tf32, one warpgroup per 64 rows), which leaves
// an error of ~2^-22 per product - the dropped lo*lo term and the hardware's truncation of lo - i.e. that of an fp32 FMA.
//
// One CTA per 128x64 output tile and K-split.  Per 32-wide k-block:
//   cp.async (16 B where the operand's layout allows, else 4 B; zero-fill at every edge) -> raw fp32 ring, 4 stages deep
//   -> all threads split + transpose the raw tile into K-major, 128B-swizzled hi/lo operand tiles (2 stages)
//   -> each warpgroup issues its 12 MMAs and retires them one k-block later (wgmma.wait_group 1).
// The raw ring keeps three k-blocks of global loads in flight per SM; these GEMMs are tiny (<= 1 GFLOP) so the kernel is
// bound by that latency, not by the tensor pipe.  Split-K partials go through the same deterministic reduce pass as the
// CUDA-core SGEMM.
#include "gemm_common.cuh"
#include "wgmma.cuh"
#include "serl_b200.h"

namespace serl {

constexpr int TM = 128, TN = 64, TK = 32;
constexpr int T_RS = 4;                                   // raw stages
constexpr int RAW_A = TM * TK * 4, RAW_B = TN * TK * 4, RAW_STAGE = RAW_A + RAW_B;
constexpr int OP_A = TM * 128, OP_B = TN * 128, OP_STAGE = 2 * OP_A + 2 * OP_B;   // hi + lo of each operand
constexpr int T_SMEM = 2 * OP_STAGE + T_RS * RAW_STAGE + 1024;

__global__ void __launch_bounds__(T_THREADS, 1) gemm_tf32x3_kernel(const GemmArgs g) {
  pdl_prologue();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sOp = smem;                                     // 2 x [A_hi | A_lo | B_hi | B_lo]
  uint8_t* sRaw = smem + 2 * OP_STAGE;                     // T_RS x [A raw | B raw]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;                                // warpgroup = 64-row half of the output tile
  const int z = blockIdx.z / g.S, s = blockIdx.z - z * g.S;
  const int m0 = blockIdx.x * TM, n0 = blockIdx.y * TN;
  const int kbeg = s * g.kchunk, kend = min(g.K, kbeg + g.kchunk);
  const int nk = kend > kbeg ? ceil_div(kend - kbeg, TK) : 0;
  const float* A = g.A + z * g.sAz;
  const float* B = g.B + z * g.sBz;

  auto issue = [&](int kt) {
    const uint32_t dst = t_smem(sRaw + (kt % T_RS) * RAW_STAGE);
    const int k0 = kbeg + kt * TK;
    t_issue_raw<TM>(dst, A, g.M, m0, g.sAm, g.sAk, k0, kend, g.a_mode, tid);
    t_issue_raw<TN>(dst + RAW_A, B, g.N, n0, g.sBn, g.sBk, k0, kend, g.b_mode, tid);
  };

#pragma unroll
  for (int st = 0; st < T_RS - 1; ++st) {
    if (st < nk) issue(st);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;

  for (int kt = 0; kt < nk; ++kt) {
    asm volatile("cp.async.wait_group %0;" ::"n"(T_RS - 2) : "memory");
    // raw stage kt complete; raw stage kt-1 fully converted by everyone; every warpgroup has retired the MMAs of k-block
    // kt-2 (wgmma.wait_group 1 at the end of the previous iteration), so operand stage kt & 1 may be overwritten
    __syncthreads();
    if (kt + T_RS - 1 < nk) issue(kt + T_RS - 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    const int os = kt & 1;
    uint8_t* op = sOp + os * OP_STAGE;
    const float* raw = reinterpret_cast<const float*>(sRaw + (kt % T_RS) * RAW_STAGE);
    t_convert<TM>(raw, op, op + OP_A, (g.a_mode & 1) != 0, tid);
    t_convert<TN>(raw + TM * TK, op + 2 * OP_A, op + 2 * OP_A + OP_B, (g.b_mode & 1) != 0, tid);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> tensor-core reads
    __syncthreads();
    const uint64_t a_hi = wg_desc(t_smem(op) + wg * 8192), a_lo = wg_desc(t_smem(op + OP_A) + wg * 8192);
    const uint64_t b_hi = wg_desc(t_smem(op + 2 * OP_A)), b_lo = wg_desc(t_smem(op + 2 * OP_A + OP_B));
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
    for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
#pragma unroll
    for (int k = 0; k < 4; ++k) wg_mma_tf32(acc, a_hi + 2 * k, b_hi + 2 * k, 1u);
    wg_commit();
    wg_wait<1>();
  }
  wg_wait<0>();
  asm volatile("cp.async.wait_all;" ::: "memory");

  // epilogue straight from the accumulator fragments (see wgmma.cuh): two rows x 16 column pairs per thread
  float* dst; long long ld; const float* bias = nullptr; bool accum = false;
  if (g.to_ws) { dst = g.ws + ((size_t)blockIdx.z * g.M) * g.N; ld = g.N; }
  else { dst = g.C + z * g.sCz; ld = g.ldc; bias = g.bias ? g.bias + z * g.sBiasZ : nullptr; accum = g.accumulate != 0; }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (m >= g.M) continue;
    float* row = dst + (size_t)m * ld;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + 8 * j + 2 * (lane & 3) + e;
        if (n < g.N) {
          const float o = acc[4 * j + 2 * h + e] + (bias ? bias[n] : 0.f);
          row[n] = accum ? row[n] + o : o;
        }
      }
    }
  }
}

}  // namespace serl

using namespace serl;

extern "C" int serl_gemm_tf32x3(const serl_gemm_desc* d, void* stream) {
  if (!d || d->M < 1 || d->N < 1 || d->K < 1 || d->Z < 1 || !d->A || !d->B || !d->C) {
    set_last_error("serl_gemm_tf32x3: invalid descriptor");
    return SERL_ERR_INVALID;
  }
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(gemm_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, T_SMEM) != cudaSuccess) {
      set_last_error("serl_gemm_tf32x3: cannot reserve %d bytes of shared memory", T_SMEM);
      return SERL_ERR_CUDA;
    }
    attr_done = true;
  }
  GemmArgs g{};
  g.A = d->A; g.B = d->B; g.C = d->C; g.bias = d->bias; g.ws = d->workspace;
  g.M = d->M; g.N = d->N; g.K = d->K; g.Z = d->Z;
  g.sAz = d->sAz; g.sAm = d->sAm; g.sAk = d->sAk; g.sBz = d->sBz; g.sBk = d->sBk; g.sBn = d->sBn;
  g.sCz = d->sCz; g.sBiasZ = d->sBiasZ; g.ldc = d->ldc; g.accumulate = d->accumulate;
  g.a_mode = pick_mode(d->A, d->sAz, d->sAm, d->sAk, d->Z);
  g.b_mode = pick_mode(d->B, d->sBz, d->sBn, d->sBk, d->Z);
  const int tiles = ceil_div(d->M, TM) * ceil_div(d->N, TN) * d->Z;
  // one CTA per SM (~193 KB of staging): split K until about one wave of CTAs exists, >= 2 k-blocks per split
  int S = 1;
  if (tiles < 132 && d->K >= 128) {
    S = 132 / tiles;
    if (S > d->K / 64) S = d->K / 64;
    if (S < 1) S = 1;
  }
  const size_t part = (size_t)d->M * d->N * sizeof(float);
  if (d->reduce_z || S > 1) {
    while (S > 1 && part * (size_t)d->Z * S > d->workspace_bytes) --S;
    if ((d->reduce_z || S > 1) && (!d->workspace || part * (size_t)d->Z * S > d->workspace_bytes)) {
      if (d->reduce_z) { set_last_error("serl_gemm_tf32x3: reduce_z needs %zu workspace bytes", part * (size_t)d->Z); return SERL_ERR_INVALID; }
      S = 1;
    }
  }
  g.kchunk = ceil_div(ceil_div(d->K, S), TK) * TK;
  S = ceil_div(d->K, g.kchunk);                            // no empty splits
  g.S = S;
  g.to_ws = (d->reduce_z || S > 1) ? 1 : 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(ceil_div(d->M, TM), ceil_div(d->N, TN), d->Z * S);
  launch_k(gemm_tf32x3_kernel, grid, T_THREADS, T_SMEM, st, g);
  if (int e = check_launch("gemm_tf32x3_kernel")) return e;
  if (g.to_ws) return launch_gemm_reduce(g, d->reduce_z, st);
  return SERL_OK;
}
