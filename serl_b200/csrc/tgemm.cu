// Heads of the 16-bit builds: fp32 GEMM on the Hopper tensor cores (wgmma tf32) with fused epilogues.
//   * operands come from the fp32 tensors as they are: K-major (k contiguous) or MN-major (m / n contiguous), so X @ W (W stored
//     (K,N) row-major: MN-major B), dZ @ W^T (K-major B) and X^T @ dZ (both MN-major) - forward, input gradient and weight
//     gradient of a Dense layer (networks/mlp.py:22-31 and its jax.grad transposes) - all read the same row-major arrays.  They
//     are staged by cp.async (zero-fill at every edge) into a raw ring, and all threads split each element into tf32 hi + lo
//     parts in K-major, 128-byte-swizzled tiles: wgmma takes tf32 operands K-major only;
//   * one CTA (two warpgroups) per 128 x 256 output tile (x k-split x batch member); warpgroup w computes rows [64 w, 64 w + 64)
//     as four m64n64 accumulators in registers, then hands them to the row-per-thread epilogue through shared memory;
//   * fused epilogues: bias; bias + LayerNorm(eps 1e-6, fast variance) + tanh with the statistics the backward pass needs
//     (a thread owns half an output row, so the row reductions are nearly thread-local); + the value head (Q = h . w + b,
//     networks/actor_critic_nets.py:64-72) or the policy's mean / log-std heads with the tanh-Gaussian sample and its
//     log-probability (actor_critic_nets.py:187-227, 230-272) in the same pass.
// Accuracy: a_lo b_hi + a_hi b_lo + a_hi b_hi per k-step ("3xTF32", as gemm_tf32x3.cu), fp32 accumulation: ~2^-22 per product,
// so the fused heads agree with the per-op chain to fp32 rounding.  These GEMMs are small and bound by load latency, not by
// the tensor pipe.  Up to TG_MAXG problem groups (e.g. the three encoder passes x two cameras of a critic step) share one launch.
#include "gemm_common.cuh"
#include "wgmma.cuh"
#include "serl_b200.h"

namespace serl {

constexpr int TG_BM = 128, TG_BN = 256, TG_BK = 32;           // 32 fp32 = 128 B = one swizzle row
constexpr int TG_RAW = 2;                                     // raw fp32 stages (cp.async ring)
constexpr int TG_THREADS = T_THREADS;                         // two warpgroups: MMA, then the epilogue
constexpr int TG_EPI_THREADS = 256;
constexpr int TG_MAXG = SERL_TGEMM_MAX_PROBLEMS;
constexpr int TG_A_STAGE = TG_BM * 128, TG_B_STAGE = TG_BN * 128, TG_STAGE = TG_A_STAGE + TG_B_STAGE;   // raw fp32 = tf32 operand size
constexpr int TG_MAXHEAD = 8;
// main loop: TG_RAW raw stages + one operand stage (tf32 hi and lo parts of both operands); epilogue (same bytes): accumulator tile 128 x 256 fp32, row sums, head
// partials, per-warp store staging tiles
constexpr int TG_ACC = TG_BM * TG_BN * 4;
constexpr int TG_EPI_BYTES = TG_ACC + (2 * TG_BM * 2 + TG_BM * 16) * 4 + 8 * 2048 * 4;
constexpr int TG_LOOP_BYTES = (TG_RAW + 2) * TG_STAGE;
constexpr int TG_WORK = TG_EPI_BYTES > TG_LOOP_BYTES ? TG_EPI_BYTES : TG_LOOP_BYTES;
// epilogue vectors: bias, ln scale, ln bias (3 x 256), head weights (2 x 256 x 8), head biases (16)
constexpr int TG_SMEM = TG_WORK + (3 * TG_BN + 2 * TG_BN * TG_MAXHEAD + 16) * 4 + 1024;
static_assert(TG_SMEM <= 232448, "tgemm_tf32_kernel: shared memory budget exceeded");

struct TgGroup {
  const float* A; const float* B; long long sAz, sAm, sAk, sBz, sBn, sBk;
  float* C; const float* bias; const float* ln_scale; const float* ln_bias; float* xhat; float* rstd;
  const float* head_w; const float* head_b; float* head_out;
  const float* head_w2; const float* head_b2; float* head_out2;
  const float* noise; float* act; float* logp; float* u_out; float* std_out;
  long long sCz, sBiasZ, sLnZ, sXhatZ, sRstdZ, sHeadWz, sHeadBz, sHeadOutZ;
  int ldc, ld_head, ld_act, z0, Z, a_bcast, b_bcast;
};
struct TgArgs {
  TgGroup g[TG_MAXG];
  float* ws;
  int32_t* error;
  int G, M, N, K, S, kchunk, epi, a_mode, b_mode, accumulate, to_ws, head_n, deterministic;
  float eps, std_min, std_max;
};

// tanh(x) = 1 - 2 / (exp(2x) + 1) on the special-function unit (ex2.approx + rcp.approx): absolute error < 3e-7, exact limits
__device__ inline float tg_tanh(float x) { return 1.f - __fdividef(2.f, __expf(2.f * x) + 1.f); }
__device__ inline float tg_softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// MLP Dropout of the LayerNorm epilogues (serl_tgemm_tf32_masked): problem i's (M, 256) keep mask, shared by its Z members
struct TgMask {
  const uint8_t* mask[TG_MAXG];
  float inv_keep;
};

// v = dropout(acc + bias) for columns c .. c + 31 of row m of a (M, 256) keep mask (rows past M read none)
__device__ __forceinline__ void tg_drop32(const uint8_t* mask, int m, int M, int c, const float* sBias, float inv_keep, float (&v)[32]) {
  uint4 w[2] = {make_uint4(0u, 0u, 0u, 0u), make_uint4(0u, 0u, 0u, 0u)};
  if (m < M) {
    const uint4* mrow = reinterpret_cast<const uint4*>(mask + (size_t)m * TG_BN + c);
    w[0] = mrow[0]; w[1] = mrow[1];
  }
  const uint8_t* keep = reinterpret_cast<const uint8_t*>(w);
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = keep[i] ? (v[i] + sBias[c + i]) * inv_keep : 0.f;
}

// kMask: z' = mask ? (acc + bias) * inv_keep : 0 ahead of the LayerNorm statistics; the saved xhat / rstd are those of z'.  The
// <false> instantiation (mk unused) compiles to the SASS of the kernel before the mask existed (scripts/sass_unchanged.py).
template <bool kMask>
__global__ void __launch_bounds__(TG_THREADS, 1) tgemm_tf32_kernel(const __grid_constant__ TgArgs a, const __grid_constant__ TgMask mk) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sRaw = smem;                                                  // TG_RAW x [A raw 16 KB | B raw 32 KB]
  uint8_t* sOp = smem + TG_RAW * TG_STAGE;                               // [A hi | B hi | A lo | B lo] tf32, K-major, swizzled
  float* sVec = reinterpret_cast<float*>(smem + TG_WORK);                // bias | ln scale | ln bias | head w | head w2 | head b, b2
  float* sBias = sVec, *sLs = sVec + TG_BN, *sLb = sVec + 2 * TG_BN, *sHw = sVec + 3 * TG_BN, *sHw2 = sHw + TG_BN * TG_MAXHEAD, *sHb = sHw2 + TG_BN * TG_MAXHEAD;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int zz = blockIdx.z / a.S, ks = blockIdx.z - zz * a.S;
  int gi = 0;
#pragma unroll
  for (int i = 1; i < TG_MAXG; ++i) if (i < a.G && zz >= a.g[i].z0) gi = i;
  const TgGroup& g = a.g[gi];
  const int z = zz - g.z0;
  const int m0 = blockIdx.x * TG_BM, n0 = blockIdx.y * TG_BN;
  const int kbeg = ks * a.kchunk, kend = min(a.K, kbeg + a.kchunk);
  const int nk = kend > kbeg ? ceil_div(kend - kbeg, TG_BK) : 0;
  // Programmatic dependent launch: nothing below reads or writes before the previous kernel has completed.
  pdl_prologue();
  const float* A = g.A + z * g.sAz;
  const float* B = g.B + z * g.sBz;

  auto issue = [&](int kt) {
    const uint32_t dst = t_smem(sRaw + (kt % TG_RAW) * TG_STAGE);
    const int k0 = kbeg + kt * TG_BK;
    t_issue_raw<TG_BM>(dst, A, a.M, m0, g.sAm, g.sAk, k0, kend, a.a_mode, tid);
    t_issue_raw<TG_BN>(dst + TG_A_STAGE, B, a.N, n0, g.sBn, g.sBk, k0, kend, a.b_mode, tid);
  };
#pragma unroll
  for (int st = 0; st < TG_RAW - 1; ++st) {
    if (st < nk) issue(st);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  const bool ln = a.epi >= SERL_TGEMM_EPI_LN_TANH && a.epi <= SERL_TGEMM_EPI_LN_TANH_POLICY;
  // stage the epilogue vectors while the first operands are in flight
  if (!a.to_ws) {
    const float* bias = g.bias ? g.bias + z * g.sBiasZ : nullptr;
    for (int c = tid; c < TG_BN; c += TG_EPI_THREADS) {
      const int n = n0 + c;
      sBias[c] = (bias && n < a.N) ? bias[n] : 0.f;
      if (ln) { sLs[c] = g.ln_scale[z * g.sLnZ + n]; sLb[c] = g.ln_bias[z * g.sLnZ + n]; }
    }
    if (ln && a.epi >= SERL_TGEMM_EPI_LN_TANH_HEAD) {
      const float* hw = g.head_w + z * g.sHeadWz;
      for (int i = tid; i < TG_BN * a.head_n; i += TG_EPI_THREADS) sHw[i] = hw[i];
      if (tid < a.head_n) sHb[tid] = g.head_b ? g.head_b[z * g.sHeadBz + tid] : 0.f;
      if (a.epi == SERL_TGEMM_EPI_LN_TANH_POLICY) {
        for (int i = tid; i < TG_BN * a.head_n; i += TG_EPI_THREADS) sHw2[i] = g.head_w2[i];
        if (tid < a.head_n) sHb[8 + tid] = g.head_b2 ? g.head_b2[tid] : 0.f;
      }
    }
  }

  // ---- main loop: warpgroup wg computes rows [64 wg, 64 wg + 64) x 256 columns (four m64n64 n-chunks) ----
  float acc[4][32];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
  for (int kt = 0; kt < nk; ++kt) {
    asm volatile("cp.async.wait_group %0;" ::"n"(TG_RAW - 2) : "memory");
    __syncthreads();                                                     // raw stage kt landed; the MMAs of kt-1 retired
    if (kt + TG_RAW - 1 < nk) issue(kt + TG_RAW - 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    const float* raw = reinterpret_cast<const float*>(sRaw + (kt % TG_RAW) * TG_STAGE);
    // fp32 x = hi + lo, hi = tf32 round-to-nearest of x, lo exact: K-major 128B-swizzled
    t_convert<TG_BM>(raw, sOp, sOp + TG_STAGE, (a.a_mode & 1) != 0, tid);
    t_convert<TG_BN>(raw + TG_BM * TG_BK, sOp + TG_A_STAGE, sOp + TG_STAGE + TG_A_STAGE, (a.b_mode & 1) != 0, tid);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint32_t sa = t_smem(sOp) + wg * 8192, sb = t_smem(sOp + TG_A_STAGE), lo = TG_STAGE;
    wg_fence();
    // a_lo b_hi + a_hi b_lo + a_hi b_hi ("3xTF32"): ~2^-22 per product, the accuracy of an fp32 FMA
#pragma unroll
    for (int k = 0; k < TG_BK / 8; ++k)                                  // k-step = 8 tf32 = 32 B: start address + 2 (x16 B)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const uint64_t ah = wg_desc(sa) + 2 * k, al = wg_desc(sa + lo) + 2 * k;
        const uint64_t bh = wg_desc(sb + c * 8192) + 2 * k, bl = wg_desc(sb + lo + c * 8192) + 2 * k;
        wg_mma_tf32(acc[c], al, bh, 1u);
        wg_mma_tf32(acc[c], ah, bl, 1u);
        wg_mma_tf32(acc[c], ah, bh, 1u);
      }
    wg_commit();
    wg_wait<0>();
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();                                                       // every MMA and copy is done: the work area is free

  // ---- accumulators -> shared tile [128 rows][256 columns] fp32, 16-byte chunks XOR-swizzled by (row & 7) ----
  float* sAcc = reinterpret_cast<float*>(smem);
  {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = c * 64 + 8 * j + 2 * (lane & 3);
          *reinterpret_cast<float2*>(sAcc + r * TG_BN + (col ^ ((r & 7) << 2))) = make_float2(acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]);
        }
    }
  }
  __syncthreads();

  {
    // =============================== epilogue: 8 warps, thread = (output row, column half) ===============================
    // Two warps per 32-row quarter, 128 columns each: with one warp per scheduler the dependent chains of the LayerNorm /
    // tanh arithmetic ran at a fraction of the issue rate; the two halves of a row meet through shared memory.
    const int q = warp & 3;                                              // row quarter of this warp
    const int hh = warp >> 2;                                            // column half
    const int row = q * 32 + lane, m = m0 + row;
    const int c_lo = hh * (TG_BN / 2), c_hi = c_lo + TG_BN / 2;
    const bool have = nk > 0;
    const float* accrow = sAcc + row * TG_BN;
    const int sw = (row & 7) << 2;
    auto tg_ld32 = [&](int c, float (&v)[32]) {                           // columns c .. c + 31 of this thread's row
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 f = *reinterpret_cast<const float4*>(accrow + ((c + 4 * i) ^ sw));
        v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w;
      }
    };
    uint8_t* sEpi = smem + TG_ACC;
    float* sPart = reinterpret_cast<float*>(sEpi);                       // [2 halves][128 rows][2]: sum, sum of squares
    float* sHeadPart = sPart + 2 * TG_BM * 2;                            // [128 rows][16]: half 1's head partial sums
    // Output rows leave through a per-warp staging tile (32 rows x 32 columns, 16-byte chunks XOR-swizzled by row): a thread owns
    // a ROW of the accumulator, so direct stores put the 32 lanes of an instruction on 32 different lines; staged, one
    // instruction writes 4 rows x 128 contiguous bytes.
    float* sTile = sHeadPart + TG_BM * 16 + warp * 2048;                 // two tiles per warp: activation | xhat
    const int row_w = m0 + q * 32;                                       // first global row of this warp
    auto stage = [&](float* tile, const float (&v)[32]) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<float4*>(tile + lane * 32 + ((j ^ (lane & 7)) << 2)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    };
    auto flush = [&](const float* tile, float* gbase, long long ld, int col, bool acc, bool live) {
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int rr = 4 * i + (lane >> 3), j = lane & 7;
        float4 o = *reinterpret_cast<const float4*>(tile + rr * 32 + ((j ^ (rr & 7)) << 2));
        if (live && row_w + rr < a.M) {
          float4* p = reinterpret_cast<float4*>(gbase + (size_t)(row_w + rr) * ld + col + 4 * j);
          if (acc) { const float4 old = *p; o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w; }
          *p = o;
        }
      }
      __syncwarp();
    };
    if (a.to_ws || !ln) {
      float* dst; long long ld;
      if (a.to_ws) { dst = a.ws + ((size_t)blockIdx.z * a.M) * a.N; ld = a.N; }
      else { dst = g.C + z * g.sCz; ld = g.ldc; }
      const bool vec = ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) && (ld % 4 == 0);
      const bool acc = !a.to_ws && a.accumulate;
#pragma unroll 1
      for (int c = c_lo; c < c_hi; c += 32) {
        if (n0 + c >= a.N) break;                                        // warp-uniform
        float v[32];
        tg_ld32(c, v);
        if (vec && n0 + c + 32 <= a.N) {                                 // warp-uniform
          if (!a.to_ws) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] += sBias[c + i];
          }
          stage(sTile, v);
          flush(sTile, dst, ld, n0 + c, acc, true);
        } else if (m < a.M) {
          float* rowp = dst + (size_t)m * ld + n0 + c;
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            if (n0 + c + i < a.N) {
              float o = v[i] + (a.to_ws ? 0.f : sBias[c + i]);
              rowp[i] = acc ? rowp[i] + o : o;
            }
          }
        }
      }
    } else {
      // ---- bias + LayerNorm + tanh (N == 256: a row = this thread's 128 columns + its partner's) ----
      float s = 0.f, ss = 0.f;
#pragma unroll 1
      for (int c = c_lo; c < c_hi; c += 32) {
        float v[32];
        tg_ld32(c, v);
        if constexpr (kMask) {
          tg_drop32(mk.mask[gi], m, a.M, c, sBias, mk.inv_keep, v);
#pragma unroll
          for (int i = 0; i < 32; ++i) { s += v[i]; ss += v[i] * v[i]; }
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) { const float x = v[i] + sBias[c + i]; s += x; ss += x * x; }
        }
      }
      *reinterpret_cast<float2*>(sPart + (hh * TG_BM + row) * 2) = make_float2(s, ss);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      {
        const float2 o = *reinterpret_cast<const float2*>(sPart + ((hh ^ 1) * TG_BM + row) * 2);
        // fixed summation order (half 0 + half 1) so that both threads of a row hold bit-identical statistics
        const float2 p0 = hh ? o : make_float2(s, ss), p1 = hh ? make_float2(s, ss) : o;
        s = p0.x + p1.x; ss = p0.y + p1.y;
      }
      const float mean = s * (1.f / TG_BN);
      const float var = fmaxf(ss * (1.f / TG_BN) - mean * mean, 0.f);
      const float rstd = rsqrtf(var + a.eps);
      float hacc[2 * TG_MAXHEAD];
#pragma unroll
      for (int i = 0; i < 2 * TG_MAXHEAD; ++i) hacc[i] = 0.f;
      float* hbase = g.C ? g.C + z * g.sCz : nullptr;
      float* xbase = g.xhat ? g.xhat + z * g.sXhatZ : nullptr;
      const bool hvec = hbase && ((reinterpret_cast<uintptr_t>(hbase) & 15) == 0) && (g.ldc % 4 == 0);
      const bool valid = have && m < a.M;
#pragma unroll 1
      for (int c = c_lo; c < c_hi; c += 32) {
        float v[32];
        tg_ld32(c, v);
        if constexpr (kMask) tg_drop32(mk.mask[gi], m, a.M, c, sBias, mk.inv_keep, v);
        float h[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const float xh = ((kMask ? v[i] : v[i] + sBias[c + i]) - mean) * rstd;
          v[i] = xh;
          h[i] = tg_tanh(fmaf(xh, sLs[c + i], sLb[c + i]));
        }
        if (hbase) {
          if (hvec) { stage(sTile, h); flush(sTile, hbase, g.ldc, c, false, have); }
          else if (valid) {
#pragma unroll
            for (int i = 0; i < 32; ++i) hbase[(size_t)m * g.ldc + c + i] = h[i];
          }
        }
        if (xbase) { stage(sTile + 1024, v); flush(sTile + 1024, xbase, TG_BN, c, false, have); }
        if (a.epi >= SERL_TGEMM_EPI_LN_TANH_HEAD) {
#pragma unroll
          for (int j = 0; j < TG_MAXHEAD; ++j) {
            if (j < a.head_n) {
              float t = hacc[j], t2 = hacc[TG_MAXHEAD + j];
#pragma unroll
              for (int i = 0; i < 32; ++i) {
                t = fmaf(h[i], sHw[(c + i) * a.head_n + j], t);
                if (a.epi == SERL_TGEMM_EPI_LN_TANH_POLICY) t2 = fmaf(h[i], sHw2[(c + i) * a.head_n + j], t2);
              }
              hacc[j] = t; hacc[TG_MAXHEAD + j] = t2;
            }
          }
        }
      }
      if (valid && g.rstd && hh == 0) g.rstd[z * g.sRstdZ + m] = rstd;
      if (a.epi >= SERL_TGEMM_EPI_LN_TANH_HEAD) {
        // half 1 hands its partial head sums to half 0, which finishes the row
        if (hh == 1) {
#pragma unroll
          for (int j = 0; j < 2 * TG_MAXHEAD; ++j) sHeadPart[row * 16 + j] = hacc[j];
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (hh == 0) {
#pragma unroll
          for (int j = 0; j < 2 * TG_MAXHEAD; ++j) hacc[j] += sHeadPart[row * 16 + j];
        }
      }
      if (valid && hh == 0) {
        if (a.epi == SERL_TGEMM_EPI_LN_TANH_HEAD) {
          float* o = g.head_out + z * g.sHeadOutZ + (size_t)m * g.ld_head;
#pragma unroll
          for (int j = 0; j < TG_MAXHEAD; ++j) if (j < a.head_n) o[j] = hacc[j] + sHb[j];
        } else if (a.epi == SERL_TGEMM_EPI_LN_TANH_POLICY) {
          // means / log-stds -> tanh-Gaussian sample and its log-probability (same arithmetic as tanh_gaussian_fwd_kernel, sac_ops.cu)
          const int A = a.head_n;
          float lp = 0.f;
#pragma unroll
          for (int j = 0; j < TG_MAXHEAD; ++j) {
            if (j >= A) break;
            const float mu = hacc[j] + sHb[j], lsd = hacc[TG_MAXHEAD + j] + sHb[8 + j];
            if (g.head_out) g.head_out[(size_t)m * A + j] = mu;
            if (g.head_out2) g.head_out2[(size_t)m * A + j] = lsd;
            const float sd = fminf(fmaxf(expf(lsd), a.std_min), a.std_max);
            const float e = a.deterministic ? 0.f : g.noise[(size_t)m * A + j];
            const float u = mu + sd * e;
            const float zn = (u - mu) / sd;
            lp += -0.5f * zn * zn - logf(sd) - 0.918938533204672742f;
            lp -= 2.f * (0.693147180559945309f - u - tg_softplus(-2.f * u));
            g.act[(size_t)m * g.ld_act + j] = tanhf(u);
            if (g.u_out) g.u_out[(size_t)m * A + j] = u;
            if (g.std_out) g.std_out[(size_t)m * A + j] = sd;
          }
          if (g.logp) g.logp[m] = lp;
        }
      }
    }
  }
}


// Operand seen as (rows R, depth K) with element (r, k) at base + z*sZ + r*sR + k*sK (floats): K-major (sK == 1) or
// MN-major (sR == 1), 16-byte aligned, the other stride a multiple of 4 floats -> staging mode 0 / 1 of t_issue_raw.
static bool tg_operand(const float* base, int R, int K, int Z, long long sZ, long long sR, long long sK, int* mode) {
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return false;
  const bool kmaj = (sK == 1) && (sR % 4 == 0) && sR >= K;
  const bool mmaj = (sR == 1) && (sK % 4 == 0) && sK >= R;
  if (!kmaj && !mmaj) return false;
  if (Z > 1 && sZ != 0 && sZ % 4 != 0) return false;
  *mode = kmaj ? 0 : 1;
  return true;
}

}  // namespace serl

using namespace serl;

// masks: NULL (tgemm_tf32_kernel<false>) or, for a LayerNorm epilogue, one (M, 256) keep mask per problem (tgemm_tf32_kernel<true>)
static int tg_launch(const serl_tgemm_desc* d, const uint8_t* const* masks, float inv_keep, void* stream) {
  if (!d || !d->problems || d->num_problems < 1 || d->num_problems > TG_MAXG || d->M < 1 || d->N < 1 || d->K < 1) {
    set_last_error("serl_tgemm_tf32: invalid descriptor"); return SERL_ERR_INVALID;
  }
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(tgemm_tf32_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM) != cudaSuccess ||
        cudaFuncSetAttribute(tgemm_tf32_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM) != cudaSuccess) {
      set_last_error("serl_tgemm_tf32: cannot reserve %d bytes of shared memory", TG_SMEM); return SERL_ERR_CUDA;
    }
    attr_done = true;
  }
  const bool ln = d->epilogue >= SERL_TGEMM_EPI_LN_TANH && d->epilogue <= SERL_TGEMM_EPI_LN_TANH_POLICY;
  const bool partial = d->epilogue == SERL_TGEMM_EPI_PARTIAL;
  if (d->epilogue < 0 || d->epilogue > SERL_TGEMM_EPI_PARTIAL) { set_last_error("serl_tgemm_tf32: unknown epilogue %d", d->epilogue); return SERL_ERR_INVALID; }
  if (ln && (d->N != TG_BN || d->reduce_z || d->splits > 1)) { set_last_error("serl_tgemm_tf32: LayerNorm epilogues need N == 256, no k-split, no reduce_z"); return SERL_ERR_UNSUPPORTED; }
  if (ln && d->epilogue >= SERL_TGEMM_EPI_LN_TANH_HEAD && (d->head_n < 1 || d->head_n > TG_MAXHEAD)) { set_last_error("serl_tgemm_tf32: head_n in [1, 8]"); return SERL_ERR_UNSUPPORTED; }
  TgMask mk{};
  if (masks) {
    if (!ln || !(inv_keep > 0.f)) { set_last_error("serl_tgemm_tf32_masked: a LayerNorm epilogue and inv_keep > 0 required"); return SERL_ERR_INVALID; }
    for (int i = 0; i < d->num_problems; ++i) {
      if (!masks[i] || (reinterpret_cast<uintptr_t>(masks[i]) & 15) != 0) {
        set_last_error("serl_tgemm_tf32_masked: problem %d: a 16-byte aligned (M, 256) mask required", i); return SERL_ERR_INVALID;
      }
      mk.mask[i] = masks[i];
    }
    mk.inv_keep = inv_keep;
  }
  TgArgs a{};
  a.G = d->num_problems; a.M = d->M; a.N = d->N; a.K = d->K; a.epi = d->epilogue; a.accumulate = d->accumulate; a.head_n = d->head_n;
  a.eps = d->ln_eps; a.std_min = d->std_min; a.std_max = d->std_max; a.deterministic = d->deterministic; a.error = d->error;
  int ztotal = 0;
  for (int i = 0; i < d->num_problems; ++i) {
    const serl_tgemm_problem& p = d->problems[i];
    TgGroup& g = a.g[i];
    if (!p.A || !p.B || p.Z < 1) { set_last_error("serl_tgemm_tf32: problem %d: A, B, Z required", i); return SERL_ERR_INVALID; }
    int amode = 0, bmode = 0;
    if (!tg_operand(p.A, d->M, d->K, p.Z, p.sAz, p.sAm, p.sAk, &amode) || !tg_operand(p.B, d->N, d->K, p.Z, p.sBz, p.sBn, p.sBk, &bmode)) {
      set_last_error("serl_tgemm_tf32: problem %d: operands must be 16-byte aligned with one unit stride and the other a multiple of 4 floats", i);
      return SERL_ERR_UNSUPPORTED;
    }
    if (i == 0) { a.a_mode = amode; a.b_mode = bmode; }
    else if (a.a_mode != amode || a.b_mode != bmode) { set_last_error("serl_tgemm_tf32: all problems of a launch share the operand layouts"); return SERL_ERR_UNSUPPORTED; }
    g.A = p.A; g.B = p.B; g.sAz = p.sAz; g.sAm = p.sAm; g.sAk = p.sAk; g.sBz = p.sBz; g.sBn = p.sBn; g.sBk = p.sBk;
    g.C = p.C; g.bias = p.bias; g.ln_scale = p.ln_scale; g.ln_bias = p.ln_bias; g.xhat = p.xhat; g.rstd = p.rstd;
    g.head_w = p.head_w; g.head_b = p.head_b; g.head_out = p.head_out; g.head_w2 = p.head_w2; g.head_b2 = p.head_b2; g.head_out2 = p.head_out2;
    g.noise = p.noise; g.act = p.act; g.logp = p.logp; g.u_out = p.u_out; g.std_out = p.std_out;
    g.sCz = p.sCz; g.sBiasZ = p.sBiasZ; g.sLnZ = p.sLnZ; g.sXhatZ = p.sXhatZ; g.sRstdZ = p.sRstdZ; g.sHeadWz = p.sHeadWz; g.sHeadBz = p.sHeadBz;
    g.sHeadOutZ = p.sHeadOutZ; g.ldc = p.ldc; g.ld_head = p.ld_head; g.ld_act = p.ld_act; g.z0 = ztotal; g.Z = p.Z;
    if (!d->reduce_z && !p.C && !ln && !partial) { set_last_error("serl_tgemm_tf32: problem %d: C required", i); return SERL_ERR_INVALID; }
    if (ln && (!p.ln_scale || !p.ln_bias)) { set_last_error("serl_tgemm_tf32: problem %d: LayerNorm scale / bias required", i); return SERL_ERR_INVALID; }
    if (ln && d->epilogue >= SERL_TGEMM_EPI_LN_TANH_HEAD && (!p.head_w || !p.head_out)) { set_last_error("serl_tgemm_tf32: problem %d: head_w / head_out required", i); return SERL_ERR_INVALID; }
    if (d->epilogue == SERL_TGEMM_EPI_LN_TANH_POLICY && (!p.head_w2 || !p.act || (!d->deterministic && !p.noise) || p.Z != 1)) {
      set_last_error("serl_tgemm_tf32: problem %d: policy epilogue needs head_w2, act, noise and Z == 1", i); return SERL_ERR_INVALID;
    }
    ztotal += p.Z;
  }
  // k-splits: these GEMMs are tiny (<= 1 GFLOP); with fewer tiles than SMs split K until about one wave exists
  const int tiles = ceil_div(d->M, TG_BM) * ceil_div(d->N, TG_BN) * ztotal;
  int S = 1;
  if (!ln) {
    if (d->splits > 0) S = d->splits;
    else if (tiles < 66 && d->K >= 512) { S = 132 / tiles; if (S > d->K / 128) S = d->K / 128; if (S < 1) S = 1; }
  }
  const size_t part = (size_t)d->M * d->N * sizeof(float);
  if (partial) {
    // the caller reduces: partial products of split s of member zz (counted across the problems) at workspace[(zz * S + s)][M][N]
    S = d->splits > 0 ? d->splits : 1;
    if (d->reduce_z || !d->workspace) { set_last_error("serl_tgemm_tf32: the PARTIAL epilogue needs a workspace and no reduce_z"); return SERL_ERR_INVALID; }
    const int kc = ceil_div(ceil_div(d->K, S), TG_BK) * TG_BK;
    if (ceil_div(d->K, kc) != S) { set_last_error("serl_tgemm_tf32: %d splits of K = %d leave empty splits", S, d->K); return SERL_ERR_INVALID; }
    if (part * (size_t)ztotal * S > d->workspace_bytes) { set_last_error("serl_tgemm_tf32: PARTIAL needs %zu workspace bytes", part * (size_t)ztotal * S); return SERL_ERR_INVALID; }
  } else if (d->reduce_z || S > 1) {
    if (d->num_problems != 1) { set_last_error("serl_tgemm_tf32: k-split / reduce_z launches take one problem"); return SERL_ERR_UNSUPPORTED; }
    while (S > 1 && part * (size_t)ztotal * S > d->workspace_bytes) --S;
    if (!d->workspace || part * (size_t)ztotal * S > d->workspace_bytes) {
      if (d->reduce_z) { set_last_error("serl_tgemm_tf32: reduce_z needs %zu workspace bytes", part * (size_t)ztotal); return SERL_ERR_INVALID; }
      S = 1;
    }
  }
  a.kchunk = ceil_div(ceil_div(d->K, S), TG_BK) * TG_BK;
  S = ceil_div(d->K, a.kchunk);
  a.S = S;
  a.to_ws = (partial || d->reduce_z || S > 1) ? 1 : 0;
  a.ws = d->workspace;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(ceil_div(d->M, TG_BM), ceil_div(d->N, TG_BN), ztotal * S);
  if (masks) {
    launch_k(tgemm_tf32_kernel<true>, grid, TG_THREADS, TG_SMEM, st, a, mk);
    return check_launch("tgemm_tf32_kernel<mask>");             // (LayerNorm epilogues: no k-split, nothing to reduce)
  }
  launch_k(tgemm_tf32_kernel<false>, grid, TG_THREADS, TG_SMEM, st, a, mk);
  if (int e = check_launch("tgemm_tf32_kernel")) return e;
  if (a.to_ws && !partial) {
    const serl_tgemm_problem& p = d->problems[0];
    GemmArgs r{};
    r.C = p.C; r.bias = p.bias; r.ws = d->workspace; r.M = d->M; r.N = d->N; r.K = d->K; r.Z = p.Z; r.S = S;
    r.sCz = p.sCz; r.sBiasZ = p.sBiasZ; r.ldc = p.ldc; r.accumulate = d->accumulate;
    return launch_gemm_reduce(r, d->reduce_z, st);
  }
  return SERL_OK;
}

extern "C" int serl_tgemm_tf32(const serl_tgemm_desc* d, void* stream) { return tg_launch(d, nullptr, 1.f, stream); }

extern "C" int serl_tgemm_tf32_masked(const serl_tgemm_desc* d, const uint8_t* const* masks, float inv_keep, void* stream) {
  if (!masks) { set_last_error("serl_tgemm_tf32_masked: masks required"); return SERL_ERR_INVALID; }
  return tg_launch(d, masks, inv_keep, stream);
}
