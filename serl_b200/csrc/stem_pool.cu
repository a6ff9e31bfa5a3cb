// conv_init of the 16-bit trunk fused with the 3x3/2 SAME max-pool that follows its GroupNorm + ReLU
// (vision/resnet_v1.py:247-261): the 64x64x64 conv output never reaches HBM.
//
// The 7x7/2 conv is computed exactly as a 4x4/1 conv over the 2x2 space-to-depth image xs (N,67,67,16) that
// serl_trunk_stem_prep_h16 writes (12 real + 4 zero channels, padding materialised), K = 4 kernel rows x 4 taps x 16 ch.
#include "common.cuh"
#include "conv_common.cuh"
#include "serl_b200.h"
#include "wgmma.cuh"

namespace serl {

// ---------------------------------------------------------------------------------------------------------------------------
// stem_pool_kernel: one cluster of 4 CTAs per image, CTA rank k owns conv rows 16k..16k+15 (pooled rows 8k..8k+7), walked as
// four chunks of 4 conv rows = 256 output pixels x 64 channels.
// Roles (288 threads): warpgroups 0 and 1 issue the MMAs (m64 n64 k16, 128 pixels each: 64 fp32 accumulators per thread) and
// run the epilogue; warp 8 issues the TMA loads.
// Operands:
//   weights   the packed [64][256] stem weight (32 KB, 128B swizzle), loaded once and kept resident;
//   input     per chunk, four boxes of 16 ch x 64 cols x 7 rows of xs at x offsets s' = 0..3 (32-byte rows, 32B swizzle).
//             Tap (r', s') is box s' shifted by r' rows = r' x 2048 bytes, a whole number of swizzle atoms, so every A tile is
//             a plain descriptor.  The 16 taps are issued r' outer, s' inner, one k16 step each: the exact sequence of the
//             raw stem conv (conv_tc_kernel, kStem), so the fp32 accumulators and every 16-bit value equal that conv's bit
//             for bit.  The boxes form a 2-stage ring, so the next chunk (or image) loads during this chunk's taps.
// Epilogue: the sign-adjusted 16-bit values (bit c of neg_mask set <=> GroupNorm scale of channel c negative, so max commutes
// with relu(a x + b)) go to one of two staging tiles; the 3x3/2 pooling of a chunk runs while the next chunk's MMAs are in
// flight.  Per CTA: pooled rows 8k..8k+6 are complete; row 8k+7 holds max(conv 16k+14, 16k+15) and side[k] the column-pooled
// conv row 16k, which serl_pool_finish_h16 joins (row 31 is complete: row 64 is padding).
// GroupNorm sums: per-thread sums over the image's fragments, warp shuffles, warps in order; every CTA writes its partials into
// each peer's shared memory (st.async, transaction mbarrier) and rank 0 adds the rank-ordered total into stats once (stats is
// zeroed per pass), so the statistics are deterministic.  The producer thread runs the exchange, one image behind the MMAs.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int SP_THREADS = 288;
constexpr int SP_BOX = 7 * 64 * 32;                      // one 16 ch x 64 col x 7 row box: 14 KB
constexpr int SP_STAGE = 4 * SP_BOX;                     // the four x offsets of one chunk
constexpr int SP_STAGES = 2;
constexpr int SP_OFF_A = 4 * 8192;                       // after the resident weight (4 kernel rows x [64 co][64 K])
constexpr int SP_OFF_STG = SP_OFF_A + SP_STAGES * SP_STAGE;        // 2 x [256 px][64 ch] 16-bit staging tiles
constexpr int SP_OFF_RED = SP_OFF_STG + 2 * 256 * 128;             // [8 warps][4 groups][2] warp partial sums of an image
constexpr int SP_OFF_SLOT = SP_OFF_RED + 8 * 8 * 4;                // [2 image parities][4 ranks][4 groups][2] CTA partials
constexpr int SP_OFF_BAR = SP_OFF_SLOT + 2 * 4 * 8 * 4;
constexpr int SP_SMEM = SP_OFF_BAR + 8 * (2 * SP_STAGES + 4) + 1024;   // + alignment of the dynamic base to 1024
static_assert((SP_BOX % 1024) == 0 && SP_SMEM <= 232448, "stem_pool_kernel: shared memory layout");

struct StemPoolArgs {
  uint32_t* pooled; uint32_t* side; float* stats; int32_t* error;   // pooled / side as pairs of 16-bit channels
  unsigned long long neg_mask; int N;
};

__device__ inline bool sp_bar_and(bool v) {              // named barrier over the 256 MMA threads, ANDs a flag across them
  uint32_t r;
  asm volatile("{\n .reg .pred p, q;\n setp.ne.u32 p, %1, 0;\n barrier.red.and.pred q, 1, 256, p;\n selp.u32 %0, 1, 0, q;\n}"
               : "=r"(r) : "r"((uint32_t)v) : "memory");
  return r != 0;
}

template <class F>
__global__ void __launch_bounds__(SP_THREADS, 1)
stem_pool_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap wmap, const StemPoolArgs a) {
  pdl_prologue();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sW = smem;
  uint8_t* sA = smem + SP_OFF_A;
  uint32_t* stg = reinterpret_cast<uint32_t*>(smem + SP_OFF_STG);
  float* red = reinterpret_cast<float*>(smem + SP_OFF_RED);
  float* slot = reinterpret_cast<float*>(smem + SP_OFF_SLOT);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + SP_OFF_BAR);
  uint64_t* empty = full + SP_STAGES;
  uint64_t* wbar = empty + SP_STAGES;
  uint64_t* redbar = wbar + 1;                               // red holds an image's warp partials (one arrival per MMA warp)
  uint64_t* gnbar = redbar + 1;                              // [2]: the cluster exchange, one per image parity

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int band = blockIdx.x & 3;                           // rank in the cluster
  const int img0 = blockIdx.x >> 2, img_step = gridDim.x >> 2;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SP_STAGES; ++s) { tc_mbar_init(&full[s], 1); tc_mbar_init(&empty[s], 8); }
    tc_mbar_init(wbar, 1); tc_mbar_init(redbar, 8); tc_mbar_init(&gnbar[0], 1); tc_mbar_init(&gnbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  asm volatile("barrier.cluster.arrive.release;\n barrier.cluster.wait.acquire;" ::: "memory");   // peers' st.async target gnbar

  if (warp == 8) {
    // ------------------------------- TMA producer + GroupNorm exchange -------------------------------
    if (lane == 0) {
      // rank 0: the rank-ordered GroupNorm total of image n (the cluster's item-th) into stats, once every rank's partials arrived
      auto collect = [&](int n, int item) -> bool {
        const int par = item & 1;
        if (!tc_mbar_wait_cluster(&gnbar[par], (uint32_t)(item >> 1) & 1u, a.error)) return false;
        for (int q = 0; q < 8; ++q) {
          float v = 0.f;
          for (int rk = 0; rk < 4; ++rk) v += slot[(par * 4 + rk) * 8 + q];
          if (band == 0) atomicAdd(a.stats + (size_t)n * 8 + q, v);
        }
        return true;
      };
      // once the MMA warps have left image n's partials in red: collect the previous image, send this one's partials into
      // every CTA of the cluster (this one included).  A peer sends image t only after collecting t - 1, which needs this
      // CTA's t - 1, sent after this CTA collected t - 2: so a slot parity is never overwritten before it was read.
      auto exchange = [&](int n, int item) -> bool {
        const int par = item & 1;
        if (!tc_mbar_wait(redbar, (uint32_t)item & 1u, a.error)) return false;
        float v[8];
        for (int q = 0; q < 8; ++q) {
          v[q] = 0.f;
          for (int w = 0; w < 8; ++w) v[q] += red[w * 8 + q];
        }
        if (item > 0 && !collect(n - img_step, item - 1)) return false;
        tc_mbar_expect_tx(&gnbar[par], 4u * 8u * 4u);
        for (int rk = 0; rk < 4; ++rk) {
          uint32_t rdst, rbar;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rdst) : "r"(smem_u32(slot + (par * 4 + band) * 8)), "r"(rk));
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbar) : "r"(smem_u32(&gnbar[par])), "r"(rk));
          for (int q = 0; q < 8; ++q)
            asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
                         ::"r"(rdst + 4u * q), "r"(__float_as_uint(v[q])), "r"(rbar) : "memory");
        }
        return true;
      };
      asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
      tc_mbar_expect_tx(wbar, 4u * 8192u);
      for (int t = 0; t < 4; ++t) tc_tma_2d(sW + t * 8192, &wmap, t * 64, 0, wbar);
      bool ok = true;
      int it = 0;
      for (;; ++it) {
        const int n = img0 + (it >> 2) * img_step, c = it & 3;
        if (n >= a.N) break;
        // the previous image's partials are in red long before this chunk's stage frees up; handling them here also keeps
        // the MMA warps from writing red again before it was read
        if (c == 2 && it > 4 && !(ok = exchange(n - img_step, (it >> 2) - 1))) break;
        const int s = it % SP_STAGES;
        if (!(ok = tc_mbar_wait(&empty[s], ((uint32_t)(it / SP_STAGES) & 1u) ^ 1u, a.error))) break;
        tc_mbar_expect_tx(&full[s], (uint32_t)SP_STAGE);
        for (int sx = 0; sx < 4; ++sx)                       // xs rows 16 band + 4 c .. + 6, columns sx .. sx + 63
          tc_tma_4d(sA + s * SP_STAGE + sx * SP_BOX, &xmap, 0, sx, 16 * band + 4 * c, n, &full[s]);
      }
      if (ok && it > 0) {                                    // the last image (it is a multiple of 4 here)
        const int item = (it >> 2) - 1, n = img0 + item * img_step;
        if (exchange(n, item)) collect(n, item);
      }
    }
  } else {
    // ------------------------------- MMA + epilogue (warpgroups 0, 1) -------------------------------
    const int tid = threadIdx.x, wg = tid >> 7, wl = warp & 3;
    const uint32_t a_base = smem_u32(sA) + (uint32_t)(wg * 128 * 32), w_base = smem_u32(sW);
    uint32_t flip[8];                                        // sign flips of this thread's channel pairs 8 j + 2 (lane % 4)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = 8 * j + 2 * (lane & 3);
      flip[j] = (uint32_t)((a.neg_mask >> ch) & 1ull) * 0x8000u | (uint32_t)((a.neg_mask >> (ch + 1)) & 1ull) * 0x80000000u;
    }
    // pooling: this thread owns pooled columns u = warp + 8 i (i = 0..3), channel pair `lane`; carry[i] = column-pooled
    // max(conv rows 4c + 2, 4c + 3) of the previous chunk
    uint32_t carry[4] = {0u, 0u, 0u, 0u};
    auto pool = [&](const uint32_t* t, int n, int c) {
      auto at = [&](int pix) { return t[pix * 32 + (((lane >> 2) ^ (pix & 7)) << 2) + (lane & 3)]; };
      uint32_t* out = a.pooled + (size_t)n * 32 * 32 * 32;
      const int p0 = 8 * band + 2 * c;                       // pooled row of conv rows 4c .. 4c + 2 of this chunk
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int u = warp + 8 * i, x0 = 2 * u, nx = u == 31 ? 2 : 3;   // SAME: the window of column 31 ends at the edge
        uint32_t b0 = at(x0);
        for (int dx = 1; dx < nx; ++dx) b0 = F::max2(b0, at(x0 + dx));
        uint32_t a01 = b0;
        for (int dx = 0; dx < nx; ++dx) a01 = F::max2(a01, at(64 + x0 + dx));
        uint32_t b2 = at(128 + x0);
        for (int dx = 1; dx < nx; ++dx) b2 = F::max2(b2, at(128 + x0 + dx));
        uint32_t a23 = b2;
        for (int dx = 0; dx < nx; ++dx) a23 = F::max2(a23, at(192 + x0 + dx));
        if (c > 0) out[((size_t)(p0 - 1) * 32 + u) * 32 + lane] = F::max2(carry[i], b0);
        else a.side[(((size_t)n * 4 + band) * 32 + u) * 32 + lane] = b0;
        out[((size_t)p0 * 32 + u) * 32 + lane] = F::max2(a01, b2);
        if (c == 3) out[((size_t)(p0 + 1) * 32 + u) * 32 + lane] = a23;
        carry[i] = a23;
      }
    };
    bool ok = tc_mbar_wait(wbar, 0u, a.error);
    ok = sp_bar_and(ok);
    float gs[4] = {0.f, 0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f};
    int it = 0, prev_n = -1;
    for (; ok; ++it) {
      const int n = img0 + (it >> 2) * img_step, c = it & 3, s = it % SP_STAGES;
      if (n >= a.N) break;
      float acc[2][32];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
      ok = tc_mbar_wait(&full[s], (uint32_t)(it / SP_STAGES) & 1u, a.error);
      if (!ok) break;
      const uint32_t as = a_base + (uint32_t)(s * SP_STAGE);
      wg_fence();
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int sx = 0; sx < 4; ++sx)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            wg_mma_h16<F::kBf16>(acc[h], wg_desc_sw32(as + (uint32_t)(sx * SP_BOX + (h * 64 + r * 64) * 32)),
                                 wg_desc(w_base + (uint32_t)(r * 8192)) + 2 * sx, 1u);
      wg_commit();
      if (it > 0) pool(stg + ((it - 1) & 1) * 256 * 32, prev_n, (it - 1) & 3);   // the previous chunk, under this one's MMAs
      wg_wait<0>();
      __syncwarp();
      if (lane == 0) tc_mbar_arrive(&empty[s]);
      // fragment: acc[h][4 j + 2 hf + e] = pixel 128 wg + 64 h + 16 wl + 8 hf + lane / 4, channel 8 j + 2 (lane % 4) + e
      if (c == 0) {
#pragma unroll
        for (int g = 0; g < 4; ++g) { gs[g] = 0.f; gq[g] = 0.f; }
      }
      uint32_t* t = stg + (it & 1) * 256 * 32;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float* d = &acc[h][4 * j];
          gs[j >> 1] += (d[0] + d[1]) + (d[2] + d[3]);
          gq[j >> 1] += (d[0] * d[0] + d[1] * d[1]) + (d[2] * d[2] + d[3] * d[3]);
          const int pix = wg * 128 + h * 64 + wl * 16 + (lane >> 2);
          const int w = ((j ^ (lane >> 2)) << 2) + (lane & 3);          // 16-byte chunks XOR-ed with pix % 8
          t[pix * 32 + w] = F::pack(d[0], d[1]) ^ flip[j];
          t[(pix + 8) * 32 + w] = F::pack(d[2], d[3]) ^ flip[j];
        }
      if (c == 3) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const float vs = warp_sum(gs[g]), vq = warp_sum(gq[g]);
          if (lane == 0) { red[(warp * 4 + g) * 2] = vs; red[(warp * 4 + g) * 2 + 1] = vq; }
        }
        if (lane == 0) tc_mbar_arrive(redbar);
      }
      ok = sp_bar_and(ok);
      if (!ok) break;
      prev_n = n;
    }
    if (ok && it > 0) pool(stg + ((it - 1) & 1) * 256 * 32, prev_n, (it - 1) & 3);
  }
  // no CTA leaves while a peer may still write into it
  asm volatile("barrier.cluster.arrive.release;\n barrier.cluster.wait.acquire;" ::: "memory");
}

template <class F>
static int launch_stem_pool(const serl_stem_pool_desc* d, cudaStream_t st) {
  auto kern = stem_pool_kernel<F>;
  static int clusters = 0;                                   // images in flight at once
  if (!clusters) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_SMEM) != cudaSuccess) return check_launch("cudaFuncSetAttribute(stem_pool)");
    int dev = 0, sms = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 4; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(4 * sms); cfg.blockDim = dim3(SP_THREADS); cfg.dynamicSmemBytes = SP_SMEM;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) return check_launch("cudaOccupancyMaxActiveClusters(stem_pool)");
    if (n <= 0) { set_last_error("serl_stem_conv_pool_tc_h16: stem_pool_kernel (%d B shared memory) cannot be resident", SP_SMEM); return SERL_ERR_CUDA; }
    clusters = n;
  }
  TcEncodeTiledFn enc = tc_get_encode();
  if (!enc) { set_last_error("serl_stem_conv_pool_tc_h16: cuTensorMapEncodeTiled unavailable"); return SERL_ERR_CUDA; }
  const CUtensorMapDataType dt = d->fmt == SERL_FMT_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap xmap, wmap;
  {
    const cuuint64_t gdim[4] = {16u, 67u, 67u, (cuuint64_t)d->N};
    const cuuint64_t gstr[3] = {16u * 2u, 67u * 16u * 2u, 67u * 67u * 16u * 2u};
    const cuuint32_t box[4] = {16u, 64u, 7u, 1u};
    const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult r = enc(&xmap, dt, 4, const_cast<void*>(d->xs), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_stem_conv_pool_tc_h16: cuTensorMapEncodeTiled (input) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  {
    const cuuint64_t gdim[2] = {256u, 64u};
    const cuuint64_t gstr[1] = {256u * 2u};
    const cuuint32_t box[2] = {64u, 64u};
    const cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(&wmap, dt, 2, const_cast<void*>(d->w), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_stem_conv_pool_tc_h16: cuTensorMapEncodeTiled (weights) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  StemPoolArgs a{};
  a.pooled = static_cast<uint32_t*>(d->pooled); a.side = static_cast<uint32_t*>(d->side); a.stats = d->stats; a.error = d->error;
  a.neg_mask = d->neg_mask; a.N = d->N;
  // persistent: the fewest image slots that still take ceil(N / clusters) rounds
  const int rounds = ceil_div(d->N, clusters);
  const int used = ceil_div(d->N, rounds);
  launch_k_cluster(kern, dim3(used * 4), dim3(SP_THREADS), 4, (size_t)SP_SMEM, st, xmap, wmap, a);
  return check_launch("stem_pool_kernel");
}

}  // namespace serl

using namespace serl;

/* The fused stem runs on stem_pool_kernel (TMA-fed input boxes, accumulators in registers, one 4-CTA cluster per image). */
extern "C" int serl_stem_v2_active(void) { return 1; }

extern "C" int serl_stem_conv_pool_tc_h16(const serl_stem_pool_desc* d, void* stream) {
  if (!d || !d->xs || !d->w || !d->pooled || !d->side || !d->stats || !d->error || d->N < 1) {
    set_last_error("serl_stem_conv_pool_tc_h16: invalid descriptor"); return SERL_ERR_INVALID;
  }
  return d->fmt == SERL_FMT_FP16 ? launch_stem_pool<Fp16>(d, static_cast<cudaStream_t>(stream))
                                 : launch_stem_pool<Bf16>(d, static_cast<cudaStream_t>(stream));
}
