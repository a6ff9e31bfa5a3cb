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
// four chunks of 4 conv rows = 256 output pixels x 64 channels, each computed channel by pixel: D[co][px] = W[co][k] X[px][k]^T,
// one m64 n256 k16 MMA per tap (128 fp32 accumulators per thread).
// Roles (384 threads): warpgroups 0 and 1 are ping-pong consumers.  Warpgroup g takes the CTA's images g, g + 2, ... with all
// four chunks of each, so the pooling carry between chunks and the image's GroupNorm partials stay in its registers.  The two
// alternate chunk by chunk (A0 B0 A1 B1 .. A3 B3 for the images A, B of a pair): after its 16 taps a warpgroup hands the tensor
// cores on through a named barrier, so the taps of the two never interleave and one chunk's epilogue runs under the other's
// MMAs.  One thread of warpgroup 2 issues the TMA loads in that order.  setmaxnreg: 232 registers per consumer thread, 40 per
// producer thread.
// Operands:
//   weights   (A) the packed [64][256] stem weight (32 KB, 128B swizzle), loaded once and kept resident;
//   input     (B) per chunk, one box of 64 cols x 7 rows of xs through a 4-pixel view: box row (y, x) is the 128 bytes
//             xs[y][x .. x + 3] (4 taps x 16 ch, the packed weight's K order within a kernel row; consecutive x overlap by
//             96 B), 128B swizzle.  Tap (r', s') starts r' x 64 rows = r' x 8192 bytes (whole swizzle atoms) into the box and
//             s' x 32 bytes into the row, the same k-advance as the weight's, so the 256 pixel rows of a tap are one plain
//             descriptor.  The 16 taps are issued r' outer, s' inner, one k16 step each: the exact sequence of the raw stem
//             conv (conv_tc_kernel, kStem), so the fp32 accumulators and every 16-bit value equal that conv's bit for bit.
//             The boxes form a 3-stage ring (full: TMA bytes; empty: one arrival per warp of the consuming warpgroup once its
//             taps have retired); a 4th 56 KB stage does not fit in shared memory.
// Epilogue, from registers: warp w holds channels 16 w .. 16 w + 15 (GroupNorm group w) of all 4 rows x 64 columns of the
// chunk, a thread channels c = 16 w + lane / 4 and c + 8 at columns 8 jj + 2 (lane % 4) + {0, 1}.  Each value is rounded to
// 16 bits and sign-adjusted (bit c of neg_mask set <=> GroupNorm scale of channel c negative, so max commutes with
// relu(a x + b)), c and c + 8 packed in one word, and the 3x3/2 max-pool runs in registers: pooled column u = 4 jj + lane % 4
// takes columns 2u, 2u + 1 of this thread and 2u + 2 from the next lane of the quad.  Per CTA: pooled rows 8k..8k+6 are
// complete; row 8k+7 holds max(conv 16k+14, 16k+15) and side[k] the column-pooled conv row 16k, which serl_pool_finish_h16
// joins (row 31 is complete: row 64 is padding).  A pooled row leaves through a 1 KB per-warp staging area (stmatrix .trans)
// as whole 32-byte segments of the warp's 16 channels.
// GroupNorm sums, in a fixed order: thread, warp shuffles, then the cluster's CTAs in rank order.  Every CTA writes its
// partials into each peer's shared memory (st.async, transaction mbarrier) and rank 0 adds the rank-ordered total into stats
// once (stats is zeroed per pass), so the statistics are deterministic.  A warpgroup alternates two slots between its images
// and collects an image's exchange during the next image's first epilogue.  A slot is written again two images later: a peer
// sends image m + 2 only after collecting m + 1, which needs this CTA's m + 1, sent after this CTA collected m.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int SP_STAGE = 7 * 64 * 128;                   // one chunk's box: 7 rows x 64 cols x 128 B (4 pixels x 16 ch), 56 KB
constexpr int SP_STAGES = 3;
constexpr int SP_OFF_A = 4 * 8192;                       // after the resident weight (4 kernel rows x [64 co][64 K])
constexpr int SP_OFF_STG = SP_OFF_A + SP_STAGES * SP_STAGE;        // 8 warps x [32 pooled pixels][32 B] output staging
constexpr int SP_OFF_SLOT = SP_OFF_STG + 8 * 1024;                 // [4 slots][4 ranks][4 groups][2] CTA partial sums
constexpr int SP_OFF_BAR = SP_OFF_SLOT + 4 * 4 * 4 * 2 * 4;
constexpr int SP_SMEM = SP_OFF_BAR + 8 * (2 * SP_STAGES + 5) + 1024;   // + alignment of the dynamic base to 1024
static_assert((SP_STAGE % 1024) == 0 && SP_SMEM <= 232448, "stem_pool_kernel: shared memory layout");

struct StemPoolArgs {
  uint16_t* pooled; uint16_t* side; float* stats; int32_t* error;
  unsigned long long neg_mask; int N;
};

template <class F>
__global__ void __launch_bounds__(CONV_THREADS, 1)
stem_pool_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap wmap, const StemPoolArgs a) {
  pdl_prologue();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sW = smem;
  uint8_t* sA = smem + SP_OFF_A;
  float* slot = reinterpret_cast<float*>(smem + SP_OFF_SLOT);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + SP_OFF_BAR);
  uint64_t* empty = full + SP_STAGES;
  uint64_t* wbar = empty + SP_STAGES;
  uint64_t* gnbar = wbar + 1;                                // [4]: slot 2 g + (m & 1) (cluster exchange of the partial sums)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int band = blockIdx.x & 3;                           // rank in the cluster
  const int img0 = blockIdx.x >> 2, img_step = gridDim.x >> 2;   // the CTA's i-th image: img0 + i img_step

  if (threadIdx.x == 0) {
    for (int s = 0; s < SP_STAGES; ++s) { tc_mbar_init(&full[s], 1); tc_mbar_init(&empty[s], 4); }
    tc_mbar_init(wbar, 1);
    for (int q = 0; q < 4; ++q) tc_mbar_init(&gnbar[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  cluster_sync_all();                                        // the peers' st.async target these barriers

  if (warp >= 8) {
    // ------------------------------- TMA producer (warpgroup 2) -------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
      tc_mbar_expect_tx(wbar, 4u * 8192u);
      for (int t = 0; t < 4; ++t) tc_tma_2d(sW + t * 8192, &wmap, t * 64, 0, wbar);
      bool ok = true;
      int pos = 0;                                           // ring position = the chunk's place in consumption order
      for (int m = 0; ok; ++m) {                             // image pair m: images 2m (warpgroup 0) and 2m + 1 (warpgroup 1)
        const int n0 = img0 + 2 * m * img_step;
        if (n0 >= a.N) break;
        const int imgs = n0 + img_step < a.N ? 2 : 1;
        for (int c = 0; c < 4 && ok; ++c)
          for (int g = 0; g < imgs; ++g, ++pos) {
            const int s = pos % SP_STAGES;
            if (!(ok = tc_mbar_wait(&empty[s], ((uint32_t)(pos / SP_STAGES) & 1u) ^ 1u, a.error))) break;
            tc_mbar_expect_tx(&full[s], (uint32_t)SP_STAGE);
            // xs rows 16 band + 4 c .. + 6, columns 0 .. 63 (+ 3)
            tc_tma_4d(sA + s * SP_STAGE, &xmap, 0, 0, 16 * band + 4 * c, n0 + g * img_step, &full[s]);
          }
      }
    }
  } else {
    // ------------------------------- MMA + epilogue (warpgroups 0, 1, ping-pong) -------------------------------
    // A failed wait clears ok and skips the remaining work, but every named barrier below is still passed, so the other
    // warpgroup never waits on one forever.
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int g = warp >> 2, wl = warp & 3, tid = threadIdx.x & 127, quad = lane & 3;
    const uint32_t a_base = smem_u32(sA), w_base = smem_u32(sW);
    const int ch = 16 * wl + (lane >> 2);                    // this thread's channels: ch (low half of a word), ch + 8 (high)
    const uint32_t flip = (uint32_t)((a.neg_mask >> ch) & 1ull) * 0x8000u | (uint32_t)((a.neg_mask >> (ch + 8)) & 1ull) * 0x80000000u;
    const int next = (lane & ~3) | ((lane + 1) & 3);         // the lane holding column 2u + 2
    // staging: pooled pixel u at u * 32 bytes, its two 16-byte channel halves swapped when bit 2 of u is set
    //   mrow   the row this lane addresses in stmatrix x4 (tiles (t, half 0), (t, half 1), (t + 1, half 0), (t + 1, half 1);
    //          column 2 (l % 4) + e of tile t is pooled pixel 8 t + 4 e + l % 4, so row m = lane % 8 of a tile is pixel
    //          8 t + 4 (m % 2) + m / 2)
    //   grow   the 16 bytes this lane moves to global memory: pixel lane / 2 (+ 16), half lane % 2
    uint8_t* stg = smem + SP_OFF_STG + warp * 1024;
    const uint32_t mrow = smem_u32(stg) + (uint32_t)(((lane >> 4) * 8 + (lane & 1) * 4 + ((lane >> 1) & 3)) * 32 +
                                                     ((((lane >> 3) ^ lane) & 1) << 4));
    const int gpx = lane >> 1, gh = lane & 1;
    const uint32_t grow = (uint32_t)(gpx * 32 + ((gh ^ (gpx >> 2)) & 1) * 16);
    // one pooled row of this warp's 16 channels: v[jj] = (ch, ch + 8) at pooled pixel 4 jj + lane % 4; dst = pixel 0, channel 16 wl
    auto store_row = [&](uint16_t* dst, const uint32_t (&v)[8]) {
      uint32_t o[2][4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        o[t >> 1][2 * (t & 1)] = __byte_perm(v[2 * t], v[2 * t + 1], 0x5410);
        o[t >> 1][2 * (t & 1) + 1] = __byte_perm(v[2 * t], v[2 * t + 1], 0x7632);
      }
      stsm_x4_trans(mrow, o[0]);
      stsm_x4_trans(mrow + 512, o[1]);
      __syncwarp();
#pragma unroll
      for (int e = 0; e < 2; ++e)
        *reinterpret_cast<uint4*>(dst + (size_t)(gpx + 16 * e) * 64 + 8 * gh) = *reinterpret_cast<const uint4*>(stg + grow + e * 512);
      __syncwarp();
    };
    bool ok = tc_mbar_wait(wbar, 0u, a.error);
    ok = mma_bar_and(ok);
    // rank 0: the rank-ordered GroupNorm total of this warpgroup's image m into stats, once every rank's partials arrived
    auto collect = [&](int m) {
      const int q = 2 * g + (m & 1);
      ok = tc_mbar_wait_cluster(&gnbar[q], (uint32_t)(m >> 1) & 1u, a.error);
      if (ok && band == 0 && lane < 2) {
        float v = 0.f;
#pragma unroll
        for (int rk = 0; rk < 4; ++rk) v += slot[((q * 4 + rk) * 4 + wl) * 2 + lane];
        atomicAdd(a.stats + (size_t)(img0 + (2 * m + g) * img_step) * 8 + wl * 2 + lane, v);
      }
    };
    float acc[128];
    uint32_t carry[8];                                       // column-pooled max(conv rows 4c + 2, 4c + 3) of the previous chunk
    float S = 0.f, SS = 0.f;
    int m = 0;
    for (;; ++m) {
      const int n = img0 + (2 * m + g) * img_step;
      if (n >= a.N) break;
      const bool pair = img0 + (2 * m + 1) * img_step < a.N;   // image 2m + 1 exists: the two warpgroups alternate
      const bool more = img0 + (2 * m + 2) * img_step < a.N;
      uint16_t* out = a.pooled + (size_t)n * 32 * 2048 + 16 * wl;
      for (int c = 0; c < 4; ++c) {
        const int pos = 8 * m + (pair ? 2 * c + g : c), s = pos % SP_STAGES;
        if (g == 1 || (c > 0 ? pair : m > 0)) named_bar_sync(2 + g, 256);   // the other warpgroup's chunk before is issued
        if (ok) ok = tc_mbar_wait(&full[s], (uint32_t)(pos / SP_STAGES) & 1u, a.error);
        if (ok) {
          const uint32_t bs = a_base + (uint32_t)(s * SP_STAGE);
          wg_fence();
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int sx = 0; sx < 4; ++sx)
              wg_mma_h16_n256<F::kBf16>(acc, wg_desc(w_base + (uint32_t)(r * 8192)) + 2 * sx,
                                        wg_desc(bs + (uint32_t)(r * 8192)) + 2 * sx, (uint32_t)(r | sx));
          wg_commit();
        }
        if (g == 0 ? pair : (c < 3 || more)) named_bar_arrive(3 - g, 256);   // the other warpgroup's next chunk may start
        wg_wait<0>();
        __syncwarp();
        if (!ok) continue;
        if (lane == 0) tc_mbar_arrive(&empty[s]);

        if (c == 0) {
          if (m > 0) collect(m - 1);
          S = 0.f; SS = 0.f;
        }
        // fragment: acc[4 j + 2 h + e] = channel ch + 8 h, chunk pixel 8 j + 2 (lane % 4) + e = conv row j / 8, column
        // 8 (j % 8) + 2 (lane % 4) + e
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float* d = &acc[4 * j];
          S += (d[0] + d[1]) + (d[2] + d[3]);
          SS += (d[0] * d[0] + d[1] * d[1]) + (d[2] * d[2] + d[3] * d[3]);
        }
        // the 3x3/2 pool, each max in the order of the window's rows, then columns: v (in/out) = the running max of the
        // pooled columns of this thread; first: v starts at conv row i
        uint32_t v[8];
        auto pool_row = [&](int i, bool first) {
          uint32_t w0[8], w1[8];
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const float* d = &acc[4 * (8 * i + jj)];
            w0[jj] = F::pack(d[0], d[2]) ^ flip;             // column 8 jj + 2 (lane % 4)
            w1[jj] = F::pack(d[1], d[3]) ^ flip;             // column 8 jj + 2 (lane % 4) + 1
          }
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const uint32_t nb = __shfl_sync(0xffffffffu, quad == 0 ? w0[jj < 7 ? jj + 1 : 7] : w0[jj], next);
            uint32_t x = first ? w0[jj] : F::max2(v[jj], w0[jj]);
            x = F::max2(x, w1[jj]);
            if (jj < 7 || quad != 3) x = F::max2(x, nb);     // SAME: the window of column 31 ends at the edge
            v[jj] = x;
          }
        };
        const int p0 = 8 * band + 2 * c;                     // pooled row of conv rows 4c .. 4c + 2 of this chunk
        uint32_t o[8];
        pool_row(0, true);                                   // v = row 4c
        if (c > 0) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) o[jj] = F::max2(carry[jj], v[jj]);
          store_row(out + (size_t)(p0 - 1) * 2048, o);
        } else {
          store_row(a.side + ((size_t)n * 4 + band) * 2048 + 16 * wl, v);
        }
        pool_row(1, false);                                  // v = rows 4c, 4c + 1
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) o[jj] = v[jj];
        pool_row(2, true);                                   // v = row 4c + 2
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) o[jj] = F::max2(o[jj], v[jj]);
        store_row(out + (size_t)p0 * 2048, o);
        pool_row(3, false);                                  // v = rows 4c + 2, 4c + 3
        if (c == 3) store_row(out + (size_t)(p0 + 1) * 2048, v);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) carry[jj] = v[jj];

        if (c == 3) {                                        // the image's partials of group wl into every CTA of the cluster
          S = warp_sum(S); SS = warp_sum(SS);
          const int q = 2 * g + (m & 1);
          if (tid == 0) tc_mbar_expect_tx(&gnbar[q], 4u * 4u * 2u * 4u);
          if (lane < 2) {
            const float* dst = slot + ((q * 4 + band) * 4 + wl) * 2 + lane;
#pragma unroll
            for (int rk = 0; rk < 4; ++rk) {
              uint32_t rdst, rbar;
              asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rdst) : "r"(smem_u32(dst)), "r"(rk));
              asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbar) : "r"(smem_u32(&gnbar[q])), "r"(rk));
              asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
                           ::"r"(rdst), "r"(__float_as_uint(lane ? SS : S)), "r"(rbar) : "memory");
            }
          }
        }
      }
    }
    if (ok && m > 0) collect(m - 1);
  }
  cluster_sync_all();                                        // no CTA leaves while a peer may still write into it
}

// Images stem_pool_kernel keeps in flight at once (4-CTA clusters resident), or the error to return (<= 0).
template <class F>
static int stem_pool_clusters() {
  auto kern = stem_pool_kernel<F>;
  static int clusters = 0;
  if (!clusters) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_SMEM) != cudaSuccess) return check_launch("cudaFuncSetAttribute(stem_pool)");
    int dev = 0, sms = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 4; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(4 * sms); cfg.blockDim = dim3(CONV_THREADS); cfg.dynamicSmemBytes = SP_SMEM;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) return check_launch("cudaOccupancyMaxActiveClusters(stem_pool)");
    if (n <= 0) { set_last_error("serl_stem_conv_pool_tc_h16: stem_pool_kernel (%d B shared memory) cannot be resident", SP_SMEM); return SERL_ERR_CUDA; }
    clusters = n;
  }
  return clusters;
}

int stem_pool_resident(int fmt) { return fmt == SERL_FMT_FP16 ? stem_pool_clusters<Fp16>() : stem_pool_clusters<Bf16>(); }

template <class F>
static int launch_stem_pool(const serl_stem_pool_desc* d, cudaStream_t st) {
  auto kern = stem_pool_kernel<F>;
  const int clusters = stem_pool_clusters<F>();
  if (clusters <= 0) return clusters;
  TcEncodeTiledFn enc = tc_get_encode();
  if (!enc) { set_last_error("serl_stem_conv_pool_tc_h16: cuTensorMapEncodeTiled unavailable"); return SERL_ERR_CUDA; }
  const CUtensorMapDataType dt = d->fmt == SERL_FMT_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap xmap, wmap;
  {
    // xs (N, 67, 67, 16) seen as (n, y, x, 64): element (n, y, x, i) is xs[n][y][x + i / 16][i % 16], a row of 4 pixels
    // starting at every pixel (x stride one pixel, 32 B).  x = 0..63 reads columns 0..66, all inside the padded image.
    const cuuint64_t gdim[4] = {64u, 64u, 67u, (cuuint64_t)d->N};
    const cuuint64_t gstr[3] = {16u * 2u, 67u * 16u * 2u, 67u * 67u * 16u * 2u};
    const cuuint32_t box[4] = {64u, 64u, 7u, 1u};
    const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult r = enc(&xmap, dt, 4, const_cast<void*>(d->xs), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
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
  a.pooled = static_cast<uint16_t*>(d->pooled); a.side = static_cast<uint16_t*>(d->side); a.stats = d->stats; a.error = d->error;
  a.neg_mask = d->neg_mask; a.N = d->N;
  // persistent: the fewest image slots that still take ceil(N / clusters) rounds
  const int rounds = ceil_div(d->N, clusters);
  const int used = ceil_div(d->N, rounds);
  launch_k_cluster(kern, dim3(used * 4), dim3(CONV_THREADS), 4, (size_t)SP_SMEM, st, xmap, wmap, a);
  return check_launch("stem_pool_kernel");
}

}  // namespace serl

using namespace serl;

extern "C" int serl_stem_conv_pool_tc_h16(const serl_stem_pool_desc* d, void* stream) {
  if (!d || !d->xs || !d->w || !d->pooled || !d->side || !d->stats || !d->error || d->N < 1) {
    set_last_error("serl_stem_conv_pool_tc_h16: invalid descriptor"); return SERL_ERR_INVALID;
  }
  return d->fmt == SERL_FMT_FP16 ? launch_stem_pool<Fp16>(d, static_cast<cudaStream_t>(stream))
                                 : launch_stem_pool<Bf16>(d, static_cast<cudaStream_t>(stream));
}
