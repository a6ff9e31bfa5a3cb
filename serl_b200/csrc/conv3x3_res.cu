// Stride-1 3x3 convolution + GroupNorm (+ residual) (+ ReLU) in one kernel, and the stride-2 head of ResNetBlock_1..3
// (3x3/2 conv + GroupNorm + ReLU, 1x1/2 projection + GroupNorm).
//
// GroupNorm needs the statistics of a whole image before any of its outputs can be normalised, so the fusion keeps every fp32
// accumulator of an image on chip until its last tap is done and normalises from those values (the raw conv output is never
// rounded to 16 bits and never reaches HBM).
//   32x32x64 and 16x16x128 (ResNetBlock_0's two convs, ResNetBlock_1's Conv_1): conv3x3_res_kernel below, accumulators in
//       registers, operands by TMA (each input band fetched once per CTA, weights resident in shared memory).
//   the stride-2 heads at 16x16 and 8x8, and 8x8x256: conv3x3_pp_kernel below, conv3x3_res_kernel's m64 n256 ping-pong design
//       with the weights streamed through the stage ring (the head's projection is a phase of its own).
//   the 4x4 shapes (ResNetBlock_3's head and Conv_1): conv3x3s2_res_kernel and conv3x3_deep_kernel below, items of 8 / 16
//       whole images x 128 channels (one GroupNorm group), m64 n64 MMAs, weights streamed.
// Every GroupNorm sum is reduced in a fixed order (no atomics): two launches on the same input give bit-identical outputs.
// Reference algebra: vision/resnet_v1.py:129-156 (ResNetBlock), :119-126 (MyGroupNorm).
#include "common.cuh"
#include "conv_common.cuh"
#include "serl_b200.h"
#include "wgmma.cuh"

namespace serl {

// ---------------------------------------------------------------------------------------------------------------------------
// conv3x3_res_kernel: y = [relu](GN(conv3x3 SAME (x)) [+ res | + GN_res(res)]) at W x W x C = 32x32x64 or 16x16x128.
//
// A CTA item is 256 output pixels x 64 output channels of one image, computed channel by pixel: D[co][px] = W[co][k] X[px][k]^T,
// a 64 x 256 x (9 C) implicit GEMM with one m64 n256 k16 MMA per k16 step:
//   32x32x64    4 CTAs per image (a cluster), one band of 8 output rows each, all 64 channels;
//   16x16x128   2 CTAs per image, all 16 rows each, one 64-channel half each (a GroupNorm group never straddles it, so the
//               statistics stay inside the CTA and every CTA keeps a fixed half of the weights resident).
// Roles (384 threads): warpgroups 0 and 1 are ping-pong consumers, warpgroup g takes the CTA's items g, g + 2, g + 4, ... with
// all 256 x 64 accumulators of an item in its registers (128 fp32 per thread), so one warpgroup's epilogue runs while the other
// issues the next item's MMAs.  After its last tap a warpgroup hands the tensor cores on through a named barrier, so the taps of
// consecutive items never interleave.  One thread of warpgroup 2 issues the TMA loads.  setmaxnreg: 232 registers per consumer
// thread, 40 per producer thread.
// Operands:
//   weights   (A) the CTA's 64 x 9C slice, loaded once by TMA (8 KB tiles: 64 channels x one (tap, 64-ci block)), resident;
//   input     (B) per 64-ci block, three boxes of 64 ch x W x (rows + 2) over the NHWC input at x offsets -1, 0, +1 and row
//             offset -1; out-of-range coordinates read as zeros, which is SAME padding on all four edges.  Tap (r, s) is box s
//             shifted by r rows: r W pixels = r W 128 bytes, a multiple of 1024, so the 256 pixel rows of a tap are one plain
//             128B-swizzled descriptor.  The boxes form the stage ring, filled in item order (full: TMA bytes; empty: one
//             arrival per warp of the consuming warpgroup once its taps have retired), so the next item's boxes load while the
//             last taps of this one run.
// GroupNorm: warp w of a warpgroup holds channels 16 w .. 16 w + 15 of all 256 pixels, so a group (16 or 32 channels) is one or
// two warps; each reduces (sum, sum of squares) in a fixed order: thread, warp shuffles, the group's warps in order.  In a
// cluster every CTA writes its partials into each peer's shared memory (st.async, completing a transaction barrier there) and
// sums the four in rank order, so all CTAs of an image hold bit-identical statistics; nothing depends on timing.  A warpgroup
// alternates two slots (and barriers) between its items: a slot is written again two of its items later, and a peer's partials
// of the item in between come only after that peer's warpgroup has finished the epilogue that read the slot.
// Epilogue, per round of 32 pixels: each warp loads its 16 channels of the residual (16-byte loads, issued 4 rounds ahead into
// registers) through a 1 KB staging area into the accumulator layout (ldmatrix .trans), applies the affines of its thread's
// 2 channels, ReLU and the 16-bit pack, and writes the round back through the same area (stmatrix .trans) as whole 32-byte
// pixel segments.
// ---------------------------------------------------------------------------------------------------------------------------
template <int W, int CI>
struct R3Cfg {
  static constexpr int ROWS = 256 / W;                  // output rows of a CTA
  static constexpr int BANDS = W / ROWS;                // CTAs along the rows of an image = cluster size (4 or 1)
  static constexpr int PARTS = BANDS * (CI / 64);       // CTAs per image
  static constexpr int CB = CI / 64;                    // 64-channel input blocks
  static constexpr int NBOX = 3 * CB;                   // input boxes per image
  static constexpr int STAGES = CB == 1 ? 3 : 2;
  static constexpr int BOX = W * (ROWS + 2) * 128;      // bytes of one box
  static constexpr int WTILES = 9 * CB;
  static constexpr int CG = CI / 4;                     // GroupNorm group width
  static constexpr int NG = 64 / CG;                    // groups in a CTA's 64 channels
  static constexpr int WPG = CG / 16;                   // warps of a warpgroup per group
  static constexpr int PF = 4;                          // residual rounds in flight
  static constexpr int OFF_A = WTILES * 8192;
  static constexpr int OFF_STG = OFF_A + STAGES * BOX;  // 8 warps x [32 pixels][32 B] epilogue staging
  static constexpr int OFF_RED = OFF_STG + 8 * 1024;    // [2 warpgroups][4 warps][2] warp partial sums
  static constexpr int OFF_SLOT = OFF_RED + 2 * 4 * 2 * 4;          // [4 slots][BANDS][NG][2] CTA partial sums
  static constexpr int OFF_BAR = OFF_SLOT + 4 * BANDS * NG * 2 * 4;
  static constexpr int SMEM = OFF_BAR + 8 * (2 * STAGES + 5) + 1024;  // + alignment of the dynamic base to 1024
  static_assert(ROWS * W == 256 && (BOX % 1024) == 0 && SMEM <= 232448, "conv3x3_res_kernel: shared memory layout");
};

struct Res3Args {
  uint16_t* y; const uint16_t* res; const float* gamma; const float* beta;
  const float* res_stats; const float* res_gamma; const float* res_beta;
  int32_t* error; int N, relu; float eps;
};

template <class F, int W, int CI>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3x3_res_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap wmap, const Res3Args a) {
  pdl_prologue();
  using K = R3Cfg<W, CI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sW = smem;
  uint8_t* sA = smem + K::OFF_A;
  float* red = reinterpret_cast<float*>(smem + K::OFF_RED);
  float* slot = reinterpret_cast<float*>(smem + K::OFF_SLOT);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + K::OFF_BAR);
  uint64_t* empty = full + K::STAGES;
  uint64_t* wbar = empty + K::STAGES;
  uint64_t* gnbar = wbar + 1;                                // [4]: slot 2 g + (m & 1) (cluster exchange of the partial sums)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int part = blockIdx.x % K::PARTS;
  const int band = part % K::BANDS, n0 = (part / K::BANDS) * 64;   // output rows band * ROWS.., channels n0..n0 + 63
  const int row0 = band * K::ROWS;
  const int img0 = blockIdx.x / K::PARTS, img_step = gridDim.x / K::PARTS;   // item i of the CTA: image img0 + i img_step

  if (threadIdx.x == 0) {
    for (int s = 0; s < K::STAGES; ++s) { tc_mbar_init(&full[s], 1); tc_mbar_init(&empty[s], 4); }
    tc_mbar_init(wbar, 1);
    for (int q = 0; q < 4; ++q) tc_mbar_init(&gnbar[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if constexpr (K::BANDS > 1) cluster_sync_all();           // the peers' st.async target these barriers

  if (warp >= 8) {
    // ------------------------------- TMA producer (warpgroup 2) -------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
      tc_mbar_expect_tx(wbar, (uint32_t)(K::WTILES * 8192));
      for (int t = 0; t < K::WTILES; ++t) tc_tma_2d(sW + t * 8192, &wmap, t * 64, n0, wbar);
      bool ok = true;
      int it = 0;
      for (int n = img0; n < a.N && ok; n += img_step)
        for (int b = 0; b < K::NBOX; ++b, ++it) {           // box b: input channels (b / 3) * 64.., x offset b % 3 - 1
          const int s = it % K::STAGES;
          ok = tc_mbar_wait(&empty[s], ((uint32_t)(it / K::STAGES) & 1u) ^ 1u, a.error);
          if (!ok) break;
          tc_mbar_expect_tx(&full[s], (uint32_t)K::BOX);
          tc_tma_4d(sA + s * K::BOX, &xmap, (b / 3) * 64, b % 3 - 1, row0 - 1, n, &full[s]);
        }
    }
  } else {
    // ------------------------------- MMA + epilogue (warpgroups 0, 1, ping-pong) -------------------------------
    // A failed wait clears ok and skips the remaining work, but every named barrier below is still passed, so the other
    // warpgroup never waits on one forever.
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int g = warp >> 2, wl = warp & 3, tid = threadIdx.x & 127;
    const uint32_t a_base = smem_u32(sA), w_base = smem_u32(sW);
    const float count = (float)(W * W) * (float)K::CG;
    const int grp = wl / K::WPG;                             // this warp's GroupNorm group among the CTA's NG
    const int cl = 16 * wl + (lane >> 2);                    // this thread's channels: n0 + cl, n0 + cl + 8
    // staging: pixel p of a round at p * 32 bytes, its two 16-byte channel halves swapped when bit 2 of p is set
    //   mrow   the row this lane addresses in ldmatrix / stmatrix x4 (tiles (j, half 0), (j, half 1), (j + 1, half 0),
    //          (j + 1, half 1): pixels 8 (lane / 16) + lane % 8, half (lane / 8) % 2)
    //   grow   the 16 bytes this lane moves to or from global memory: pixel lane / 2 (+ 16), half lane % 2
    uint8_t* stg = smem + K::OFF_STG + warp * 1024;
    const uint32_t mrow = smem_u32(stg) + (uint32_t)(((lane >> 4) * 8 + (lane & 7)) * 32 + ((((lane >> 3) ^ (lane >> 2)) & 1) << 4));
    const int gpx = lane >> 1, gh = lane & 1;
    const uint32_t grow = (uint32_t)(gpx * 32 + ((gh ^ (gpx >> 2)) & 1) * 16);
    bool ok = tc_mbar_wait(wbar, 0u, a.error);
    ok = mma_bar_and(ok);
    float acc[128];
    for (int m = 0;; ++m) {
      const int i = g + 2 * m;                               // the CTA's item
      const int n = img0 + i * img_step;
      if (n >= a.N) break;
      if (i > 0) named_bar_sync(2 + g, 256);                 // the other warpgroup has issued the taps of item i - 1
      int it = i * K::NBOX;                                  // ring position of the item's first box
      // the first k-step of an item overwrites the accumulators
      for (int b = 0; b < K::NBOX && ok; ++b, ++it) {
        const int s = it % K::STAGES;
        ok = tc_mbar_wait(&full[s], (uint32_t)(it / K::STAGES) & 1u, a.error);
        if (!ok) break;
        const int cb = b / 3, sx = b % 3;
        const uint32_t bs = a_base + (uint32_t)(s * K::BOX);
        wg_fence();
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const uint32_t ws = w_base + (uint32_t)(((r * 3 + sx) * K::CB + cb) * 8192);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wg_mma_h16_n256<F::kBf16>(acc, wg_desc(ws) + 2 * k, wg_desc(bs + (uint32_t)(r * W * 128)) + 2 * k, (uint32_t)(b | r | k));
        }
        wg_commit();
        if (b > 0) {                                         // the previous box's taps have retired: its stage is free
          wg_wait<1>();
          __syncwarp();
          if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);
        }
      }
      if (n + img_step < a.N) named_bar_arrive(3 - g, 256);  // item i + 1's taps may start

      // the first residual rounds of this warp's 16 channels: issued now, so they load while the last taps run
      const size_t pix0 = (size_t)n * W * W + (size_t)row0 * W;
      const uint16_t* rsrc = a.res + (pix0 + gpx) * CI + n0 + 16 * wl + 8 * gh;
      uint4 rbuf[K::PF][2];
      if (a.res && ok) {
#pragma unroll
        for (int p = 0; p < K::PF; ++p)
#pragma unroll
          for (int e = 0; e < 2; ++e) rbuf[p][e] = __ldg(reinterpret_cast<const uint4*>(rsrc + (size_t)(32 * p + 16 * e) * CI));
      }
      wg_wait<0>();
      __syncwarp();
      if (ok && lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);

      // ---- GroupNorm sums of this warp's group, in a fixed order ----
      // fragment: acc[4 j + 2 h + e] = channel n0 + cl + 8 h, pixel 8 j + 2 (lane % 4) + e of the item
      float S = 0.f, SS = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float* d = &acc[4 * j];
        S += (d[0] + d[1]) + (d[2] + d[3]);
        SS += (d[0] * d[0] + d[1] * d[1]) + (d[2] * d[2] + d[3] * d[3]);
      }
      S = warp_sum(S); SS = warp_sum(SS);
      if constexpr (K::WPG > 1) {                            // the group's warps in order
        if (lane == 0) *reinterpret_cast<float2*>(red + (g * 4 + wl) * 2) = make_float2(S, SS);
        named_bar_sync(4 + g, 128);
        S = 0.f; SS = 0.f;
#pragma unroll
        for (int k = 0; k < K::WPG; ++k) {
          const float2 v = *reinterpret_cast<const float2*>(red + (g * 4 + grp * K::WPG + k) * 2);
          S += v.x; SS += v.y;
        }
      }
      if constexpr (K::BANDS > 1) {                          // the cluster's CTAs in rank order
        const int q = 2 * g + (m & 1);
        if (ok) {
          if (tid == 0) tc_mbar_expect_tx(&gnbar[q], (uint32_t)(K::BANDS * K::NG * 2 * 4));
          if (lane < 2) {
            const float v = lane ? SS : S;
            float* dst = slot + ((q * K::BANDS + band) * K::NG + grp) * 2 + lane;
#pragma unroll
            for (int rk = 0; rk < K::BANDS; ++rk) {          // into every CTA of the cluster (this one included)
              uint32_t rdst, rbar;
              asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rdst) : "r"(smem_u32(dst)), "r"(rk));
              asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rbar) : "r"(smem_u32(&gnbar[q])), "r"(rk));
              asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
                           ::"r"(rdst), "r"(__float_as_uint(v)), "r"(rbar) : "memory");
            }
          }
          ok = tc_mbar_wait_cluster(&gnbar[q], (uint32_t)(m >> 1) & 1u, a.error);
        }
        S = 0.f; SS = 0.f;
#pragma unroll
        for (int rk = 0; rk < K::BANDS; ++rk) {
          S += slot[((q * K::BANDS + rk) * K::NG + grp) * 2];
          SS += slot[((q * K::BANDS + rk) * K::NG + grp) * 2 + 1];
        }
      }
      if (!ok) continue;

      // ---- the affines of this thread's two channels (and of the projected residual) ----
      const float mean = S / count;
      const float var = fmaxf(SS / count - mean * mean, 0.f);
      const float rstd = rsqrtf(var + a.eps);
      float ga[2], gb[2], ra[2] = {1.f, 1.f}, rb[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = n0 + cl + 8 * h;
        ga[h] = rstd * a.gamma[c];
        gb[h] = a.beta[c] - mean * ga[h];
      }
      if (a.res_stats) {
        const int rg = (n0 + cl) / K::CG;
        const float rs = a.res_stats[((size_t)n * 4 + rg) * 2], rss = a.res_stats[((size_t)n * 4 + rg) * 2 + 1];
        const float rmean = rs / count;
        const float rvar = fmaxf(rss / count - rmean * rmean, 0.f);
        const float rrstd = rsqrtf(rvar + a.eps);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int c = n0 + cl + 8 * h;
          ra[h] = rrstd * a.res_gamma[c];
          rb[h] = a.res_beta[c] - rmean * ra[h];
        }
      }

      // ---- per round of 32 pixels: residual in, normalise (+ residual) (+ ReLU), pack, out as 32-byte pixel segments ----
      uint16_t* ydst = a.y + (pix0 + gpx) * CI + n0 + 16 * wl + 8 * gh;
#pragma unroll
      for (int rd = 0; rd < 8; ++rd) {
        uint32_t rv[2][4];                                   // residual tiles of j = 4 rd + 2 x + {0, 1}: [x][2 (j & 1) + h]
        if (a.res) {
#pragma unroll
          for (int e = 0; e < 2; ++e) *reinterpret_cast<uint4*>(stg + grow + e * 512) = rbuf[rd % K::PF][e];
          __syncwarp();
          ldsm_x4_trans(mrow, rv[0]);
          ldsm_x4_trans(mrow + 512, rv[1]);
          if (rd + K::PF < 8) {
#pragma unroll
            for (int e = 0; e < 2; ++e)
              rbuf[rd % K::PF][e] = __ldg(reinterpret_cast<const uint4*>(rsrc + (size_t)(32 * (rd + K::PF) + 16 * e) * CI));
          }
        }
        uint32_t o[2][4];
#pragma unroll
        for (int x = 0; x < 2; ++x)
#pragma unroll
          for (int jj = 0; jj < 2; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float* d = &acc[4 * (4 * rd + 2 * x + jj) + 2 * h];
              float o0 = fmaf(d[0], ga[h], gb[h]), o1 = fmaf(d[1], ga[h], gb[h]);
              if (a.res) {
                const float2 r = F::unpack(rv[x][2 * jj + h]);
                o0 += a.res_stats ? fmaf(r.x, ra[h], rb[h]) : r.x;
                o1 += a.res_stats ? fmaf(r.y, ra[h], rb[h]) : r.y;
              }
              if (a.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
              o[x][2 * jj + h] = F::pack(o0, o1);
            }
        __syncwarp();                                        // the residual's tiles have been read
        stsm_x4_trans(mrow, o[0]);
        stsm_x4_trans(mrow + 512, o[1]);
        __syncwarp();
#pragma unroll
        for (int e = 0; e < 2; ++e)
          *reinterpret_cast<uint4*>(ydst + (size_t)(32 * rd + 16 * e) * CI) = *reinterpret_cast<const uint4*>(stg + grow + e * 512);
        __syncwarp();
      }
    }
  }
  if constexpr (K::BANDS > 1) cluster_sync_all();           // no CTA leaves while a peer may still write into it
}

// Images conv3x3_res_kernel keeps in flight at once (clusters / CTA pairs resident), or the error to return (<= 0).
template <class F, int W, int CI>
static int conv3x3_res_groups() {
  using K = R3Cfg<W, CI>;
  auto kern = conv3x3_res_kernel<F, W, CI>;
  static int groups = 0;
  if (!groups) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, K::SMEM) != cudaSuccess) return check_launch("cudaFuncSetAttribute(conv3x3_res)");
    int dev = 0, sms = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (K::BANDS > 1) {
      cudaLaunchConfig_t cfg = {};
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = K::BANDS; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      cfg.gridDim = dim3(K::BANDS * sms); cfg.blockDim = dim3(CONV_THREADS); cfg.dynamicSmemBytes = K::SMEM;
      cfg.attrs = attr; cfg.numAttrs = 1;
      if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) return check_launch("cudaOccupancyMaxActiveClusters(conv3x3_res)");
    } else {
      int per_sm = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, CONV_THREADS, K::SMEM) != cudaSuccess) return check_launch("cudaOccupancyMaxActiveBlocksPerMultiprocessor(conv3x3_res)");
      n = per_sm * sms / K::PARTS;
    }
    if (n <= 0) { set_last_error("serl_conv3x3_res_h16: conv3x3_res_kernel (%d B shared memory) cannot be resident", K::SMEM); return SERL_ERR_CUDA; }
    groups = n;
  }
  return groups;
}

template <class F, int W, int CI>
static int launch_conv3x3_res(const serl_conv3x3_res_desc* d, cudaStream_t st) {
  using K = R3Cfg<W, CI>;
  auto kern = conv3x3_res_kernel<F, W, CI>;
  const int groups = conv3x3_res_groups<F, W, CI>();
  if (groups <= 0) return groups;
  TcEncodeTiledFn enc = tc_get_encode();
  if (!enc) { set_last_error("serl_conv3x3_res_h16: cuTensorMapEncodeTiled unavailable"); return SERL_ERR_CUDA; }
  const CUtensorMapDataType dt = d->fmt == SERL_FMT_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap xmap, wmap;
  {
    const cuuint64_t gdim[4] = {(cuuint64_t)CI, (cuuint64_t)W, (cuuint64_t)W, (cuuint64_t)d->N};
    const cuuint64_t gstr[3] = {(cuuint64_t)CI * 2, (cuuint64_t)W * CI * 2, (cuuint64_t)W * W * CI * 2};
    const cuuint32_t box[4] = {64u, (cuuint32_t)W, (cuuint32_t)(K::ROWS + 2), 1u};
    const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult r = enc(&xmap, dt, 4, const_cast<void*>(d->x), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_conv3x3_res_h16: cuTensorMapEncodeTiled (input) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  {
    const cuuint64_t gdim[2] = {(cuuint64_t)9 * CI, (cuuint64_t)CI};
    const cuuint64_t gstr[1] = {(cuuint64_t)9 * CI * 2};
    const cuuint32_t box[2] = {64u, 64u};
    const cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(&wmap, dt, 2, const_cast<void*>(d->w), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_conv3x3_res_h16: cuTensorMapEncodeTiled (weights) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  Res3Args a{};
  a.y = static_cast<uint16_t*>(d->y); a.res = static_cast<const uint16_t*>(d->res); a.gamma = d->gamma; a.beta = d->beta;
  a.res_stats = d->res_stats; a.res_gamma = d->res_gamma; a.res_beta = d->res_beta;
  a.error = d->error; a.N = d->N; a.relu = d->relu; a.eps = d->eps;
  // persistent: the fewest image slots that still take ceil(N / groups) rounds
  const int rounds = ceil_div(d->N, groups);
  const int used = ceil_div(d->N, rounds);
  launch_k_cluster(kern, dim3(used * K::PARTS), dim3(CONV_THREADS), K::BANDS, (size_t)K::SMEM, st, xmap, wmap, a);
  return check_launch("conv3x3_res_kernel");
}

// ---------------------------------------------------------------------------------------------------------------------------
// conv3x3_pp_kernel: conv3x3_res_kernel's design with the weights streamed, for the shapes whose 9 CI x 64 weight slice does not
// fit next to the input boxes:
//   S 2   the stage heads at WO 16 (CI 64) and WO 8 (CI 128), from the block input x (N, 2 WO, 2 WO, CI):
//         y = relu(GN(conv3x3 stride 2 SAME (x)))    r = GN(conv1x1 stride 2 (x))      (N, WO, WO, 2 CI)
//         SAME on an even input pads 0 low, 1 high: output (i, j) reads input rows 2i..2i+2, columns 2j..2j+2, and the
//         projection reads (2i, 2j) - tap (0, 0)'s operand.
//   S 1   the 8x8x256 conv (Conv_1 of ResNetBlock_2): y = [relu](GN(conv3x3 SAME (x)) [+ res | + GN_res(res)]), 16-bit y or
//         fp32 out_f32.
// A CTA item is 256 output pixels (WO 16: one image, WO 8: four) x 64 output channels, computed channel by pixel with one
// m64 n256 k16 MMA per k16 step (A: a 64 x 64 weight tile, B: 256 pixel rows of an input box).  Warpgroups 0 and 1 ping-pong
// phases: an item is one phase (the conv) or, at S 2, two (the conv, then the projection through the same 128 accumulators,
// with its own statistics and epilogue, since y and r together would not fit in registers).  Warpgroup g runs the phases of
// the CTA's items g, g + 2, ..., and the tensor cores pass between the warpgroups through named barriers after each phase's
// last MMA, so the tensor-core order is conv(i), conv(i + 1), proj(i), proj(i + 1), conv(i + 2), ...: a warpgroup's
// epilogue runs under the other's MMAs.  One thread of warpgroup 2 issues the TMA loads, in that same order.
// Operands: each stage of the ring holds one input box plus the weight tiles (64 channels x 64 k, 8 KB) of the taps it serves.
//   The box is 64 ch x WO cols x IMGS images x BROWS output rows, laid out row-major over (row, image, col), so one output row
//   of the item's images is SHIFT = IMGS WO 128 bytes (a multiple of 1024) and tap (r, s) is a plain 128B-swizzled 256-row
//   descriptor at a whole number of SHIFTs into its box.  The tensor map's dimensions are (c, x, n, y) for that order.
//   S 2   element strides {1, 2, 1, 2} at (x = s, y = r): box (0, s) is one output row taller and serves taps (0, s) and
//         (2, s) (input row 2i + 2 is row 2(i + 1): one SHIFT); box (1, s) serves tap (1, s): 6 boxes per 64-ci block.  The
//         projection re-fetches box (0, 0) with the projection tile, one per 64-ci block.
//   S 1   three boxes per 64-ci block at x offsets -1, 0, +1 and row offset -1, 10 rows tall: tap (r, s) is box s shifted by
//         r SHIFTs.
//   Coordinates out of range read as zeros: the SAME padding, and the images >= N of a partial item (never stored).
// GroupNorm: warp w of a warpgroup holds channels 16 w .. 16 w + 15 of the 256 pixels; accumulator column j (pixels 8 j ..)
// belongs to image j % IMGS.  A group (32 or 64 channels: 2 or 4 warps) is reduced in a fixed order: thread, warp shuffles,
// the group's warps in order; two launches give bit-identical outputs.
// Epilogue, per round of 32 pixels (one output row of four images at WO 8): as conv3x3_res_kernel's, through a 1 KB staging
// area per warp (stmatrix / ldmatrix .trans), 32-byte pixel segments; fp32 out_f32 is stored from the fragments.
// ---------------------------------------------------------------------------------------------------------------------------
template <int S, int WO, int CI>
struct PPCfg {
  static constexpr int CO = S * CI;
  static constexpr int HW = WO * WO;
  static constexpr int IMGS = 256 / HW;                 // images of an item
  static constexpr int NSL = CO / 64;                   // 64-channel slices
  static constexpr int CB = CI / 64;                    // 64-ci blocks
  static constexpr int NB = S == 2 ? 6 : 3;             // conv boxes per 64-ci block
  static constexpr int NPH = S == 2 ? 2 : 1;            // phases per item
  static constexpr int BROWS = WO + (S == 2 ? 1 : 2);   // output rows in a box
  static constexpr int SHIFT = IMGS * WO * 128;         // bytes of one output row of the item's images
  static constexpr int BOX = BROWS * SHIFT;
  static constexpr int STAGE = BOX + (S == 2 ? 2 : 3) * 8192;
  static constexpr int STAGES = S == 2 ? 4 : 3;
  static constexpr int CG = CO / 4;                     // GroupNorm group width
  static constexpr int WPG = CG / 16;                   // warps of a warpgroup per group
  static constexpr int PF = 4;                          // residual rounds in flight
  static constexpr int OFF_STG = STAGES * STAGE;        // 8 warps x [32 pixels][32 B] epilogue staging
  static constexpr int OFF_RED = OFF_STG + 8 * 1024;    // [2 slots][2 warpgroups][4 warps][IMGS][2] warp partial sums
  static constexpr int OFF_BAR = OFF_RED + 2 * 2 * 4 * IMGS * 2 * 4;
  static constexpr int SMEM = OFF_BAR + 8 * 2 * STAGES + 1024;  // + alignment of the dynamic base to 1024
  static_assert(IMGS * HW == 256 && WPG <= 4 && (SHIFT % 1024) == 0 && (STAGE % 1024) == 0 && SMEM <= 232448,
                "conv3x3_pp_kernel: shared memory layout");
  static __host__ __device__ constexpr int nbox(int ph) { return ph ? CB : NB * CB; }
};

struct PPArgs {
  uint16_t* y; uint16_t* r; float* out_f32; const uint16_t* res;
  const float* gamma; const float* beta; const float* gamma_p; const float* beta_p;
  const float* res_stats; const float* res_gamma; const float* res_beta;
  int32_t* error; int N, relu; float eps;
};

template <class F, int S, int WO, int CI>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3x3_pp_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap wmap,
                  const __grid_constant__ CUtensorMap pmap, const PPArgs a) {
  pdl_prologue();
  using K = PPCfg<S, WO, CI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* red = reinterpret_cast<float*>(smem + K::OFF_RED);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + K::OFF_BAR);
  uint64_t* empty = full + K::STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_items = ceil_div(a.N, K::IMGS) * K::NSL;
  // phase P of the CTA belongs to warpgroup P & 1; it is that warpgroup's phase P >> 1 = NPH m + ph, of the CTA's item
  // (P & 1) + 2 m.  Returns the item's index in the grid, or -1 when the CTA has no such item.
  auto item_of = [&](int P) {
    const int q = blockIdx.x + ((P & 1) + 2 * ((P >> 1) / K::NPH)) * gridDim.x;
    return P >= 0 && q < n_items ? q : -1;
  };
  // no phase after P exists once the CTA's item 2 m of P's pair does not
  auto past_end = [&](int P) { return blockIdx.x + 2 * ((P >> 1) / K::NPH) * gridDim.x >= n_items; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < K::STAGES; ++s) { tc_mbar_init(&full[s], 1); tc_mbar_init(&empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------- TMA producer (warpgroup 2) -------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
      if (S == 2) asm volatile("prefetch.tensormap [%0];" ::"l"(&pmap) : "memory");
      bool ok = true;
      int it = 0;
      for (int P = 0; ok && !past_end(P); ++P) {
        const int q = item_of(P);
        if (q < 0) continue;
        const int ph = (P >> 1) % K::NPH;
        const int img0 = (q / K::NSL) * K::IMGS, n0 = (q % K::NSL) * 64;
        for (int b = 0; b < K::nbox(ph); ++b, ++it) {
          const int s = it % K::STAGES;
          ok = tc_mbar_wait(&empty[s], ((uint32_t)(it / K::STAGES) & 1u) ^ 1u, a.error);
          if (!ok) break;
          // box b: 64-ci block cb, kernel column sx, first kernel row row0 (S 2 conv: 0 = rows 0 and 2; S 1: all three)
          const int cb = ph ? b : b / K::NB, sx = ph ? 0 : b % 3, row0 = S == 2 && !ph ? (b % K::NB) / 3 : 0;
          const int ntap = ph ? 1 : S == 1 ? 3 : row0 == 0 ? 2 : 1;
          uint8_t* st = smem + s * K::STAGE;
          tc_mbar_expect_tx(&full[s], (uint32_t)(K::BOX + ntap * 8192));
          tc_tma_4d(st, &xmap, cb * 64, S == 2 ? sx : sx - 1, img0, S == 2 ? row0 : -1, &full[s]);
          for (int t = 0; t < ntap; ++t) {
            if (ph) tc_tma_2d(st + K::BOX, &pmap, cb * 64, n0, &full[s]);
            else tc_tma_2d(st + K::BOX + t * 8192, &wmap, (((S == 2 ? row0 + 2 * t : t) * 3 + sx) * K::CB + cb) * 64, n0, &full[s]);
          }
        }
      }
    }
  } else {
    // ------------------------------- MMA + epilogue (warpgroups 0, 1, ping-pong) -------------------------------
    // A failed wait clears ok and skips the remaining work, but every named barrier below is still passed, so the other
    // warpgroup never waits on one forever.
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int g = warp >> 2, wl = warp & 3;
    const uint32_t s_base = smem_u32(smem);
    const float count = (float)K::HW * (float)K::CG;
    const int grp = wl / K::WPG;                             // this warp's GroupNorm group among the item's 64 channels
    const int cl = 16 * wl + (lane >> 2);                    // this thread's channels: n0 + cl, n0 + cl + 8
    // staging as in conv3x3_res_kernel: pixel p of a round at p * 32 bytes, its two 16-byte channel halves swapped when bit 2
    // of p is set; mrow: this lane's ldmatrix / stmatrix row, grow: the 16 bytes this lane moves, pixel gpx (+ 16), half gh
    uint8_t* stg = smem + K::OFF_STG + warp * 1024;
    const uint32_t mrow = smem_u32(stg) + (uint32_t)(((lane >> 4) * 8 + (lane & 7)) * 32 + ((((lane >> 3) ^ (lane >> 2)) & 1) << 4));
    const int gpx = lane >> 1, gh = lane & 1;
    const uint32_t grow = (uint32_t)(gpx * 32 + ((gh ^ (gpx >> 2)) & 1) * 16);
    // pixel 32 rd + 16 e + gpx of a round's order is image im(e), pixel rd RSTEP + e ESTEP + pbase of that image
    const int pbase = K::IMGS == 1 ? gpx : gpx & 7;
    constexpr int RSTEP = K::IMGS == 1 ? 32 : 8, ESTEP = K::IMGS == 1 ? 16 : 0;
    auto im_of = [&](int e) { return K::IMGS == 1 ? 0 : 2 * e + (gpx >> 3); };
    bool ok = true;
    int it = 0;
    float acc[128];
    for (int P = 0; !past_end(P); ++P) {
      const int q = item_of(P);
      if (q < 0) continue;
      const int k = P >> 1, ph = k % K::NPH;
      if ((P & 1) != g) { it += K::nbox(ph); continue; }
      const int img0 = (q / K::NSL) * K::IMGS, n0 = (q % K::NSL) * 64;
      if (item_of(P - 1) >= 0) named_bar_sync(2 + g, 256);  // the other warpgroup has issued the MMAs of phase P - 1
      // the first k-step of a phase overwrites the accumulators
      if (ph == 0) {
        for (int cb = 0; cb < K::CB && ok; ++cb) {
          // the boxes of a 64-ci block unrolled: the taps a box serves are known at compile time
#pragma unroll
          for (int bb = 0; bb < K::NB; ++bb, ++it) {
            const int s = it % K::STAGES;
            ok = tc_mbar_wait(&full[s], (uint32_t)(it / K::STAGES) & 1u, a.error);
            if (!ok) break;
            const int ntap = S == 1 ? 3 : bb < 3 ? 2 : 1;
            const uint32_t bs = s_base + (uint32_t)(s * K::STAGE), ws = bs + (uint32_t)K::BOX;
            wg_fence();
#pragma unroll
            for (int t = 0; t < ntap; ++t)
#pragma unroll
              for (int kk = 0; kk < 4; ++kk)
                wg_mma_h16_n256<F::kBf16>(acc, wg_desc(ws + (uint32_t)(t * 8192)) + 2 * kk, wg_desc(bs + (uint32_t)(t * K::SHIFT)) + 2 * kk,
                                          (uint32_t)(cb | bb | t | kk));
            wg_commit();
            if (cb > 0 || bb > 0) {                          // the previous box's MMAs have retired: its stage is free
              wg_wait<1>();
              __syncwarp();
              if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);
            }
          }
        }
      } else {
        for (int cb = 0; cb < K::CB && ok; ++cb, ++it) {
          const int s = it % K::STAGES;
          ok = tc_mbar_wait(&full[s], (uint32_t)(it / K::STAGES) & 1u, a.error);
          if (!ok) break;
          const uint32_t bs = s_base + (uint32_t)(s * K::STAGE), ws = bs + (uint32_t)K::BOX;
          wg_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            wg_mma_h16_n256<F::kBf16>(acc, wg_desc(ws) + 2 * kk, wg_desc(bs) + 2 * kk, (uint32_t)(cb | kk));
          wg_commit();
          if (cb > 0) {
            wg_wait<1>();
            __syncwarp();
            if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);
          }
        }
      }
      if (item_of(P + 1) >= 0) named_bar_arrive(3 - g, 256);  // phase P + 1's MMAs may start

      // the first residual rounds of this warp's 16 channels: issued now, so they load while the last MMAs run
      const uint16_t* rsrc = a.res + ((size_t)img0 * K::HW + pbase) * CI + n0 + 16 * wl + 8 * gh;
      uint4 rbuf[K::PF][2];
      if (S == 1 && a.res && ok) {
#pragma unroll
        for (int p = 0; p < K::PF; ++p)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            rbuf[p][e] = img0 + im_of(e) < a.N ? __ldg(reinterpret_cast<const uint4*>(rsrc + (size_t)(im_of(e) * K::HW + p * RSTEP + e * ESTEP) * CI))
                                               : make_uint4(0u, 0u, 0u, 0u);
      }
      wg_wait<0>();
      __syncwarp();
      if (ok && lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);

      // ---- GroupNorm sums per image of this warp's group, in a fixed order ----
      // fragment: acc[4 j + 2 h + e] = channel n0 + cl + 8 h, column 8 j + 2 (lane % 4) + e (image j % IMGS)
      float sm[K::IMGS], ss[K::IMGS];
#pragma unroll
      for (int im = 0; im < K::IMGS; ++im) { sm[im] = 0.f; ss[im] = 0.f; }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float* d = &acc[4 * j];
        sm[j % K::IMGS] += (d[0] + d[1]) + (d[2] + d[3]);
        ss[j % K::IMGS] += (d[0] * d[0] + d[1] * d[1]) + (d[2] * d[2] + d[3] * d[3]);
      }
      float* rw = red + (((k & 1) * 2 + g) * 4) * K::IMGS * 2;     // two slots: a slot is written again only after every warp
#pragma unroll                                                // of the warpgroup has passed the next phase's barrier 4 + g
      for (int im = 0; im < K::IMGS; ++im) {
        sm[im] = warp_sum(sm[im]); ss[im] = warp_sum(ss[im]);
        if (lane == 0) *reinterpret_cast<float2*>(rw + (wl * K::IMGS + im) * 2) = make_float2(sm[im], ss[im]);
      }
      named_bar_sync(4 + g, 128);
      if (!ok) continue;
      float mean[K::IMGS], rstd[K::IMGS];
#pragma unroll
      for (int im = 0; im < K::IMGS; ++im) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int w = 0; w < K::WPG; ++w) {                   // the group's warps in order
          const float2 v = *reinterpret_cast<const float2*>(rw + ((grp * K::WPG + w) * K::IMGS + im) * 2);
          s0 += v.x; s1 += v.y;
        }
        mean[im] = s0 / count;
        rstd[im] = rsqrtf(fmaxf(s1 / count - mean[im] * mean[im], 0.f) + a.eps);
      }

      // ---- the affines of this thread's two channels per image (and of the normalised residual) ----
      const float* gam = ph ? a.gamma_p : a.gamma;
      const float* bet = ph ? a.beta_p : a.beta;
      const bool relu = S == 2 ? ph == 0 : a.relu != 0;
      const bool rnorm = S == 1 && a.res_stats;
      float ga[K::IMGS][2], gb[K::IMGS][2], ra[K::IMGS][2], rb[K::IMGS][2];
#pragma unroll
      for (int im = 0; im < K::IMGS; ++im) {
        float rmean = 0.f, rrstd = 1.f;
        if (rnorm && img0 + im < a.N) {
          const float* rs = a.res_stats + ((size_t)(img0 + im) * 4 + n0 / K::CG) * 2;
          rmean = rs[0] / count;
          rrstd = rsqrtf(fmaxf(rs[1] / count - rmean * rmean, 0.f) + a.eps);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int c = n0 + cl + 8 * h;
          ga[im][h] = rstd[im] * gam[c];
          gb[im][h] = bet[c] - mean[im] * ga[im][h];
          ra[im][h] = rnorm ? rrstd * a.res_gamma[c] : 1.f;
          rb[im][h] = rnorm ? a.res_beta[c] - rmean * ra[im][h] : 0.f;
        }
      }

      // ---- per round of 32 pixels: residual in, normalise (+ residual) (+ ReLU), out; images >= N are never stored ----
      uint16_t* out = S == 2 && ph ? a.r : a.y;
      const size_t obase = ((size_t)img0 * K::HW + pbase) * K::CO + n0 + 16 * wl + 8 * gh;
#pragma unroll
      for (int rd = 0; rd < 8; ++rd) {
        uint32_t rv[2][4];                                   // residual tiles of j = 4 rd + 2 x + {0, 1}: [x][2 (j & 1) + h]
        if (S == 1 && a.res) {
#pragma unroll
          for (int e = 0; e < 2; ++e) *reinterpret_cast<uint4*>(stg + grow + e * 512) = rbuf[rd % K::PF][e];
          __syncwarp();
          ldsm_x4_trans(mrow, rv[0]);
          ldsm_x4_trans(mrow + 512, rv[1]);
          if (rd + K::PF < 8) {
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (img0 + im_of(e) < a.N)
                rbuf[rd % K::PF][e] = __ldg(reinterpret_cast<const uint4*>(rsrc + (size_t)(im_of(e) * K::HW + (rd + K::PF) * RSTEP + e * ESTEP) * CI));
          }
        }
        uint32_t o[2][4];
#pragma unroll
        for (int x = 0; x < 2; ++x)
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const int j = 4 * rd + 2 * x + jj, im = j % K::IMGS;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float* d = &acc[4 * j + 2 * h];
              float o0 = fmaf(d[0], ga[im][h], gb[im][h]), o1 = fmaf(d[1], ga[im][h], gb[im][h]);
              if (S == 1 && a.res) {
                const float2 r = F::unpack(rv[x][2 * jj + h]);
                o0 += fmaf(r.x, ra[im][h], rb[im][h]);
                o1 += fmaf(r.y, ra[im][h], rb[im][h]);
              }
              if (relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
              if (S == 1 && a.out_f32 && img0 + im < a.N) {  // fp32 from the fragment: pixels 8 (j / IMGS) + 2 (lane % 4) + {0, 1}
                float* of = a.out_f32 + ((size_t)(img0 + im) * K::HW + 8 * (j / K::IMGS) + 2 * (lane & 3)) * CI + n0 + cl + 8 * h;
                of[0] = o0;
                of[CI] = o1;
              }
              o[x][2 * jj + h] = F::pack(o0, o1);
            }
          }
        __syncwarp();                                        // the residual's tiles have been read
        if (S == 2 || !a.out_f32) {
          stsm_x4_trans(mrow, o[0]);
          stsm_x4_trans(mrow + 512, o[1]);
          __syncwarp();
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (img0 + im_of(e) < a.N)
              *reinterpret_cast<uint4*>(out + obase + (size_t)(im_of(e) * K::HW + rd * RSTEP + e * ESTEP) * K::CO) =
                  *reinterpret_cast<const uint4*>(stg + grow + e * 512);
          __syncwarp();
        }
      }
    }
  }
}

// x: the block input (N, S WO, S WO, CI); w: the packed 3x3 weights (CO, 9 CI); w_proj (S 2): the 1x1 projection (CO, CI)
// CTAs of conv3x3_pp_kernel resident at once, or the error to return (<= 0).
template <class F, int S, int WO, int CI>
static int conv3x3_pp_slots(const char* name) {
  using K = PPCfg<S, WO, CI>;
  auto kern = conv3x3_pp_kernel<F, S, WO, CI>;
  static int slots = 0;
  if (!slots) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, K::SMEM) != cudaSuccess) return check_launch("cudaFuncSetAttribute(conv3x3_pp)");
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, CONV_THREADS, K::SMEM) != cudaSuccess) return check_launch("cudaOccupancyMaxActiveBlocksPerMultiprocessor(conv3x3_pp)");
    if (per_sm <= 0) { set_last_error("%s: conv3x3_pp_kernel (%d B shared memory) cannot be resident", name, K::SMEM); return SERL_ERR_CUDA; }
    slots = per_sm * sms;
  }
  return slots;
}

template <class F, int S, int WO, int CI>
static int launch_conv3x3_pp(const char* name, const void* x, const void* w, const void* w_proj, int fmt, const PPArgs& a, cudaStream_t st) {
  using K = PPCfg<S, WO, CI>;
  auto kern = conv3x3_pp_kernel<F, S, WO, CI>;
  const int slots = conv3x3_pp_slots<F, S, WO, CI>(name);
  if (slots <= 0) return slots;
  TcEncodeTiledFn enc = tc_get_encode();
  if (!enc) { set_last_error("%s: cuTensorMapEncodeTiled unavailable", name); return SERL_ERR_CUDA; }
  const CUtensorMapDataType dt = fmt == SERL_FMT_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap xmap, wmap, pmap;
  {
    // dimensions (c, x, n, y), so a box lands row-major over (row, image, col); S 2 takes every second column and row
    constexpr int WI = S * WO;
    const cuuint64_t gdim[4] = {(cuuint64_t)CI, (cuuint64_t)WI, (cuuint64_t)a.N, (cuuint64_t)WI};
    const cuuint64_t gstr[3] = {(cuuint64_t)CI * 2, (cuuint64_t)WI * WI * CI * 2, (cuuint64_t)WI * CI * 2};
    const cuuint32_t box[4] = {64u, (cuuint32_t)(S * WO), (cuuint32_t)K::IMGS, (cuuint32_t)(S * K::BROWS)};
    const cuuint32_t estr[4] = {1u, (cuuint32_t)S, 1u, (cuuint32_t)S};
    CUresult r = enc(&xmap, dt, 4, const_cast<void*>(x), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("%s: cuTensorMapEncodeTiled (input) failed (%d)", name, (int)r); return SERL_ERR_CUDA; }
  }
  for (int pj = 0; pj < S; ++pj) {
    const cuuint64_t kdim = (cuuint64_t)(pj ? 1 : 9) * CI;
    const cuuint64_t gdim[2] = {kdim, (cuuint64_t)K::CO};
    const cuuint64_t gstr[1] = {kdim * 2};
    const cuuint32_t box[2] = {64u, 64u};
    const cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(pj ? &pmap : &wmap, dt, 2, const_cast<void*>(pj ? w_proj : w), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("%s: cuTensorMapEncodeTiled (weights) failed (%d)", name, (int)r); return SERL_ERR_CUDA; }
  }
  if (S == 1) pmap = wmap;                                   // no projection
  const int items = ceil_div(a.N, K::IMGS) * K::NSL;
  const int rounds = ceil_div(items, slots);                 // persistent: the fewest CTAs that still take `rounds` items each
  launch_k(kern, dim3(ceil_div(items, rounds)), dim3(CONV_THREADS), (size_t)K::SMEM, st, xmap, wmap, pmap, a);
  return check_launch("conv3x3_pp_kernel");
}

template <class F, int WO, int CI>
static int launch_conv3x3s2_pp(const serl_conv3x3s2_res_desc* d, cudaStream_t st) {
  PPArgs a{};
  a.y = static_cast<uint16_t*>(d->y); a.r = static_cast<uint16_t*>(d->r);
  a.gamma = d->gamma; a.beta = d->beta; a.gamma_p = d->gamma_proj; a.beta_p = d->beta_proj;
  a.error = d->error; a.N = d->N; a.relu = 1; a.eps = d->eps;
  return launch_conv3x3_pp<F, 2, WO, CI>("serl_conv3x3s2_res_h16", d->x, d->w, d->w_proj, d->fmt, a, st);
}

template <class F>
static int launch_conv3x3_res8_pp(const serl_conv3x3_res_desc* d, cudaStream_t st) {
  PPArgs a{};
  a.out_f32 = d->out_f32; a.y = d->out_f32 ? nullptr : static_cast<uint16_t*>(d->y);
  a.res = static_cast<const uint16_t*>(d->res); a.gamma = d->gamma; a.beta = d->beta;
  a.res_stats = d->res_stats; a.res_gamma = d->res_gamma; a.res_beta = d->res_beta;
  a.error = d->error; a.N = d->N; a.relu = d->relu; a.eps = d->eps;
  return launch_conv3x3_pp<F, 1, 8, 256>("serl_conv3x3_res_h16", d->x, d->w, nullptr, d->fmt, a, st);
}

// ---------------------------------------------------------------------------------------------------------------------------
// conv3x3s2_res_kernel: head of ResNetBlock_1..3 from one read of the block input x (N, 2 WO, 2 WO, CI):
//   y = relu(GN(conv3x3 stride 2 SAME (x)))    r = GN(conv1x1 stride 2 (x))      (N, WO, WO, 2 CI)
// SAME on an even input pads 0 low, 1 high: output (i, j) reads input rows 2i..2i+2, columns 2j..2j+2, and the projection
// reads (2i, 2j) - exactly the A operand of tap (0, 0).
//
// Runs the WO 4 head (CI 256); the WO 16 and WO 8 heads run on conv3x3_pp_kernel above.  A CTA item is 128 output pixels
// (8 whole images) x 128 output channels (one GroupNorm group), a 128 x 128 x 9 CI implicit GEMM plus the 128 x 128 x CI
// projection, so every GroupNorm group of the item lies inside the CTA.
// Roles (384 threads): warpgroups 0 and 1 issue the MMAs (m64 n64 k16 on two 64 x 64 sub-tiles each: 64 fp32 accumulators
// per thread for y, 64 for r) and run the epilogue; one thread of warpgroup 2 issues the TMA loads.  setmaxnreg moves the
// registers: 232 per MMA thread, 40 per producer thread (the 128 accumulators and the epilogue do not fit in 168).
// Operands: each stage of the ring holds one input box plus the weight tiles (BN channels x 64 k) of the taps it serves.
//   input   a 4-D NHWC box with element strides {1, 2, 2, 1} at (x = s, y = r): it gathers input (r + 2i, s + 2j) of every
//           output pixel of the item's images, so the A tile of tap (r, s) is a plain 128B-swizzled descriptor; coordinates
//           past the edge read as zeros, which is the high-side padding.  An m64 tile spans 4 images, so a row shift would not
//           be a uniform core-matrix stride: one box per tap.
//   weights streamed with the boxes; tap (0, 0)'s stage also carries the projection tile, whose MMAs reuse that A operand.
// GroupNorm: per-thread sums, warp shuffles, then a fixed (warp, sub-tile) order per (image, group): no atomics, so two
// launches give bit-identical outputs.  The next item's first stages load while the epilogue of this one runs.
// ---------------------------------------------------------------------------------------------------------------------------
template <int WO, int CI>
struct S2Cfg {
  static constexpr int CO = 2 * CI;
  static constexpr int BN = 128;                        // output channels of an item
  static constexpr int M = 128;                         // output pixels of an item
  static constexpr int HW = WO * WO;
  static constexpr int IMGS = M / HW;                   // images of an item
  static constexpr int NSL = CO / BN;                   // channel slices
  static constexpr int CB = CI / 64;
  static constexpr int NB = 9;                          // boxes per 64-ci block: one per tap
  static constexpr int NBOX = NB * CB;
  static constexpr int BOX = IMGS * HW * 128;
  static constexpr int TILE = BN * 128;                 // one weight tile: BN channels x 64 k
  static constexpr int STAGE = BOX + 2 * TILE;          // the box, its tap's tile and (tap (0, 0)) the projection tile
  static constexpr int STAGES = 4;
  static constexpr int CG = CO / 4;                     // GroupNorm group width
  static constexpr int CGS = 64;                        // channels of a group inside a 64-channel sub-tile
  static constexpr int GPS = 64 / CGS;                  // groups of a sub-tile
  static constexpr int NGC = BN / CG;                   // groups of an item's channels (whole groups only)
  static constexpr int OFF_STG = STAGES * STAGE;        // 8 warps x [8 rows][128 B] output staging
  static constexpr int OFF_PAR = OFF_STG + 8 * 1024;    // [BN][4]: gamma, beta, gamma_proj, beta_proj
  static constexpr int OFF_RED = OFF_PAR + BN * 16;     // [8 warps][2 sub-tiles][GPS][4]: warp partial sums of y and r
  static constexpr int OFF_ST = OFF_RED + 8 * 2 * GPS * 16;     // [IMGS][NGC][4]: mean, rstd of y; mean, rstd of r
  static constexpr int OFF_BAR = OFF_ST + IMGS * NGC * 16;
  static constexpr int SMEM = OFF_BAR + 8 * 2 * STAGES + 1024;  // + alignment of the dynamic base to 1024
  static_assert(WO == 4 && BN % CG == 0, "conv3x3s2_res_kernel: the WO 4 head, an item holds whole GroupNorm groups");
  static_assert(M % HW == 0 && (BOX % 1024) == 0 && (STAGE % 1024) == 0 && SMEM <= 232448, "conv3x3s2_res_kernel: shared memory layout");
  // first output pixel and first channel of sub-tile h of warpgroup wg: two n64 halves
  __device__ static constexpr int m_off(int wg, int) { return wg * 64; }
  __device__ static constexpr int n_off(int h) { return h * 64; }
};

struct S2Args {
  uint16_t* y; uint16_t* r; const float* gamma; const float* beta; const float* gamma_p; const float* beta_p;
  int32_t* error; int N; float eps;
};

template <class F, int WO, int CI>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3x3s2_res_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap wmap,
                     const __grid_constant__ CUtensorMap pmap, const S2Args a) {
  pdl_prologue();
  using K = S2Cfg<WO, CI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* par = reinterpret_cast<float*>(smem + K::OFF_PAR);
  float* red = reinterpret_cast<float*>(smem + K::OFF_RED);
  float* gst = reinterpret_cast<float*>(smem + K::OFF_ST);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + K::OFF_BAR);
  uint64_t* empty = full + K::STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_items = ceil_div(a.N, K::IMGS) * K::NSL;

  if (threadIdx.x == 0) {
    for (int s = 0; s < K::STAGES; ++s) { tc_mbar_init(&full[s], 1); tc_mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------- TMA producer (warpgroup 2) -------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&pmap) : "memory");
      bool ok = true;
      int it = 0;
      for (int item = blockIdx.x; item < n_items && ok; item += gridDim.x) {
        const int img = (item / K::NSL) * K::IMGS, n0 = (item % K::NSL) * K::BN;
        for (int b = 0; b < K::NBOX; ++b, ++it) {
          const int s = it % K::STAGES;
          ok = tc_mbar_wait(&empty[s], ((uint32_t)(it / K::STAGES) & 1u) ^ 1u, a.error);
          if (!ok) break;
          const int cb = b / K::NB, row = (b % K::NB) / 3, sx = b % 3;      // tap (row, sx)
          const bool proj = row == 0 && sx == 0;
          uint8_t* st = smem + s * K::STAGE;
          tc_mbar_expect_tx(&full[s], (uint32_t)(K::BOX + (1 + (int)proj) * K::TILE));
          tc_tma_4d(st, &xmap, cb * 64, sx, row, img, &full[s]);
          tc_tma_2d(st + K::BOX, &wmap, ((row * 3 + sx) * K::CB + cb) * 64, n0, &full[s]);
          if (proj) tc_tma_2d(st + K::BOX + K::TILE, &pmap, cb * 64, n0, &full[s]);
        }
      }
    }
  } else {
    // ------------------------------- MMA + epilogue (warpgroups 0, 1) -------------------------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int tid = threadIdx.x, wg = tid >> 7, wl = warp & 3;
    const uint32_t s_base = smem_u32(smem);
    uint32_t a_off[2], b_off[2];                             // sub-tile h: its first A row in a box (tap shift 0), B row
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = K::m_off(wg, h);
      a_off[h] = (uint32_t)(m * 128);
      b_off[h] = (uint32_t)(K::n_off(h) * 128);
    }
    const float count = (float)K::HW * (float)K::CG;
    bool ok = true;
    int it = 0;
    float acc[2][32], pacc[2][32];
    for (int item = blockIdx.x; item < n_items && ok; item += gridDim.x) {
      const int img0 = (item / K::NSL) * K::IMGS, n0 = (item % K::NSL) * K::BN;
      // the first k-step of an item overwrites the accumulators (no zeroing between the wgmmas of a pipeline stage)
      for (int cb = 0; cb < K::CB && ok; ++cb) {
        // the boxes of a 64-ci block unrolled: which taps (and the projection) a box serves is known at compile time, so
        // no wgmma sits on a divergent path
#pragma unroll
        for (int bb = 0; bb < K::NB; ++bb, ++it) {
          const int s = it % K::STAGES;
          ok = tc_mbar_wait(&full[s], (uint32_t)(it / K::STAGES) & 1u, a.error);
          if (!ok) break;
          const uint32_t as = s_base + (uint32_t)(s * K::STAGE), ws = as + (uint32_t)K::BOX;
          wg_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              wg_mma_h16<F::kBf16>(acc[h], wg_desc(as + a_off[h]) + 2 * k, wg_desc(ws + b_off[h]) + 2 * k, (uint32_t)(cb | bb | k));
          if (bb == 0) {                                     // tap (0, 0): the projection on the same A tiles
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
              for (int h = 0; h < 2; ++h)
                wg_mma_h16<F::kBf16>(pacc[h], wg_desc(as + a_off[h]) + 2 * k, wg_desc(ws + (uint32_t)K::TILE + b_off[h]) + 2 * k,
                                     (uint32_t)(cb | k));
          }
          wg_commit();
          if (cb > 0 || bb > 0) {                            // the previous box's MMAs have retired: its stage is free
            wg_wait<1>();
            __syncwarp();
            if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);
          }
        }
      }
      wg_wait<0>();
      ok = mma_bar_and(ok);
      if (!ok) break;
      __syncwarp();
      if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);

      // ---- GroupNorm partial sums: thread, warp shuffles, then (warp, sub-tile) in a fixed order ----
      // fragment: acc[h][4 j + 2 hf + e] = pixel m_off(wg, h) + 16 wl + 8 hf + lane / 4, channel n_off(h) + 8 j + 2 (lane % 4) + e
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int g = 0; g < K::GPS; ++g) {
          float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int j = g * K::CGS / 8; j < (g + 1) * K::CGS / 8; ++j) {
            const float* d = &acc[h][4 * j];
            const float* p = &pacc[h][4 * j];
            v[0] += (d[0] + d[1]) + (d[2] + d[3]);
            v[1] += (d[0] * d[0] + d[1] * d[1]) + (d[2] * d[2] + d[3] * d[3]);
            v[2] += (p[0] + p[1]) + (p[2] + p[3]);
            v[3] += (p[0] * p[0] + p[1] * p[1]) + (p[2] * p[2] + p[3] * p[3]);
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            v[q] = warp_sum(v[q]);
            if (lane == 0) red[((warp * 2 + h) * K::GPS + g) * 4 + q] = v[q];
          }
        }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid < K::BN)
        *reinterpret_cast<float4*>(par + tid * 4) = make_float4(a.gamma[n0 + tid], a.beta[n0 + tid], a.gamma_p[n0 + tid], a.beta_p[n0 + tid]);
      if (tid < K::IMGS * K::NGC) {
        const int im = tid / K::NGC, gc = tid % K::NGC;
        float S[4] = {0.f, 0.f, 0.f, 0.f};
        for (int w = 0; w < 8; ++w)
          for (int h = 0; h < 2; ++h)
            for (int g = 0; g < K::GPS; ++g) {
              if ((K::m_off(w >> 2, h) + 16 * (w & 3)) / K::HW != im || (K::n_off(h) + g * K::CGS) / K::CG != gc) continue;
              for (int q = 0; q < 4; ++q) S[q] += red[((w * 2 + h) * K::GPS + g) * 4 + q];
            }
        const float mean = S[0] / count, pmean = S[2] / count;
        const float var = fmaxf(S[1] / count - mean * mean, 0.f), pvar = fmaxf(S[3] / count - pmean * pmean, 0.f);
        *reinterpret_cast<float4*>(gst + tid * 4) = make_float4(mean, rsqrtf(var + a.eps), pmean, rsqrtf(pvar + a.eps));
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");

      // ---- normalise, pack, store whole 128-byte rows (y with ReLU, then r); images >= N are never stored ----
      uint8_t* stg = smem + K::OFF_STG + warp * 1024;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int m8 = K::m_off(wg, h) + wl * 16 + hf * 8;        // first of this warp's 8 rows (one image)
          const int im = m8 / K::HW;
          if (img0 + im >= a.N) continue;
          const int rr = lane >> 2;
          const size_t pix0 = (size_t)img0 * K::HW + m8;
#pragma unroll 1
          for (int o = 0; o < 2; ++o) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int c = K::n_off(h) + 8 * j + 2 * (lane & 3);
              const float4 sv = *reinterpret_cast<const float4*>(gst + (im * K::NGC + c / K::CG) * 4);
              const float4 p0 = *reinterpret_cast<const float4*>(par + c * 4), p1 = *reinterpret_cast<const float4*>(par + c * 4 + 4);
              float o0, o1;
              if (o == 0) {
                const float g0 = sv.y * p0.x, g1 = sv.y * p1.x;
                o0 = fmaxf(fmaf(acc[h][4 * j + 2 * hf], g0, p0.y - sv.x * g0), 0.f);
                o1 = fmaxf(fmaf(acc[h][4 * j + 2 * hf + 1], g1, p1.y - sv.x * g1), 0.f);
              } else {
                const float g0 = sv.w * p0.z, g1 = sv.w * p1.z;
                o0 = fmaf(pacc[h][4 * j + 2 * hf], g0, p0.w - sv.z * g0);
                o1 = fmaf(pacc[h][4 * j + 2 * hf + 1], g1, p1.w - sv.z * g1);
              }
              *reinterpret_cast<uint32_t*>(stg + rr * 128 + ((j ^ rr) << 4) + (lane & 3) * 4) = F::pack(o0, o1);
            }
            __syncwarp();
            uint16_t* out = o == 0 ? a.y : a.r;
#pragma unroll
            for (int e = lane; e < 64; e += 32) {
              const int q = e >> 3, ch = e & 7;
              const uint4 v = *reinterpret_cast<const uint4*>(stg + q * 128 + ((ch ^ q) << 4));
              *reinterpret_cast<uint4*>(out + (pix0 + q) * K::CO + n0 + K::n_off(h) + ch * 8) = v;
            }
            __syncwarp();
          }
        }
    }
  }
}

// CTAs of conv3x3s2_res_kernel resident at once, or the error to return (<= 0).
template <class F, int WO, int CI>
static int conv3x3s2_res_slots() {
  using K = S2Cfg<WO, CI>;
  auto kern = conv3x3s2_res_kernel<F, WO, CI>;
  static int slots = 0;
  if (!slots) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, K::SMEM) != cudaSuccess) return check_launch("cudaFuncSetAttribute(conv3x3s2_res)");
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, CONV_THREADS, K::SMEM) != cudaSuccess) return check_launch("cudaOccupancyMaxActiveBlocksPerMultiprocessor(conv3x3s2_res)");
    if (per_sm <= 0) { set_last_error("serl_conv3x3s2_res_h16: conv3x3s2_res_kernel (%d B shared memory) cannot be resident", K::SMEM); return SERL_ERR_CUDA; }
    slots = per_sm * sms;
  }
  return slots;
}

template <class F, int WO, int CI>
static int launch_conv3x3s2_res(const serl_conv3x3s2_res_desc* d, cudaStream_t st) {
  using K = S2Cfg<WO, CI>;
  auto kern = conv3x3s2_res_kernel<F, WO, CI>;
  const int slots = conv3x3s2_res_slots<F, WO, CI>();
  if (slots <= 0) return slots;
  TcEncodeTiledFn enc = tc_get_encode();
  if (!enc) { set_last_error("serl_conv3x3s2_res_h16: cuTensorMapEncodeTiled unavailable"); return SERL_ERR_CUDA; }
  const CUtensorMapDataType dt = d->fmt == SERL_FMT_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap xmap, wmap, pmap;
  {
    // every second column and row: a box of boxDim / 2 elements along x and y
    const cuuint64_t gdim[4] = {(cuuint64_t)CI, (cuuint64_t)(2 * WO), (cuuint64_t)(2 * WO), (cuuint64_t)d->N};
    const cuuint64_t gstr[3] = {(cuuint64_t)CI * 2, (cuuint64_t)2 * WO * CI * 2, (cuuint64_t)4 * WO * WO * CI * 2};
    const cuuint32_t box[4] = {64u, (cuuint32_t)(2 * WO), (cuuint32_t)(2 * WO), (cuuint32_t)K::IMGS};
    const cuuint32_t estr[4] = {1u, 2u, 2u, 1u};
    CUresult r = enc(&xmap, dt, 4, const_cast<void*>(d->x), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_conv3x3s2_res_h16: cuTensorMapEncodeTiled (input) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  for (int pj = 0; pj < 2; ++pj) {
    const cuuint64_t kdim = (cuuint64_t)(pj ? 1 : 9) * CI;
    const cuuint64_t gdim[2] = {kdim, (cuuint64_t)K::CO};
    const cuuint64_t gstr[1] = {kdim * 2};
    const cuuint32_t box[2] = {64u, (cuuint32_t)K::BN};
    const cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(pj ? &pmap : &wmap, dt, 2, const_cast<void*>(pj ? d->w_proj : d->w), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_conv3x3s2_res_h16: cuTensorMapEncodeTiled (weights) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  S2Args a{};
  a.y = static_cast<uint16_t*>(d->y); a.r = static_cast<uint16_t*>(d->r);
  a.gamma = d->gamma; a.beta = d->beta; a.gamma_p = d->gamma_proj; a.beta_p = d->beta_proj;
  a.error = d->error; a.N = d->N; a.eps = d->eps;
  const int items = ceil_div(d->N, K::IMGS) * K::NSL;
  const int rounds = ceil_div(items, slots);                 // persistent: the fewest CTAs that still take `rounds` items each
  launch_k(kern, dim3(ceil_div(items, rounds)), dim3(CONV_THREADS), (size_t)K::SMEM, st, xmap, wmap, pmap, a);
  return check_launch("conv3x3s2_res_kernel");
}

// ---------------------------------------------------------------------------------------------------------------------------
// conv3x3_deep_kernel: y = [relu](GN(conv3x3 SAME (x)) [+ res | + GN_res(res)]) at W x W x C = 4x4x512 (the Conv_1 of
// ResNetBlock_3), written as 16-bit y or as fp32 out_f32 (the trunk's features).  8x8x256 runs on conv3x3_pp_kernel above.
//
// A CTA item is 256 output pixels (16 whole images) x 128 output channels (one GroupNorm group), a 256 x 128 x 9 C implicit
// GEMM, so every GroupNorm group of the item lies inside the CTA.
// Roles (384 threads): warpgroups 0 and 1 issue the MMAs (m64 n64 k16 on 2 x 2 sub-tiles: 128 rows x 128 channels, 128 fp32
// accumulators per thread) and run the epilogue; one thread of warpgroup 2 issues the TMA loads.  setmaxnreg: 232 registers
// per MMA thread, 40 per producer thread.
// Operands: each stage of the ring holds one input box plus the weight tile (128 channels x 64 k) of its tap.
//   input one box of 64 ch x 4 x 4 x 16 images per tap at offsets (s - 1, r - 1): an m64 tile spans 4 images, so a row shift
//         (512 B) is not a uniform core-matrix stride.  Coordinates out of range read as zeros: the SAME padding on all four
//         edges, and the images >= N of a partial item (those are never stored).
//   residual  the item's 256 pixels x 128 channels (two 64-channel TMA boxes per 128 rows, 128B-swizzled) take the ring
//         position(s) after its last box, so they load while the last taps run and need no registers (128 accumulators
//         fill the MMA threads' budget).
// GroupNorm: per-thread sums, warp shuffles, then a fixed (warp, sub-tile) order per (image, group): no atomics, so two
// launches give bit-identical outputs.  The next item's first stages load while this item's epilogue runs.  Each warp stages
// 8 rows x 64 channels in shared memory and stores them as whole rows (128 B of 16-bit, 256 B of fp32).
// ---------------------------------------------------------------------------------------------------------------------------
template <int W, int CI>
struct DeepCfg {
  static constexpr int BN = 128;                        // output channels of an item
  static constexpr int HW = W * W;
  static constexpr int IMGS = 256 / HW;                 // images of an item
  static constexpr int NSL = CI / BN;                   // channel slices
  static constexpr int CB = CI / 64;
  static constexpr int NB = 9;                          // boxes per 64-ci block: one per tap
  static constexpr int NBOX = NB * CB;
  static constexpr int BOX = IMGS * HW * 128;
  static constexpr int TILE = BN * 128;                 // one weight tile: BN channels x 64 k
  static constexpr int STAGE = BOX + TILE;
  static constexpr int STAGES = 4;
  static constexpr int RES = 128 * 128 * 2;             // residual of one warpgroup's 128 rows
  static constexpr int RPS = STAGE / RES;               // of those per stage (2 or 1)
  static constexpr int NRES = 2 / RPS;                  // ring positions of an item's residual
  static constexpr int CG = CI / 4;                     // GroupNorm group width (64 or 128)
  static constexpr int NGC = BN / CG;                   // groups of an item's channels
  static constexpr int OFF_STG = STAGES * STAGE;        // 8 warps x [8 rows][256 B] output staging
  static constexpr int OFF_PAR = OFF_STG + 8 * 2048;    // [BN][4]: gamma, beta, res_gamma, res_beta
  static constexpr int OFF_RED = OFF_PAR + BN * 16;     // [8 warps][2 m sub-tiles][2 n sub-tiles][2]: warp partial sums
  static constexpr int OFF_ST = OFF_RED + 8 * 2 * 2 * 8;        // [IMGS][NGC][4]: mean, rstd of y; mean, rstd of res
  static constexpr int OFF_BAR = OFF_ST + IMGS * NGC * 16;
  static constexpr int SMEM = OFF_BAR + 8 * 2 * STAGES + 1024;  // + alignment of the dynamic base to 1024
  static_assert(CG >= 64 && BN % CG == 0, "conv3x3_deep_kernel: an n64 sub-tile lies in one group, an item holds whole groups");
  static_assert(RPS >= 1 && NRES < STAGES, "conv3x3_deep_kernel: the residual fits the ring");
  static_assert(HW >= 16 && (BOX % 1024) == 0 && (STAGE % 1024) == 0 && SMEM <= 232448, "conv3x3_deep_kernel: shared memory layout");
  // first output pixel of m sub-tile h of warpgroup wg
  __device__ static constexpr int m_off(int wg, int h) { return wg * 128 + h * 64; }
};

struct DeepArgs {
  uint16_t* y; float* out_f32; const uint16_t* res; const float* gamma; const float* beta;
  const float* res_stats; const float* res_gamma; const float* res_beta;
  int32_t* error; int N, relu; float eps;
};

template <class F, int W, int CI>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3x3_deep_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap wmap,
                    const __grid_constant__ CUtensorMap rmap, const DeepArgs a) {
  pdl_prologue();
  using K = DeepCfg<W, CI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* par = reinterpret_cast<float*>(smem + K::OFF_PAR);
  float* red = reinterpret_cast<float*>(smem + K::OFF_RED);
  float* gst = reinterpret_cast<float*>(smem + K::OFF_ST);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + K::OFF_BAR);
  uint64_t* empty = full + K::STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_items = ceil_div(a.N, K::IMGS) * K::NSL;

  if (threadIdx.x == 0) {
    for (int s = 0; s < K::STAGES; ++s) { tc_mbar_init(&full[s], 1); tc_mbar_init(&empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------- TMA producer (warpgroup 2) -------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
      if (a.res) asm volatile("prefetch.tensormap [%0];" ::"l"(&rmap) : "memory");
      bool ok = true;
      int it = 0;
      for (int item = blockIdx.x; item < n_items && ok; item += gridDim.x) {
        const int img = (item / K::NSL) * K::IMGS, n0 = (item % K::NSL) * K::BN;
        for (int b = 0; b < K::NBOX + (a.res ? K::NRES : 0); ++b, ++it) {
          const int s = it % K::STAGES;
          ok = tc_mbar_wait(&empty[s], ((uint32_t)(it / K::STAGES) & 1u) ^ 1u, a.error);
          if (!ok) break;
          uint8_t* st = smem + s * K::STAGE;
          if (b >= K::NBOX) {                                // the residual: rows of RPS warpgroups, [64-ch half][128 rows][128 B]
            tc_mbar_expect_tx(&full[s], (uint32_t)(K::RPS * K::RES));
            for (int q = 0; q < K::RPS; ++q)
              for (int c = 0; c < 2; ++c)
                tc_tma_2d(st + q * K::RES + c * (K::RES / 2), &rmap, n0 + c * 64, img * K::HW + ((b - K::NBOX) * K::RPS + q) * 128, &full[s]);
            continue;
          }
          const int cb = b / K::NB, row = (b % K::NB) / 3, sx = b % 3;      // tap (row, sx)
          tc_mbar_expect_tx(&full[s], (uint32_t)K::STAGE);
          tc_tma_4d(st, &xmap, cb * 64, sx - 1, row - 1, img, &full[s]);
          tc_tma_2d(st + K::BOX, &wmap, ((row * 3 + sx) * K::CB + cb) * 64, n0, &full[s]);
        }
      }
    }
  } else {
    // ------------------------------- MMA + epilogue (warpgroups 0, 1) -------------------------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int tid = threadIdx.x, wg = tid >> 7, wl = warp & 3;
    const uint32_t s_base = smem_u32(smem);
    uint32_t a_off[2];                                       // m sub-tile h: its first A row in a box
#pragma unroll
    for (int h = 0; h < 2; ++h) a_off[h] = (uint32_t)(K::m_off(wg, h) * 128);
    const float count = (float)K::HW * (float)K::CG;
    bool ok = true;
    int it = 0;
    float acc[2][2][32];                                     // [m sub-tile][n sub-tile]
    for (int item = blockIdx.x; item < n_items && ok; item += gridDim.x) {
      const int img0 = (item / K::NSL) * K::IMGS, n0 = (item % K::NSL) * K::BN;
      // the first k-step of an item overwrites the accumulators (no zeroing between the wgmmas of a pipeline stage)
      for (int cb = 0; cb < K::CB && ok; ++cb) {
        // the boxes of a 64-ci block unrolled, so no wgmma sits on a divergent path
#pragma unroll
        for (int bb = 0; bb < K::NB; ++bb, ++it) {
          const int s = it % K::STAGES;
          ok = tc_mbar_wait(&full[s], (uint32_t)(it / K::STAGES) & 1u, a.error);
          if (!ok) break;
          const uint32_t as = s_base + (uint32_t)(s * K::STAGE), ws = as + (uint32_t)K::BOX;
          wg_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int c = 0; c < 2; ++c)
                wg_mma_h16<F::kBf16>(acc[h][c], wg_desc(as + a_off[h]) + 2 * k, wg_desc(ws + (uint32_t)(c * 64 * 128)) + 2 * k,
                                     (uint32_t)(cb | bb | k));
          wg_commit();
          if (cb > 0 || bb > 0) {                            // the previous box's MMAs have retired: its stage is free
            wg_wait<1>();
            __syncwarp();
            if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);
          }
        }
      }
      wg_wait<0>();
      ok = mma_bar_and(ok);
      if (!ok) break;
      __syncwarp();
      if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % K::STAGES]);

      // ---- GroupNorm partial sums: thread, warp shuffles, then (warp, sub-tile) in a fixed order ----
      // fragment: acc[h][c][4 j + 2 hf + e] = pixel m_off(wg, h) + 16 wl + 8 hf + lane / 4, channel 64 c + 8 j + 2 (lane % 4) + e
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          float v0 = 0.f, v1 = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float* d = &acc[h][c][4 * j];
            v0 += (d[0] + d[1]) + (d[2] + d[3]);
            v1 += (d[0] * d[0] + d[1] * d[1]) + (d[2] * d[2] + d[3] * d[3]);
          }
          v0 = warp_sum(v0); v1 = warp_sum(v1);
          if (lane == 0) *reinterpret_cast<float2*>(red + ((warp * 2 + h) * 2 + c) * 2) = make_float2(v0, v1);
        }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid < K::BN) {
        const int ch = n0 + tid;
        *reinterpret_cast<float4*>(par + tid * 4) = a.res_stats ? make_float4(a.gamma[ch], a.beta[ch], a.res_gamma[ch], a.res_beta[ch])
                                                                : make_float4(a.gamma[ch], a.beta[ch], 1.f, 0.f);
      }
      if (tid < K::IMGS * K::NGC) {
        const int im = tid / K::NGC, gc = tid % K::NGC;
        float S = 0.f, SS = 0.f;
        for (int w = 0; w < 8; ++w)
          for (int h = 0; h < 2; ++h)
            for (int c = 0; c < 2; ++c) {
              if ((K::m_off(w >> 2, h) + 16 * (w & 3)) / K::HW != im || c * 64 / K::CG != gc) continue;
              S += red[((w * 2 + h) * 2 + c) * 2];
              SS += red[((w * 2 + h) * 2 + c) * 2 + 1];
            }
        const float mean = S / count;
        const float var = fmaxf(SS / count - mean * mean, 0.f);
        float rmean = 0.f, rrstd = 1.f;
        if (a.res_stats && img0 + im < a.N) {
          const float* rs = a.res_stats + ((size_t)(img0 + im) * 4 + (n0 / K::CG + gc)) * 2;
          rmean = rs[0] / count;
          rrstd = rsqrtf(fmaxf(rs[1] / count - rmean * rmean, 0.f) + a.eps);
        }
        *reinterpret_cast<float4*>(gst + tid * 4) = make_float4(mean, rsqrtf(var + a.eps), rmean, rrstd);
      }
      // this warpgroup's residual: [64-ch half][128 rows][128 B], row m - 128 wg at (m & 7)-swizzled 16-byte chunks
      const int rpos = it + wg / K::RPS;
      const uint8_t* rsm = smem + (rpos % K::STAGES) * K::STAGE + (wg % K::RPS) * K::RES;
      if (a.res) ok = tc_mbar_wait(&full[rpos % K::STAGES], (uint32_t)(rpos / K::STAGES) & 1u, a.error);
      ok = mma_bar_and(ok);
      if (!ok) break;

      // ---- normalise (+ residual) (+ ReLU), stage, store whole rows; images >= N are never stored ----
      uint8_t* stg = smem + K::OFF_STG + warp * 2048;
      const int rr = lane >> 2;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int m8 = K::m_off(wg, h) + wl * 16 + hf * 8;        // first of this warp's 8 rows (one image)
          const int im = m8 / K::HW;
          if (img0 + im >= a.N) continue;
          const size_t pix0 = (size_t)img0 * K::HW + m8;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const float4 sv = *reinterpret_cast<const float4*>(gst + (im * K::NGC + c * 64 / K::CG) * 4);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int cl = c * 64 + 8 * j + 2 * (lane & 3);
              const float4 p0 = *reinterpret_cast<const float4*>(par + cl * 4), p1 = *reinterpret_cast<const float4*>(par + cl * 4 + 4);
              const float g0 = sv.y * p0.x, g1 = sv.y * p1.x;
              float o0 = fmaf(acc[h][c][4 * j + 2 * hf], g0, p0.y - sv.x * g0);
              float o1 = fmaf(acc[h][c][4 * j + 2 * hf + 1], g1, p1.y - sv.x * g1);
              if (a.res) {
                const float2 rv = F::unpack(*reinterpret_cast<const uint32_t*>(
                    rsm + c * (K::RES / 2) + (m8 - wg * 128 + rr) * 128 + ((j ^ rr) << 4) + (lane & 3) * 4));
                if (a.res_stats) {
                  const float r0 = sv.w * p0.z, r1 = sv.w * p1.z;
                  o0 += fmaf(rv.x, r0, p0.w - sv.z * r0);
                  o1 += fmaf(rv.y, r1, p1.w - sv.z * r1);
                } else {
                  o0 += rv.x; o1 += rv.y;
                }
              }
              if (a.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
              if (a.out_f32)                                 // row rr: 32-byte pairs of 16-byte chunks, pair j at (j ^ rr)
                *reinterpret_cast<float2*>(stg + rr * 256 + ((j ^ rr) << 5) + (lane & 3) * 8) = make_float2(o0, o1);
              else
                *reinterpret_cast<uint32_t*>(stg + rr * 128 + ((j ^ rr) << 4) + (lane & 3) * 4) = F::pack(o0, o1);
            }
            __syncwarp();
            if (a.out_f32) {
#pragma unroll
              for (int e = lane; e < 128; e += 32) {
                const int q = e >> 4, ch = e & 15;
                const uint4 v = *reinterpret_cast<const uint4*>(stg + q * 256 + (((ch >> 1) ^ q) << 5) + (ch & 1) * 16);
                *reinterpret_cast<uint4*>(a.out_f32 + (pix0 + q) * CI + n0 + c * 64 + ch * 4) = v;
              }
            } else {
#pragma unroll
              for (int e = lane; e < 64; e += 32) {
                const int q = e >> 3, ch = e & 7;
                const uint4 v = *reinterpret_cast<const uint4*>(stg + q * 128 + ((ch ^ q) << 4));
                *reinterpret_cast<uint4*>(a.y + (pix0 + q) * CI + n0 + c * 64 + ch * 8) = v;
              }
            }
            __syncwarp();
          }
        }
      if (a.res) {                                           // the residual's stages are free
        __syncwarp();
        if (lane == 0)
          for (int p = 0; p < K::NRES; ++p) tc_mbar_arrive(&empty[(it + p) % K::STAGES]);
        it += K::NRES;
      }
    }
  }
}

// CTAs of conv3x3_deep_kernel resident at once, or the error to return (<= 0).
template <class F, int W, int CI>
static int conv3x3_deep_slots() {
  using K = DeepCfg<W, CI>;
  auto kern = conv3x3_deep_kernel<F, W, CI>;
  static int slots = 0;
  if (!slots) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, K::SMEM) != cudaSuccess) return check_launch("cudaFuncSetAttribute(conv3x3_deep)");
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, CONV_THREADS, K::SMEM) != cudaSuccess) return check_launch("cudaOccupancyMaxActiveBlocksPerMultiprocessor(conv3x3_deep)");
    if (per_sm <= 0) { set_last_error("serl_conv3x3_res_h16: conv3x3_deep_kernel (%d B shared memory) cannot be resident", K::SMEM); return SERL_ERR_CUDA; }
    slots = per_sm * sms;
  }
  return slots;
}

template <class F, int W, int CI>
static int launch_conv3x3_deep(const serl_conv3x3_res_desc* d, cudaStream_t st) {
  using K = DeepCfg<W, CI>;
  auto kern = conv3x3_deep_kernel<F, W, CI>;
  const int slots = conv3x3_deep_slots<F, W, CI>();
  if (slots <= 0) return slots;
  TcEncodeTiledFn enc = tc_get_encode();
  if (!enc) { set_last_error("serl_conv3x3_res_h16: cuTensorMapEncodeTiled unavailable"); return SERL_ERR_CUDA; }
  const CUtensorMapDataType dt = d->fmt == SERL_FMT_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap xmap, wmap, rmap;
  {
    const cuuint64_t gdim[4] = {(cuuint64_t)CI, (cuuint64_t)W, (cuuint64_t)W, (cuuint64_t)d->N};
    const cuuint64_t gstr[3] = {(cuuint64_t)CI * 2, (cuuint64_t)W * CI * 2, (cuuint64_t)W * W * CI * 2};
    const cuuint32_t box[4] = {64u, (cuuint32_t)W, (cuuint32_t)W, (cuuint32_t)K::IMGS};
    const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult r = enc(&xmap, dt, 4, const_cast<void*>(d->x), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_conv3x3_res_h16: cuTensorMapEncodeTiled (input) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  {
    const cuuint64_t gdim[2] = {(cuuint64_t)9 * CI, (cuuint64_t)CI};
    const cuuint64_t gstr[1] = {(cuuint64_t)9 * CI * 2};
    const cuuint32_t box[2] = {64u, (cuuint32_t)K::BN};
    const cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(&wmap, dt, 2, const_cast<void*>(d->w), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_conv3x3_res_h16: cuTensorMapEncodeTiled (weights) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  rmap = wmap;                                               // not read without a residual
  if (d->res) {
    const cuuint64_t gdim[2] = {(cuuint64_t)CI, (cuuint64_t)d->N * W * W};
    const cuuint64_t gstr[1] = {(cuuint64_t)CI * 2};
    const cuuint32_t box[2] = {64u, 128u};
    const cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(&rmap, dt, 2, const_cast<void*>(d->res), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_last_error("serl_conv3x3_res_h16: cuTensorMapEncodeTiled (residual) failed (%d)", (int)r); return SERL_ERR_CUDA; }
  }
  DeepArgs a{};
  a.out_f32 = d->out_f32; a.y = d->out_f32 ? nullptr : static_cast<uint16_t*>(d->y);
  a.res = static_cast<const uint16_t*>(d->res); a.gamma = d->gamma; a.beta = d->beta;
  a.res_stats = d->res_stats; a.res_gamma = d->res_gamma; a.res_beta = d->res_beta;
  a.error = d->error; a.N = d->N; a.relu = d->relu; a.eps = d->eps;
  const int items = ceil_div(d->N, K::IMGS) * K::NSL;
  const int rounds = ceil_div(items, slots);                 // persistent: the fewest CTAs that still take `rounds` items each
  launch_k(kern, dim3(ceil_div(items, rounds)), dim3(CONV_THREADS), (size_t)K::SMEM, st, xmap, wmap, rmap, a);
  return check_launch("conv3x3_deep_kernel");
}

int stem_pool_resident(int fmt);                              // stem_pool.cu

}  // namespace serl

using namespace serl;

extern "C" int serl_trunk_resident_units(int launch, int fmt) {
  if (fmt != SERL_FMT_FP16 && fmt != SERL_FMT_BF16) { set_last_error("serl_trunk_resident_units: unknown format %d", fmt); return SERL_ERR_INVALID; }
  const bool h = fmt == SERL_FMT_FP16;
  switch (launch) {
    case SERL_TRUNK_STEM: return stem_pool_resident(fmt);
    case SERL_TRUNK_RES32: return h ? conv3x3_res_groups<Fp16, 32, 64>() : conv3x3_res_groups<Bf16, 32, 64>();
    case SERL_TRUNK_RES16: return h ? conv3x3_res_groups<Fp16, 16, 128>() : conv3x3_res_groups<Bf16, 16, 128>();
    case SERL_TRUNK_HEAD16: return h ? conv3x3_pp_slots<Fp16, 2, 16, 64>("serl_conv3x3s2_res_h16") : conv3x3_pp_slots<Bf16, 2, 16, 64>("serl_conv3x3s2_res_h16");
    case SERL_TRUNK_HEAD8: return h ? conv3x3_pp_slots<Fp16, 2, 8, 128>("serl_conv3x3s2_res_h16") : conv3x3_pp_slots<Bf16, 2, 8, 128>("serl_conv3x3s2_res_h16");
    case SERL_TRUNK_RES8: return h ? conv3x3_pp_slots<Fp16, 1, 8, 256>("serl_conv3x3_res_h16") : conv3x3_pp_slots<Bf16, 1, 8, 256>("serl_conv3x3_res_h16");
    case SERL_TRUNK_HEAD4: return h ? conv3x3s2_res_slots<Fp16, 4, 256>() : conv3x3s2_res_slots<Bf16, 4, 256>();
    case SERL_TRUNK_RES4: return h ? conv3x3_deep_slots<Fp16, 4, 512>() : conv3x3_deep_slots<Bf16, 4, 512>();
  }
  set_last_error("serl_trunk_resident_units: unknown launch %d", launch);
  return SERL_ERR_INVALID;
}

extern "C" int serl_conv3x3s2_res_h16(const serl_conv3x3s2_res_desc* d, void* stream) {
  if (!d || !d->x || !d->w || !d->w_proj || !d->y || !d->r || !d->gamma || !d->beta || !d->gamma_proj || !d->beta_proj || !d->error || d->N < 1) {
    set_last_error("serl_conv3x3s2_res_h16: invalid descriptor"); return SERL_ERR_INVALID;
  }
  if (d->Co != 2 * d->Ci) { set_last_error("serl_conv3x3s2_res_h16: Co == 2 Ci only (ResNet-10 stage heads)"); return SERL_ERR_UNSUPPORTED; }
  if (!((d->Wo == 16 && d->Co == 128) || (d->Wo == 8 && d->Co == 256) || (d->Wo == 4 && d->Co == 512))) {
    set_last_error("serl_conv3x3s2_res_h16: unsupported shape (Wo=%d, Ci=%d, Co=%d)", d->Wo, d->Ci, d->Co); return SERL_ERR_UNSUPPORTED;
  }
  const bool h = d->fmt == SERL_FMT_FP16;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (d->Wo == 16) return h ? launch_conv3x3s2_pp<Fp16, 16, 64>(d, st) : launch_conv3x3s2_pp<Bf16, 16, 64>(d, st);
  if (d->Wo == 8) return h ? launch_conv3x3s2_pp<Fp16, 8, 128>(d, st) : launch_conv3x3s2_pp<Bf16, 8, 128>(d, st);
  return h ? launch_conv3x3s2_res<Fp16, 4, 256>(d, st) : launch_conv3x3s2_res<Bf16, 4, 256>(d, st);
}

extern "C" int serl_conv3x3_res_h16(const serl_conv3x3_res_desc* d, void* stream) {
  if (!d || !d->x || !d->w || !d->gamma || !d->beta || !d->error || (!d->y && !d->out_f32) || d->N < 1) {
    set_last_error("serl_conv3x3_res_h16: invalid descriptor"); return SERL_ERR_INVALID;
  }
  if ((d->res_stats != nullptr) != (d->res_gamma != nullptr) || (d->res_stats != nullptr) != (d->res_beta != nullptr) || (d->res_stats && !d->res)) {
    set_last_error("serl_conv3x3_res_h16: res_stats / res_gamma / res_beta go together (and need res)"); return SERL_ERR_INVALID;
  }
  if (d->H != d->W || d->Co != d->Ci) { set_last_error("serl_conv3x3_res_h16: square maps with Ci == Co only"); return SERL_ERR_UNSUPPORTED; }
  if (!((d->W == 32 && d->Ci == 64) || (d->W == 16 && d->Ci == 128) || (d->W == 8 && d->Ci == 256) || (d->W == 4 && d->Ci == 512))) {
    set_last_error("serl_conv3x3_res_h16: unsupported shape (H=W=%d, Ci=%d, Co=%d): ResNet-10 block shapes at 128x128 input only", d->W, d->Ci, d->Co);
    return SERL_ERR_UNSUPPORTED;
  }
  if (d->out_f32 && d->W >= 16) {
    set_last_error("serl_conv3x3_res_h16: out_f32 at 8x8 and 4x4 only"); return SERL_ERR_UNSUPPORTED;
  }
  if (d->W == 32) {
    return d->fmt == SERL_FMT_FP16 ? launch_conv3x3_res<Fp16, 32, 64>(d, static_cast<cudaStream_t>(stream))
                                   : launch_conv3x3_res<Bf16, 32, 64>(d, static_cast<cudaStream_t>(stream));
  }
  if (d->W == 16) {
    return d->fmt == SERL_FMT_FP16 ? launch_conv3x3_res<Fp16, 16, 128>(d, static_cast<cudaStream_t>(stream))
                                   : launch_conv3x3_res<Bf16, 16, 128>(d, static_cast<cudaStream_t>(stream));
  }
  if (d->W == 8) {
    return d->fmt == SERL_FMT_FP16 ? launch_conv3x3_res8_pp<Fp16>(d, static_cast<cudaStream_t>(stream))
                                   : launch_conv3x3_res8_pp<Bf16>(d, static_cast<cudaStream_t>(stream));
  }
  return d->fmt == SERL_FMT_FP16 ? launch_conv3x3_deep<Fp16, 4, 512>(d, static_cast<cudaStream_t>(stream))
                                 : launch_conv3x3_deep<Bf16, 4, 512>(d, static_cast<cudaStream_t>(stream));
}
