// Frozen ResNet-10 trunk, 16-bit build: the input prep of the stem (stem_prep_kernel) and the second half of its fused max-pool
// (pool_finish_kernel), both on the product path, plus the unfused stem that the fused one (stem_pool.cu) is pinned to bit for
// bit: an implicit-GEMM conv on the Hopper tensor cores (conv_tc_kernel, wgmma with fp32 accumulators in registers,
// warp-specialised and persistent), serl_gn_finalize and maxpool_affine_kernel.  The other convs are conv3x3_res.cu.
//
// Layer algebra replaced (reference, relative to serl_launcher/serl_launcher): vision/resnet_v1.py:217-286
// (conv_init 7x7/2 -> GroupNorm(4) -> ReLU -> max_pool -> 4 ResNetBlocks), :129-156 (ResNetBlock).
// The 7x7/2 stem on 3 channels is rewritten exactly as a 4x4/1 convolution over a 2x2 space-to-depth image with
// 12 channels (zero-extended 8x8 kernel), which gives K = 4 kernel rows x (4 taps x 12 ch = 48, padded to 64).
// bf16 operands, fp32 accumulation: the 1e-2 tolerance build (north_star); the fp32 build is trunk_fp32.cu.

#include "common.cuh"
#include "conv_common.cuh"
#include "serl_b200.h"
#include "wgmma.cuh"

namespace serl {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;
constexpr int TC_A_STAGE = TC_BM * TC_BK * 2;          // 16 KiB
constexpr int TC_THREADS = 320;

struct ConvTcArgs {
  const uint16_t* x;             // 16-bit elements (bf16 or fp16, see the F template parameter)
  const uint16_t* w;             // [Co][num_kb * 64], K-major
  uint16_t* y;              // (M, Co) raw convolution output (pre-GroupNorm)
  float* stats;                  // (N, groups, 2): sum, sum of squares of the fp32 accumulators
  const float* in_a;             // unused (null)
  const float* in_b;
  int N, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad;
  int M, num_kb, cblocks, Cg;
  int32_t* error;
  int debug;                     // always 0; kept so the stem reference's SASS stays the one stem_pool_kernel was pinned to
};

// Persistent, role-decoupled implicit-GEMM convolution (im2col gather).  320 threads:
//   warps 0-3  one warpgroup: wgmma issue (two m64 halves x BN/64 n-chunks per k-step, fp32 accumulators in registers), then
//              the epilogue straight from the accumulator fragments (GroupNorm partial sums, 16-bit pack, NHWC store)
//   warps 4-7  A-operand producers (cp.async gather of 128 pixels x 64 K into 128B-swizzled smem, zero-fill at the padding)
//   warp 8     idle                     warp 9   TMA issuer for the weight (B) tile of every k-block
// A/B share one stage ring (full = 128 deferred cp.async arrivals + 1 expect_tx arrival; empty = one arrival per MMA warp once
// the k-block's MMAs have retired).  The producers run up to STAGES k-blocks ahead, across tile boundaries, so the next tile's
// operands arrive while the warpgroup stores the current one.
//
// Work items: a CTA walks tiles of 128 output positions x one BN-channel slice; the epilogue stores the raw 16-bit output and
// adds the GroupNorm sums to a.stats.  serl_conv2d_tc_h16 launches it as the stem only (<F, 64, 4, true>).
template <class F, int BN, int STAGES, bool kStem>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap wmap, const ConvTcArgs a) {
  pdl_prologue();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int B_STAGE = BN * TC_BK * 2;
  constexpr int NW = BN < 64 ? BN : 64;                      // MMA width: n-chunks of NW output channels
  constexpr int NC = BN / NW;
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * TC_A_STAGE;
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * B_STAGE);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles_n = a.Co / BN;                           // channel slices
  const int n_items = ceil_div(a.M, TC_BM) * n_tiles_n;
  const int HoWo = a.Ho * a.Wo;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { tc_mbar_init(&full[s], 129); tc_mbar_init(&empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == 9 && lane == 0) asm volatile("prefetch.tensormap [%0];" ::"l"(&wmap) : "memory");
  __syncthreads();

  if (warp >= 4 && warp < 8) {
    // ------------------------------- A producers -------------------------------
    // cp.async (LDGSTS) straight into the swizzled stage: no register staging, so a producer never waits for its own loads;
    // it only waits for a free stage, and up to STAGES k-blocks of gathers are in flight per CTA.  Completion is signalled
    // by cp.async.mbarrier.arrive.noinc (one deferred arrival per producer thread).
    const int tid = threadIdx.x - 128;
    const int chunk = tid & 7, rsub = tid >> 3;
    const int cpp = kStem ? 16 : a.Ci;                      // channels per input pixel (stem: 12 real + 4 zero-pad)
    bool ok = true;
    int it = 0;                                             // k-blocks produced so far (ring position)
    for (int item = blockIdx.x; item < n_items && ok; item += gridDim.x) {
      const int m0 = (item / n_tiles_n) * TC_BM;
      int rh[8], rw[8], rbase[8];                           // top-left input coords (rh = -100000 for rows past M), element offset
      {
        const int gm0 = m0 + rsub;
        int n = gm0 / HoWo; const int rem = gm0 - n * HoWo; int ho = rem / a.Wo; int wo = rem - ho * a.Wo;
#pragma unroll
        for (int i = 0; i < 8; ++i) {                       // rows rsub + 16 i: walk the output raster instead of dividing
          if (m0 + rsub + 16 * i < a.M) {
            rh[i] = ho * a.stride - a.pad; rw[i] = wo * a.stride - a.pad;
            rbase[i] = ((n * a.Hi + rh[i]) * a.Wi + rw[i]) * cpp;
          } else { rh[i] = -100000; rw[i] = 0; rbase[i] = 0; }
          wo += 16;
          while (wo >= a.Wo) { wo -= a.Wo; ++ho; }
          while (ho >= a.Ho) { ho -= a.Ho; ++n; }
        }
      }
      int tap_r = 0, tap_s = 0, cblk = 0;                   // k-block -> (kernel row, kernel col, channel block)
      for (int kb = 0; kb < a.num_kb && ok; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
        const int r = tap_r, sx = tap_s;
        const int tap_off = kStem ? kb * a.Wi * 16 : (r * a.Wi + sx) * a.Ci + cblk * TC_BK;
        if (!kStem) { if (++cblk == a.cblocks) { cblk = 0; if (++tap_s == a.kw) { tap_s = 0; ++tap_r; } } }
        ok = tc_mbar_wait(&empty[s], ph ^ 1u, a.error);
        const uint32_t As = smem_u32(sA + s * TC_A_STAGE);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = rsub + 16 * i;
          const uint32_t dst = As + (row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4);
          if (kStem) {
            // k-block = kernel row kb of the 4x4 space-to-depth kernel: 4 taps x 16 ch (12 real + 4 zero) = one aligned 128-byte row
            const bool inb = rh[i] > -100000;
            const uint16_t* src = a.x + (inb ? (size_t)(uint32_t)(rbase[i] + tap_off + chunk * 8) : 0);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(inb ? 16u : 0u) : "memory");
          } else {
            const int hi_ = rh[i] + r, wi_ = rw[i] + sx;
            const bool inb = hi_ >= 0 && hi_ < a.Hi && wi_ >= 0 && wi_ < a.Wi;
            const uint16_t* src = a.x + (inb ? (size_t)(uint32_t)(rbase[i] + tap_off + chunk * 8) : 0);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(inb ? 16u : 0u) : "memory");
          }
        }
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&full[s])) : "memory");
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else if (warp < 4) {
    // ------------------------------- MMA + epilogue (warpgroup 0) --------------------------------
    const uint32_t a_base = smem_u32(sA), b_base = smem_u32(sB);
    bool ok = true;
    int it = 0;
    for (int item = blockIdx.x; item < n_items && ok; item += gridDim.x) {
      const int m0 = (item / n_tiles_n) * TC_BM, n0 = (item % n_tiles_n) * BN;
      float acc[2][NC][NW / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int c = 0; c < NC; ++c)
#pragma unroll
          for (int i = 0; i < NW / 2; ++i) acc[h][c][i] = 0.f;
      for (int kb = 0; kb < a.num_kb && ok; ++kb, ++it) {
        const int s = it % STAGES;
        ok = tc_mbar_wait(&full[s], (uint32_t)(it / STAGES) & 1u, a.error);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // cp.async (generic proxy) writes -> tensor-core (async proxy) reads
        const uint32_t as = a_base + (uint32_t)(s * TC_A_STAGE), bs = b_base + (uint32_t)(s * B_STAGE);
        wg_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k)                 // k-step = 16 elements = 32 B: start address + 2 (x16 B)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int c = 0; c < NC; ++c)
              wg_mma_h16_n<F::kBf16, NW / 2>(acc[h][c], wg_desc(as + h * 8192) + 2 * k, wg_desc(bs + c * NW * 128) + 2 * k, 1u);
        wg_commit();
        if (kb > 0) {                                        // k-block kb-1 has retired: its stage is free
          wg_wait<1>();
          __syncwarp();
          if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % STAGES]);
        }
      }
      wg_wait<0>();
      __syncwarp();
      if (lane == 0) tc_mbar_arrive(&empty[(it - 1) % STAGES]);
      // rows 16 w .. 16 w + 15 of each m64 half belong to one image (Ho*Wo is a power of two >= 16)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rb = m0 + h * 64 + warp * 16;              // first row of this warp's 16-row block
        const bool valid = ok && rb < a.M;
        const int n_img = valid ? rb / HoWo : 0;
        const int r0 = rb + (lane >> 2);
#pragma unroll
        for (int c = 0; c < NC; ++c) {
#pragma unroll
          for (int j2 = 0; j2 < NW / 16; ++j2) {             // 16-channel chunks: one GroupNorm group (Cg >= 16)
            float s = 0.f, ss = 0.f;
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
              const int j = 2 * j2 + jj;
              const float* d = &acc[h][c][4 * j];
              s += (d[0] + d[1]) + (d[2] + d[3]);
              ss += (d[0] * d[0] + d[1] * d[1]) + (d[2] * d[2] + d[3] * d[3]);
              const int col = c * NW + 8 * j + 2 * (lane & 3);          // within the slice
              if (valid && !(a.debug & 1)) {
                *reinterpret_cast<uint32_t*>(a.y + (size_t)r0 * a.Co + n0 + col) = F::pack(d[0], d[1]);
                *reinterpret_cast<uint32_t*>(a.y + (size_t)(r0 + 8) * a.Co + n0 + col) = F::pack(d[2], d[3]);
              }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ss += __shfl_xor_sync(0xffffffffu, ss, o); }
            if (valid && lane == 0 && !(a.debug & 2)) {
              float* st = a.stats + ((size_t)n_img * 4 + ((n0 + c * NW + 16 * j2) / a.Cg)) * 2;
              atomicAdd(st, s); atomicAdd(st + 1, ss);
            }
          }
        }
      }
    }
  } else if (warp == 9) {
    // ------------------------------- weight TMA issuer ------------------------
    if (lane == 0) {
      bool ok = true;
      int it = 0;
      for (int item = blockIdx.x; item < n_items && ok; item += gridDim.x) {
        const int n0 = (item % n_tiles_n) * BN;
        for (int kb = 0; kb < a.num_kb && ok; ++kb, ++it) {
          const int s = it % STAGES;
          ok = tc_mbar_wait(&empty[s], ((uint32_t)(it / STAGES) & 1u) ^ 1u, a.error);
          if (!ok) break;
          tc_mbar_expect_tx(&full[s], (uint32_t)B_STAGE);
          tc_tma_2d(sB + s * B_STAGE, &wmap, kb * TC_BK, n0, &full[s]);
        }
      }
    }
  }
}

// ---- stem input: uint8 crops -> normalised 16-bit, 2x2 space-to-depth, zero padded: (N,67,67,16) [12 real + 4 zero ch] ----
template <class F>
__global__ void stem_prep_kernel(const uint8_t* __restrict__ x, uint16_t* __restrict__ xs, int N, int H, int W, int Hs, int Ws) {
  pdl_prologue();
  // a byte has 256 values: normalise each (channel, value) pair once per block (true fp32 divisions, as the fp32 build and
  // the oracle do) and look the 16-bit result up afterwards
  __shared__ uint16_t lut[3][256];
  {
    const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
    for (int i = threadIdx.x; i < 768; i += blockDim.x) {
      const int c = i >> 8, v = i & 255;
      lut[c][v] = (uint16_t)(F::pack(((float)v / 255.0f - mean[c]) / stdv[c], 0.f) & 0xFFFFu);
    }
  }
  __syncthreads();
  // blockIdx.x: 256 pixels of an image's Hs x Ws; blockIdx.y: images n, n + gridDim.y, ...  A thread keeps its pixel (aa, b)
  // across images, so the index arithmetic is one 32-bit division per thread rather than two 64-bit ones per pixel.
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= Hs * Ws) return;
  const int aa = e / Ws, b = e - aa * Ws;
  for (int n = blockIdx.y; n < N; n += gridDim.y) {
    uint32_t out[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};                    // 16 channels: (p, q, c) at pq*3 + c, channels 12..15 zero
#pragma unroll
    for (int pq = 0; pq < 4; ++pq) {
      const int p = pq >> 1, q = pq & 1;
      const int hi = 2 * aa + p - 3, wi = 2 * b + q - 3;          // explicit padding (3,3) of conv_init (resnet_v1.py:247)
      if (hi >= 0 && hi < H && wi >= 0 && wi < W) {
        const uint8_t* px = x + (((size_t)n * H + hi) * W + wi) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int ei = pq * 3 + c;
          const uint32_t h = lut[c][px[c]];
          out[ei >> 1] |= (ei & 1) ? (h << 16) : h;
        }
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(xs + ((size_t)n * Hs * Ws + e) * 16);
    dst[0] = make_uint4(out[0], out[1], out[2], out[3]); dst[1] = make_uint4(out[4], out[5], out[6], out[7]);
  }
}

// ---- GroupNorm finalize: sums -> per-(image, channel) affine  y = a*x + b --------------------------------
__global__ void gn_finalize_kernel(const float* __restrict__ stats, const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float* __restrict__ oa, float* __restrict__ ob, int N, int C, int Cg, float count, float eps) {
  pdl_prologue();
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * C) return;
  const int n = e / C, c = e - n * C, g = c / Cg;
  const float s = stats[((size_t)n * 4 + g) * 2], ss = stats[((size_t)n * 4 + g) * 2 + 1];
  const float mean = s / count;
  const float var = fmaxf(ss / count - mean * mean, 0.f);
  const float a = rsqrtf(var + eps) * gamma[c];
  oa[e] = a; ob[e] = beta[c] - mean * a;
}

// ---- max_pool 3x3/2 SAME over relu(a*x+b), bf16 in/out; thread per 8 channels ------------------------------
template <class F>
__global__ void maxpool_affine_kernel(const uint16_t* __restrict__ x, const float* __restrict__ ga, const float* __restrict__ gb,
                                     uint16_t* __restrict__ y, int N, int Hi, int Wi, int C, int Ho, int Wo) {
  pdl_prologue();
  const int c8n = C >> 3;
  const size_t total = (size_t)N * Ho * Wo * c8n;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(e % c8n); size_t r = e / c8n;
    const int wo = (int)(r % Wo); r /= Wo; const int ho = (int)(r % Ho); const int n = (int)(r / Ho);
    const float4 a0 = *reinterpret_cast<const float4*>(ga + (size_t)n * C + c8 * 8), a1 = *reinterpret_cast<const float4*>(ga + (size_t)n * C + c8 * 8 + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(gb + (size_t)n * C + c8 * 8), b1 = *reinterpret_cast<const float4*>(gb + (size_t)n * C + c8 * 8 + 4);
    const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w}, bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = 0.f;                               // relu output >= 0
    uint4 v[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) {                                         // all nine loads in flight before the first use
      const int hi = ho * 2 + t / 3, wi = wo * 2 + t % 3;                 // SAME on even sizes: pad low 0 / high 1
      v[t] = make_uint4(0u, 0u, 0u, 0u);
      if (hi < Hi && wi < Wi) v[t] = *reinterpret_cast<const uint4*>(x + (((size_t)n * Hi + hi) * Wi + wi) * C + c8 * 8);
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hi = ho * 2 + t / 3, wi = wo * 2 + t % 3;
      if (hi < Hi && wi < Wi) {
        const uint32_t u[4] = {v[t].x, v[t].y, v[t].z, v[t].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = F::unpack(u[j]);
          m[2 * j] = fmaxf(m[2 * j], fmaf(f.x, av[2 * j], bv[2 * j]));
          m[2 * j + 1] = fmaxf(m[2 * j + 1], fmaf(f.y, av[2 * j + 1], bv[2 * j + 1]));
        }
      }
    }
    *reinterpret_cast<uint4*>(y + (((size_t)n * Ho + ho) * Wo + wo) * C + c8 * 8) =
        make_uint4(F::pack(m[0], m[1]), F::pack(m[2], m[3]), F::pack(m[4], m[5]), F::pack(m[6], m[7]));
  }
}

// ---- second half of the fused stem max-pool: join unit-boundary rows with the side buffer, then relu(|a|*x' + b) ----
template <class F>
__global__ void pool_finish_kernel(const uint16_t* __restrict__ pooled, const uint16_t* __restrict__ side, const GnSrc g,
                                   uint16_t* __restrict__ y, int N) {
  pdl_prologue();
  const size_t total = (size_t)N * 32 * 32 * 8;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(e & 7); size_t r = e >> 3;
    const int j = (int)(r & 31); r >>= 5; const int p = (int)(r & 31); const int n = (int)(r >> 5);
    uint4 v = *reinterpret_cast<const uint4*>(pooled + e * 8);
    if ((p & 7) == 7 && p != 31) {
      const uint4 u = *reinterpret_cast<const uint4*>(side + (((size_t)n * 4 + ((p + 1) >> 3)) * 32 + j) * 64 + c8 * 8);
      v.x = F::max2(v.x, u.x); v.y = F::max2(v.y, u.y); v.z = F::max2(v.z, u.z); v.w = F::max2(v.w, u.w);
    }
    float a[8], b[8];
    gn_load8(g, n, 64, c8 * 8, a, b);
    v.x = affine_relu_x2<F>(v.x, fabsf(a[0]), b[0], fabsf(a[1]), b[1]); v.y = affine_relu_x2<F>(v.y, fabsf(a[2]), b[2], fabsf(a[3]), b[3]);
    v.z = affine_relu_x2<F>(v.z, fabsf(a[4]), b[4], fabsf(a[5]), b[5]); v.w = affine_relu_x2<F>(v.w, fabsf(a[6]), b[6], fabsf(a[7]), b[7]);
    *reinterpret_cast<uint4*>(y + e * 8) = v;
  }
}

template <class F, int BN, int STAGES, bool kStem>
static int launch_conv_tc(ConvTcArgs a, int fmt, cudaStream_t st) {
  const size_t smem = (size_t)STAGES * (TC_A_STAGE + BN * TC_BK * 2) + 1024 + 256;
  auto kern = conv_tc_kernel<F, BN, STAGES, kStem>;
  static size_t configured = 0;
  if (configured < smem) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return check_launch("cudaFuncSetAttribute(conv_tc)");
    configured = smem;
  }
  TcEncodeTiledFn enc = tc_get_encode();
  if (!enc) { set_last_error("serl_conv2d_tc_h16: cuTensorMapEncodeTiled unavailable"); return SERL_ERR_CUDA; }
  CUtensorMap map;
  const cuuint64_t Kp = (cuuint64_t)a.num_kb * TC_BK;
  const cuuint64_t gdim[2] = {Kp, (cuuint64_t)a.Co};
  const cuuint64_t gstr[1] = {Kp * 2};
  const cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)BN};
  const cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(&map, fmt == SERL_FMT_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                   const_cast<uint16_t*>(a.w), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("serl_conv2d_tc_h16: cuTensorMapEncodeTiled failed (%d)", (int)r); return SERL_ERR_CUDA; }
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
  const int items = ceil_div(a.M, TC_BM) * (a.Co / BN);
  const int grid = items < 2 * sms ? items : 2 * sms;                 // persistent: the CTAs walk the item list
  launch_k(kern, grid, TC_THREADS, smem, st, map, a);
  return check_launch("conv_tc_kernel");
}

}  // namespace serl

using namespace serl;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int serl_trunk_stem_prep_h16(const uint8_t* x, void* xs, int N, int H, int W, int fmt, void* stream) {
  const int Hs = H / 2 + 3, Ws = W / 2 + 3;
  // about 132 x 16 blocks in all, as many images per block as that leaves, so each block's LUT serves several images
  const int bx = ceil_div(Hs * Ws, 256);
  const dim3 blocks(bx, std::max(1, std::min(std::min(N, 132 * 16 / bx), 65535)));
  if (fmt == SERL_FMT_FP16) launch_k(stem_prep_kernel<Fp16>, blocks, 256, 0, ST(stream), x, static_cast<uint16_t*>(xs), N, H, W, Hs, Ws);
  else launch_k(stem_prep_kernel<Bf16>, blocks, 256, 0, ST(stream), x, static_cast<uint16_t*>(xs), N, H, W, Hs, Ws);
  return check_launch("stem_prep_kernel");
}

extern "C" int serl_conv2d_tc_h16(const serl_conv_tc_desc* d, void* stream) {
  if (!d || !d->x || !d->w || !d->y || !d->stats || !d->error) { set_last_error("serl_conv2d_tc_h16: invalid descriptor"); return SERL_ERR_INVALID; }
  if (!d->stem || d->in_a) {
    set_last_error("serl_conv2d_tc_h16: only the stem conv (stem=1, no operand transform) is supported; the trunk's other convs are "
                   "serl_conv3x3_res_h16 / serl_conv3x3s2_res_h16");
    return SERL_ERR_UNSUPPORTED;
  }
  ConvTcArgs a{};
  a.x = static_cast<const uint16_t*>(d->x); a.w = static_cast<const uint16_t*>(d->w); a.y = static_cast<uint16_t*>(d->y);
  a.stats = d->stats; a.error = d->error;
  a.N = d->N; a.Hi = d->Hi; a.Wi = d->Wi; a.Ci = d->Ci; a.Co = d->Co; a.kh = d->kh; a.kw = d->kw; a.stride = d->stride; a.pad = d->pad_lo;
  a.Ho = d->Ho; a.Wo = d->Wo; a.M = d->N * d->Ho * d->Wo; a.Cg = d->Co / 4;
  a.num_kb = 4; a.cblocks = 1;
  const int HoWo = d->Ho * d->Wo;
  if (d->Co != 64 || (HoWo & (HoWo - 1)) != 0 || HoWo < 16) {
    set_last_error("serl_conv2d_tc_h16: unsupported stem shape (Co=%d Ho*Wo=%d; expects Co=64)", d->Co, HoWo); return SERL_ERR_UNSUPPORTED;
  }
  return d->fmt == SERL_FMT_FP16 ? launch_conv_tc<Fp16, 64, 4, true>(a, d->fmt, ST(stream)) : launch_conv_tc<Bf16, 64, 4, true>(a, d->fmt, ST(stream));
}

static GnSrc gn_table(const float* a, const float* b) { GnSrc g{}; g.a = a; g.b = b; return g; }
static GnSrc gn_sums(const float* stats, const float* gamma, const float* beta, int C, int HW, float eps) {
  GnSrc g{}; g.stats = stats; g.gamma = gamma; g.beta = beta; g.Cg = C / 4; g.count = (float)HW * (float)(C / 4); g.eps = eps; return g;
}

static int launch_pool_finish(const void* pooled, const void* side, const GnSrc& g, void* y, int N, int fmt, void* stream) {
  const size_t total = (size_t)N * 32 * 32 * 8;
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
  if (fmt == SERL_FMT_FP16)
    launch_k(pool_finish_kernel<Fp16>, blocks, 256, 0, ST(stream), static_cast<const uint16_t*>(pooled), static_cast<const uint16_t*>(side), g, static_cast<uint16_t*>(y), N);
  else
    launch_k(pool_finish_kernel<Bf16>, blocks, 256, 0, ST(stream), static_cast<const uint16_t*>(pooled), static_cast<const uint16_t*>(side), g, static_cast<uint16_t*>(y), N);
  return check_launch("pool_finish_kernel");
}
extern "C" int serl_pool_finish_h16(const void* pooled, const void* side, const float* a, const float* b, void* y, int N, int fmt, void* stream) {
  return launch_pool_finish(pooled, side, gn_table(a, b), y, N, fmt, stream);
}
extern "C" int serl_pool_finish_gn_h16(const void* pooled, const void* side, const float* stats, const float* gamma, const float* beta, void* y,
                                       int N, float eps, int fmt, void* stream) {
  return launch_pool_finish(pooled, side, gn_sums(stats, gamma, beta, 64, 64 * 64, eps), y, N, fmt, stream);
}

extern "C" int serl_gn_finalize(const float* stats, const float* gamma, const float* beta, float* out_a, float* out_b, int N, int C,
                                int HW, float eps, void* stream) {
  const int Cg = C / 4;
  launch_k(gn_finalize_kernel, ceil_div(N * C, 256), 256, 0, ST(stream), stats, gamma, beta, out_a, out_b, N, C, Cg, (float)HW * (float)Cg, eps);
  return check_launch("gn_finalize_kernel");
}

extern "C" int serl_maxpool_affine_h16(const void* x, const float* a, const float* b, void* y, int N, int Hi, int Wi, int C, int fmt, void* stream) {
  const int Ho = Hi / 2, Wo = Wi / 2;
  size_t total = (size_t)N * Ho * Wo * (C / 8);
  int blocks = (int)((total + 255) / 256); if (blocks > 132 * 16) blocks = 132 * 16;
  auto xi = static_cast<const uint16_t*>(x); auto yo = static_cast<uint16_t*>(y);
  if (fmt == SERL_FMT_FP16) launch_k(maxpool_affine_kernel<Fp16>, blocks, 256, 0, ST(stream), xi, a, b, yo, N, Hi, Wi, C, Ho, Wo);
  else launch_k(maxpool_affine_kernel<Bf16>, blocks, 256, 0, ST(stream), xi, a, b, yo, N, Hi, Wi, C, Ho, Wo);
  return check_launch("maxpool_affine_kernel");
}
