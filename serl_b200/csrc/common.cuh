// Shared device helpers for libserl_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define SERL_OK 0
#define SERL_ERR_INVALID (-1)
#define SERL_ERR_CUDA (-2)
#define SERL_ERR_UNSUPPORTED (-3)

namespace serl {

void set_last_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError -> SERL_OK / SERL_ERR_CUDA (+ message)

// ---------------------------------------------------------------------------------------------
// Kernel launches.
// `pdl_prologue()` is the first statement of every kernel.  Its two griddepcontrol instructions act only on a launch that sets
// cudaLaunchAttributeProgrammaticStreamSerialization, and no launch here sets it, so they are no-ops.  They stay so that the
// kernels' SASS, including the hand-scheduled trunk kernels', is unchanged; removing them wants a timed change of its own.
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_prologue() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
#endif

template <class... P, class... A>
inline void launch_k(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchKernelEx(&cfg, kern, static_cast<P>(args)...);          // errors are picked up by check_launch()
}
// launch_k for thread-block clusters of cluster_x CTAs along x (cluster_x == 1: no cluster attribute)
template <class... P, class... A>
inline void launch_k_cluster(void (*kern)(P...), dim3 grid, dim3 block, int cluster_x, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  if (cluster_x > 1) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster_x; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
  }
  cudaLaunchKernelEx(&cfg, kern, static_cast<P>(args)...);
}

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
// Grid of a persistent one-CTA-per-SM kernel that walks `items` work items: the makespan is ceil(items / grid) items whatever the
// grid, so take the SMALLEST grid with the same number of waves as a full one (512 items on 132 SMs: 4 waves either way -> 128
// CTAs).  The SMs left over run the short kernels of the other streams (heads of the current step next to the trunk of the next,
// the other camera's trunk) instead of making them wait for a whole persistent kernel.
int balanced_grid(int items, int sms);

__host__ __device__ inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------------------
// Threefry-2x32-20: the JAX PRNG block function (restated in oracle/jax_prng.py, same KATs).
// ---------------------------------------------------------------------------------------------
struct u32x2 { uint32_t x, y; };

__host__ __device__ inline uint32_t rotl32(uint32_t v, int d) { return (v << d) | (v >> (32 - d)); }

__host__ __device__ inline u32x2 threefry2x32(u32x2 key, uint32_t c0, uint32_t c1) {
  const uint32_t ks0 = key.x, ks1 = key.y, ks2 = key.x ^ key.y ^ 0x1BD11BDAu;
  uint32_t x0 = c0 + ks0, x1 = c1 + ks1;
#define SERL_TF_R(d) { x0 += x1; x1 = rotl32(x1, d); x1 ^= x0; }
  SERL_TF_R(13) SERL_TF_R(15) SERL_TF_R(26) SERL_TF_R(6)
  x0 += ks1; x1 += ks2 + 1u;
  SERL_TF_R(17) SERL_TF_R(29) SERL_TF_R(16) SERL_TF_R(24)
  x0 += ks2; x1 += ks0 + 2u;
  SERL_TF_R(13) SERL_TF_R(15) SERL_TF_R(26) SERL_TF_R(6)
  x0 += ks0; x1 += ks1 + 3u;
  SERL_TF_R(17) SERL_TF_R(29) SERL_TF_R(16) SERL_TF_R(24)
  x0 += ks1; x1 += ks2 + 4u;
  SERL_TF_R(13) SERL_TF_R(15) SERL_TF_R(26) SERL_TF_R(6)
  x0 += ks2; x1 += ks0 + 5u;
#undef SERL_TF_R
  return u32x2{x0, x1};
}

// jax.random.split(key, n)[i] in the original (non-partitionable) layout:
// flat = concat(y0[0..n), y1[0..n)) with (y0[j], y1[j]) = TF(key, (j, n + j)); key_i = (flat[2i], flat[2i+1]).
__host__ __device__ inline u32x2 jax_split_at(u32x2 key, uint32_t n, uint32_t i) {
  uint32_t f[2];
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    uint32_t pos = 2u * i + (uint32_t)s;            // index into flat (length 2n)
    uint32_t j = pos < n ? pos : pos - n;
    u32x2 y = threefry2x32(key, j, n + j);
    f[s] = pos < n ? y.x : y.y;
  }
  return u32x2{f[0], f[1]};
}

// jax.random.fold_in(key, data) (data < 2^32).
__host__ __device__ inline u32x2 jax_fold_in(u32x2 key, uint32_t data) { return threefry2x32(key, 0u, data); }

// Element j of jax's random_bits(key, 32, shape) with `size` total elements.
__host__ __device__ inline uint32_t jax_random_bits_at(u32x2 key, uint32_t size, uint32_t j) {
  uint32_t h = (size + 1u) >> 1;                    // half length after padding to even
  if (j < h) {
    uint32_t c1 = (j + h < size) ? j + h : 0u;      // the pad element is a zero counter
    return threefry2x32(key, j, c1).x;
  }
  return threefry2x32(key, j - h, j).y;
}

// jax.random.randint(key, (2,), 0, span) for small spans (span^2 < 2^32): both elements.
__host__ __device__ inline void jax_randint2(u32x2 key, uint32_t span, int* out0, int* out1) {
  u32x2 k1 = jax_split_at(key, 2, 0), k2 = jax_split_at(key, 2, 1);
  u32x2 hb = threefry2x32(k1, 0u, 1u);              // random_bits(k1, (2,)): counters [0],[1]
  u32x2 lb = threefry2x32(k2, 0u, 1u);
  uint32_t mult = 65536u % span; mult = (mult * mult) % span;
  *out0 = (int)(((hb.x % span) * mult + (lb.x % span)) % span);
  *out1 = (int)(((hb.y % span) * mult + (lb.y % span)) % span);
}

__device__ inline float bits_to_uniform01(uint32_t bits) {
  return __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f;
}

// Giles' single-precision erfinv (the polynomial XLA uses for f32 erf_inv).
__device__ inline float erfinv_giles(float x) {
  float w = -log1pf(-x * x);
  float p;
  if (w < 5.0f) {
    w = w - 2.5f;
    p = 2.81022636e-08f;
    p = fmaf(p, w, 3.43273939e-07f);  p = fmaf(p, w, -3.5233877e-06f);
    p = fmaf(p, w, -4.39150654e-06f); p = fmaf(p, w, 0.00021858087f);
    p = fmaf(p, w, -0.00125372503f);  p = fmaf(p, w, -0.00417768164f);
    p = fmaf(p, w, 0.246640727f);     p = fmaf(p, w, 1.50140941f);
  } else {
    w = sqrtf(w) - 3.0f;
    p = -0.000200214257f;
    p = fmaf(p, w, 0.000100950558f);  p = fmaf(p, w, 0.00134934322f);
    p = fmaf(p, w, -0.00367342844f);  p = fmaf(p, w, 0.00573950773f);
    p = fmaf(p, w, -0.0076224613f);   p = fmaf(p, w, 0.00943887047f);
    p = fmaf(p, w, 1.00167406f);      p = fmaf(p, w, 2.83297682f);
  }
  return p * x;
}

// jax.random.normal element from its 32 random bits.
__device__ inline float bits_to_normal(uint32_t bits) {
  const float lo = -0.99999994f;                    // nextafter(-1, 0)
  float f = bits_to_uniform01(bits);
  float u = fmaxf(lo, __fadd_rn(__fmul_rn(f, 2.0f), lo));   // (hi - lo) rounds to 2.0f in fp32
  return 1.41421356237f * erfinv_giles(u);
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10: replay index draws (repo spec, see oracle/replay.py::draw_indices).
// ---------------------------------------------------------------------------------------------
struct u32x4 { uint32_t x, y, z, w; };

__host__ __device__ inline u32x4 philox4x32_10(u32x4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c.x;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c.z;
    u32x4 n;
    n.x = (uint32_t)(p1 >> 32) ^ c.y ^ k0;
    n.y = (uint32_t)p1;
    n.z = (uint32_t)(p0 >> 32) ^ c.w ^ k1;
    n.w = (uint32_t)p0;
    c = n;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c;
}

// ---------------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------------
__device__ inline float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ inline float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum of two values; result broadcast to all threads.  blockDim.x multiple of 32, <= 1024.
__device__ inline void block_sum2(float& a, float& b, float* smem /* >= 64 floats */) {
  a = warp_sum(a); b = warp_sum(b);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) { smem[w] = a; smem[32 + w] = b; }
  __syncthreads();
  float x = (l < nw) ? smem[l] : 0.f, y = (l < nw) ? smem[32 + l] : 0.f;
  a = warp_sum(x); b = warp_sum(y);
}

}  // namespace serl
