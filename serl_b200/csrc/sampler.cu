// Replay minibatch sampler for the HBM-resident frame-dedup ring.
//
// ONE kernel per (buffer, step): draws uniform indices (Philox4x32-10 + Lemire, bounded redraw on
// invalid slots), gathers (s, a, r, s', mask, done) and the T+1 adjacent camera frames, and applies
// the DrQ random shift (edge-replicating crop) on the way out.  Frames are staged global->shared with
// a TMA bulk copy (cp.async.bulk, 16-byte aligned row ranges) and written back with 128-bit stores.
//
// Replaces (reference, relative to serl_launcher/serl_launcher):
//   data/memory_efficient_replay_buffer.py:91-164  sample()      (host python loop + numpy gather)
//   data/replay_buffer.py:77-90                    get_iterator  (host->device copy of the batch)
//   utils/train_utils.py:44-66                     _unpack
//   vision/data_augmentations.py:7-36 + agents/continuous/drq.py:244-253  batched_random_crop
// Semantics are restated in oracle/replay.py (draw_indices, gather_packed, random_shift) and
// oracle/jax_prng.py (crop_offsets).  serl_replay_sample_crop_nstep runs the same kernels instantiated with kNStep: each
// row then carries the n-step window that starts at its slot (nstep_window / nstep_scalars; oracle/nstep.py).
#include <cstring>

#include "common.cuh"
#include "serl_b200.h"

namespace serl {

constexpr int kBandRows = 32;
constexpr int kSamplerThreads = 128;
constexpr int kMaxDrawAttempts = 64;

struct SamplerArgs {
  serl_replay_view rv;
  // draw
  uint64_t seed, step;
  const uint64_t* step_dev;      // optional device counter overriding `step` (CUDA-graph replays)
  const int32_t* size_dev;       // optional device fill level overriding rv.size
  uint32_t lane_offset;          // philox lane of row 0 (independent of out_row_offset)
  const int32_t* explicit_idx;   // optional (B): skip the draw
  // crop
  const uint32_t* key_obs;       // device, 2 words: JAX key whose split(key, crop_total)[g] seeds frame g
  const uint32_t* key_next;
  const int32_t* explicit_off_obs;   // optional (crop_total, 2) [cy, cx]
  const int32_t* explicit_off_next;
  int crop_total;                // total frames in the (possibly concatenated) batch = B_total * T
  int out_row_offset;            // first output row of this launch inside the B_total-row outputs
  int padding;
  // outputs (B_total rows each)
  uint8_t* obs_pix[SERL_MAX_CAMS];    // (B_total, T, H, W, C)
  uint8_t* next_pix[SERL_MAX_CAMS];
  float* obs_state; float* next_state; float* actions; float* rewards; float* masks;
  uint8_t* dones; int32_t* idx_out; int32_t* off_obs_out; int32_t* off_next_out;   // off_*: (B_total*T, 2)
  int32_t* status;               // device int, OR-ed with 1 when a draw fails
  int batch;                     // rows produced by this launch
  // n-step window (serl_replay_sample_crop_nstep only; the kernels' kNStep = false instantiations never read these)
  int n_step;                    // window bound n, 1..SERL_MAX_NSTEP
  float discount;
  const int32_t* head_dev;       // device ring insert index: the newest written slot is head - 1
  int32_t* m_out;                // optional (B_total) window length m
  int32_t* next_idx_out;         // optional (B_total) slot i + m - 1 whose next observation the row carries
};

// Prioritized draw (serl_replay_sample_crop_prio): a kernel parameter of its own after SamplerArgs, as the shard table is, so
// the uniform kernels' parameters keep their layout.
struct PrioDraw {
  const float* tree;             // sum tree (serl_priority_tree layout), leaves first
  int levels;
  int off[SERL_MAX_TREE_LEVELS];
  float* prio_out;               // optional (B_total) leaf of each row's slot
};

// Level offsets of the sum tree over `cap` leaves (include/serl_b200.h); returns the number of levels.
__host__ __device__ inline int prio_tree_layout(int cap, int* off) {
  int n = cap, o = 0, levels = 0;
  for (;;) {
    off[levels++] = o;
    if (n == 1) return levels;
    o += n;
    n = (n + SERL_PRIO_FANOUT - 1) / SERL_PRIO_FANOUT;
  }
}

#ifdef __CUDA_ARCH__
#define PRIO_ADD(x, y) __fadd_rn(x, y)
#define PRIO_SUB(x, y) __fsub_rn(x, y)
#define PRIO_MUL(x, y) __fmul_rn(x, y)
#define PRIO_DIV(x, y) __fdiv_rn(x, y)
#else
#define PRIO_ADD(x, y) ((x) + (y))
#define PRIO_SUB(x, y) ((x) - (y))
#define PRIO_MUL(x, y) ((x) * (y))
#define PRIO_DIV(x, y) ((x) / (y))
#endif

// One attempt of the proportional draw of row b of B (include/serl_b200.h): the slot the descent lands on, or -1 when it
// meets a node whose children are all 0.  *p = that leaf.  One thread walks the <= 32 children of each node in order (a
// 1M-slot ring: 4 levels, each node's children one 128-byte line).
__host__ __device__ inline int prio_descend(const float* tree, const int* off, int levels, int b, int B, uint32_t x, float* p) {
  float u = PRIO_MUL(PRIO_DIV(PRIO_ADD((float)b, PRIO_MUL((float)x, 0x1p-32f)), (float)B), tree[off[levels - 1]]);
  int j = 0;
  for (int l = levels - 1; l >= 1; --l) {
    const float* ch = tree + off[l - 1];
    const int c0 = SERL_PRIO_FANOUT * j, c1 = min(c0 + SERL_PRIO_FANOUT, off[l] - off[l - 1]);
    float s = 0.f, s_nz = 0.f;
    int pick = -1, nz = -1;
    for (int c = c0; c < c1; ++c) {
      const float v = ch[c];
      const float s2 = PRIO_ADD(s, v);
      if (s2 > u) { pick = c; break; }
      if (v != 0.f) { nz = c; s_nz = s; }
      s = s2;
    }
    if (pick < 0) {
      if (nz < 0) return -1;
      pick = nz; s = s_nz;
    }
    u = PRIO_SUB(u, s);
    j = pick;
  }
  *p = tree[j];
  return j;
}

__device__ inline int draw_index(const SamplerArgs& a, uint32_t lane) {
  const uint32_t size = (uint32_t)(a.size_dev ? *a.size_dev : a.rv.size);
  const uint64_t step = a.step_dev ? *a.step_dev : a.step;
  if (size == 0) return -1;
  const uint32_t thresh = (uint32_t)((0x100000000ull - size) % size);
  for (int att = 0; att < kMaxDrawAttempts; ++att) {
    u32x4 r = philox4x32_10(u32x4{lane, (uint32_t)att, (uint32_t)step, (uint32_t)(step >> 32)},
                            (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
    uint64_t m = (uint64_t)r.x * size;
    if ((uint32_t)m < thresh) continue;
    uint32_t idx = (uint32_t)(m >> 32);
    if (a.rv.valid[idx]) return (int)idx;
  }
  return -1;
}

// Proportional draw of output row b of this launch (lane lane_offset + b).  A leaf is 0 while its slot is not valid; the validity
// check repeats that rule for the draw itself, as the uniform draw's does.
__device__ inline int draw_index_prio(const SamplerArgs& a, const PrioDraw& pd, int b) {
  const uint64_t step = a.step_dev ? *a.step_dev : a.step;
  for (int att = 0; att < kMaxDrawAttempts; ++att) {
    u32x4 r = philox4x32_10(u32x4{a.lane_offset + (uint32_t)b, (uint32_t)att, (uint32_t)step, (uint32_t)(step >> 32)},
                            (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
    float p;
    const int idx = prio_descend(pd.tree, pd.off, pd.levels, b, a.batch, r.x, &p);
    if (idx >= 0 && p > 0.f && a.rv.valid[idx]) return idx;
  }
  return -1;
}

template <bool kPrio>
__device__ __forceinline__ int draw_row(const SamplerArgs& a, const PrioDraw* pd, int i) {
  if (a.explicit_idx) return a.explicit_idx[i];
  if constexpr (kPrio) return draw_index_prio(a, *pd, i);
  else return draw_index(a, a.lane_offset + (uint32_t)i);
}

// n-step window of drawn slot idx: the largest m <= n such that slots idx .. idx+m-1 (mod capacity) are written (at or behind
// the newest slot, head - 1) and valid, and none of idx .. idx+m-2 ends an episode.  Returns the window's last slot j; *m_out = m.
// A written slot after idx is invalid only where the frame-dedup ring re-inserted the last T frames at the front on a mid-episode
// wrap: those copies are not the next transition, so the window stops before them.
__device__ inline int nstep_window(const SamplerArgs& a, int idx, int* m_out) {
  const int cap = a.rv.capacity;
  const int head = *a.head_dev;
  const int avail = (head - idx - 1 + 2 * cap) % cap + 1;   // slots idx .. head-1 in insertion order
  const int lim = min(a.n_step, avail);
  int j = idx, m = 1;
  while (m < lim && !a.rv.dones[j]) {
    const int nx = j + 1 == cap ? 0 : j + 1;
    if (!a.rv.valid[nx]) break;
    j = nx; ++m;
  }
  *m_out = m;
  return j;
}

// The row's n-step scalars in the documented fp32 order (no FMA contraction):
//   g = 1, R = r[idx];  for k = 1 .. m-1: g = g * discount, R = R + g * r[idx+k];  masks = g * masks[j];  dones = dones[j].
// With m = 1 this is r[idx], masks[idx], dones[idx] bit for bit.
__device__ inline void nstep_scalars(const SamplerArgs& a, int idx, int j, int m, int out_row) {
  const int cap = a.rv.capacity;
  float g = 1.f, R = a.rv.rewards[idx];
  for (int k = 1, s = idx; k < m; ++k) {
    s = s + 1 == cap ? 0 : s + 1;
    g = __fmul_rn(g, a.discount);
    R = __fadd_rn(R, __fmul_rn(g, a.rv.rewards[s]));
  }
  a.rewards[out_row] = R;
  a.masks[out_row] = __fmul_rn(g, a.rv.masks[j]);
  a.dones[out_row] = a.rv.dones[j];
  if (a.m_out) a.m_out[out_row] = m;
  if (a.next_idx_out) a.next_idx_out[out_row] = j;
}

__device__ inline void crop_offset_for(const uint32_t* key, const int32_t* expl, int crop_total, int g,
                                       int span, int* cy, int* cx) {
  if (expl) { *cy = expl[2 * g]; *cx = expl[2 * g + 1]; return; }
  u32x2 k = jax_split_at(u32x2{key[0], key[1]}, (uint32_t)crop_total, (uint32_t)g);
  jax_randint2(k, (uint32_t)span, cy, cx);
}

// Source of frame `slot` of the window that starts at slot w0 (slots w0 .. w0 + T, window end w0 + T < capacity).  kShard:
// the frames live in their owners' allocations (serl_replay_shards); the owner of the window end also stores the halo of T
// slots in front of its range, so the whole window is read from that one allocation.  !kShard: the ring's own frames.
template <bool kShard>
__device__ __forceinline__ const uint8_t* window_frame(const serl_replay_view& rv, const serl_replay_shards* sh, int cam, int w0, int slot,
                                                       size_t frame_bytes) {
  if constexpr (kShard) {
    const int o = (w0 + rv.num_stack) / sh->slots_per_rank;
    return sh->frames[cam][o] + (size_t)(slot - o * sh->slots_per_rank + sh->halo) * frame_bytes;
  } else {
    return rv.frames[cam] + (size_t)slot * frame_bytes;
  }
}

__device__ inline void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ inline void mbar_wait(uint64_t* bar, uint32_t phase) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(bar), done = 0;
  while (!done) {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(done) : "r"(addr), "r"(phase) : "memory");
  }
}
__device__ inline void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "r"(bytes),
                 "r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
}

// grid: x = band, y = (cam, which, t) flattened, z = row i.   kFast: row_bytes % 16 == 0.   kNStep: rows carry the n-step window
// (next observation, rewards, masks, dones of the window ending at slot s_nidx).  kStacked (bytewise only): the outputs are
// (B_total, H, W, T*C), frame t's channels at t*C .. t*C + C-1 (serl_batch_out.stacked).
template <bool kFast, bool kNStep, bool kShard, bool kPrio = false, bool kStacked = false>
__device__ __forceinline__ void sample_gather_crop_body(const SamplerArgs& a, const serl_replay_shards* shards, const PrioDraw* pd = nullptr) {
  static_assert(!(kFast && kStacked), "the stacked layout has no banded 16-byte path");
  pdl_prologue();
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  __shared__ int s_idx, s_nidx, s_m, s_cy, s_cx;

  const serl_replay_view& rv = a.rv;
  const int T = rv.num_stack, H = rv.height, W = rv.width, C = rv.channels;
  const int row_bytes = W * C;
  const int band = blockIdx.x;
  int yz = blockIdx.y;
  const int t = yz % T; yz /= T;
  const int which = yz & 1; yz >>= 1;
  const int cam = yz;
  const int i = blockIdx.z;
  const int out_row = a.out_row_offset + i;
  const int g = out_row * T + t;                         // frame index inside the batch
  const int y0 = band * kBandRows;
  const int rows = min(kBandRows, H - y0);
  const bool leader = (cam == 0 && which == 0 && t == 0 && band == 0);

  if (threadIdx.x == 0) {
    int idx = draw_row<kPrio>(a, pd, i);
    int cy = a.padding, cx = a.padding;
    if (rv.num_cams > 0)
      crop_offset_for(which ? a.key_next : a.key_obs, which ? a.explicit_off_next : a.explicit_off_obs,
                      a.crop_total, g, 2 * a.padding + 1, &cy, &cx);
    s_idx = idx; s_cy = cy; s_cx = cx;
    if (idx < 0) atomicOr(a.status, 1);
    if constexpr (kNStep) { if (idx >= 0 && (which || leader)) s_nidx = nstep_window(a, idx, &s_m); }
    if (cam == 0 && band == 0 && rv.num_cams > 0) {       // record offsets once per (which, t)
      int32_t* o = which ? a.off_next_out : a.off_obs_out;
      if (o) { o[2 * g] = cy; o[2 * g + 1] = cx; }
    }
    if (kFast) { mbar_init(&bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  }
  __syncthreads();
  const int idx = s_idx, cy = s_cy, cx = s_cx;
  if (idx < 0) return;
  const int nidx = kNStep && (which || leader) ? s_nidx : idx;   // slot whose next observation the row carries

  // ---- small fields: one CTA per row ---------------------------------------------------------
  if (leader) {
    const int ns = T * rv.state_dim;
    for (int k = threadIdx.x; k < ns; k += blockDim.x) {
      a.obs_state[(size_t)out_row * ns + k] = rv.state[(size_t)idx * ns + k];
      a.next_state[(size_t)out_row * ns + k] = rv.next_state[(size_t)nidx * ns + k];
    }
    for (int k = threadIdx.x; k < rv.action_dim; k += blockDim.x)
      a.actions[(size_t)out_row * rv.action_dim + k] = rv.actions[(size_t)idx * rv.action_dim + k];
    if (threadIdx.x == 0) {
      if constexpr (kNStep) {
        nstep_scalars(a, idx, nidx, s_m, out_row);
      } else {
        a.rewards[out_row] = rv.rewards[idx];
        a.masks[out_row] = rv.masks[idx];
        a.dones[out_row] = rv.dones[idx];
      }
      if (a.idx_out) a.idx_out[out_row] = idx;
      if constexpr (kPrio) { if (pd->prio_out) pd->prio_out[out_row] = pd->tree[idx]; }
    }
  }

  if (rv.num_cams == 0) return;                          // state-only ring (data/replay_buffer.py:40-75)

  // ---- frame band: slot idx - T + t + which, rows clamp(y + cy - pad) ---------------------------
  const size_t frame_bytes = (size_t)H * row_bytes;
  // window idx - T of numpy's sliding_window_view over the (capacity) slot axis; the reference indexes it with idx - T as is, so a
  // valid slot idx < T (first transition of an episode whose filler frame sits at the END of the ring) gets numpy's negative-index
  // window = the LAST one, slots capacity-T-1 .. capacity-1 (memory_efficient_replay_buffer.py:148-151; pinned by tests/golden/replay_wrap_first.npz)
  const int widx = which ? nidx : idx;
  const int w0 = widx - T + ((widx - T) < 0 ? rv.capacity - T : 0);
  const int slot = w0 + t + which;
  const uint8_t* src = window_frame<kShard>(rv, shards, cam, w0, slot, frame_bytes);
  uint8_t* dst;
  if constexpr (kStacked) dst = (which ? a.next_pix[cam] : a.obs_pix[cam]) + ((size_t)out_row * H + y0) * row_bytes * T;
  else dst = (which ? a.next_pix[cam] : a.obs_pix[cam]) + ((size_t)g * H + y0) * row_bytes;
  const int dy = cy - a.padding;
  const int sh = (cx - a.padding) * C;                   // byte shift inside a row
  const int r_lo = min(max(y0 + dy, 0), H - 1);
  const int r_hi = min(max(y0 + rows - 1 + dy, 0), H - 1);

  if (kFast) {
    const uint32_t nbytes = (uint32_t)(r_hi - r_lo + 1) * row_bytes;
    if (threadIdx.x == 0) {
      mbar_expect_tx(&bar, nbytes);
      bulk_g2s(smem, src + (size_t)r_lo * row_bytes, nbytes, &bar);
    }
    mbar_wait(&bar, 0);
    const int cpr = row_bytes >> 4;                      // 16-byte chunks per row
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(smem);
    for (int q = threadIdx.x; q < rows * cpr; q += blockDim.x) {
      const int yl = q / cpr, j = q - yl * cpr;
      const int r = min(max(y0 + yl + dy, 0), H - 1) - r_lo;
      const int b0 = j * 16;
      const int a0 = b0 + sh;                            // first source byte if no clamping
      uint4 v;
      if (a0 >= 0 && a0 + 16 <= row_bytes) {
        const int base = r * row_bytes + a0;
        const int wi = base >> 2, bs = (base & 3) * 8;
        uint32_t w0 = s32[wi], w1 = s32[wi + 1], w2 = s32[wi + 2], w3 = s32[wi + 3], w4 = s32[wi + 4];
        v.x = __funnelshift_r(w0, w1, bs); v.y = __funnelshift_r(w1, w2, bs);
        v.z = __funnelshift_r(w2, w3, bs); v.w = __funnelshift_r(w3, w4, bs);
      } else {
        uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
        for (int b = 0; b < 16; ++b) {
          const int ob = b0 + b;
          const int x = ob / C, ch = ob - x * C;
          const int xs = min(max(x + cx - a.padding, 0), W - 1);
          o[b >> 2] |= (uint32_t)smem[r * row_bytes + xs * C + ch] << ((b & 3) * 8);
        }
        v = make_uint4(o[0], o[1], o[2], o[3]);
      }
      asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst + (size_t)yl * row_bytes + b0),
                   "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    }
  } else {
    for (int q = threadIdx.x; q < rows * row_bytes; q += blockDim.x) {
      const int yl = q / row_bytes, ob = q - yl * row_bytes;
      const int r = min(max(y0 + yl + dy, 0), H - 1);
      const int x = ob / C, ch = ob - x * C;
      const int xs = min(max(x + cx - a.padding, 0), W - 1);
      if constexpr (kStacked) dst[(size_t)yl * row_bytes * T + (x * T + t) * C + ch] = src[(size_t)r * row_bytes + xs * C + ch];
      else dst[(size_t)yl * row_bytes + ob] = src[(size_t)r * row_bytes + xs * C + ch];
    }
  }
}

template <bool kFast>
__global__ void __launch_bounds__(kSamplerThreads) sample_gather_crop_kernel(const SamplerArgs a) {
  sample_gather_crop_body<kFast, false, false>(a, nullptr);
}
template <bool kFast>
__global__ void __launch_bounds__(kSamplerThreads) sample_gather_crop_nstep_kernel(const SamplerArgs a) {
  sample_gather_crop_body<kFast, true, false>(a, nullptr);
}
template <bool kFast, bool kNStep>
__global__ void __launch_bounds__(kSamplerThreads) sample_gather_crop_prio_kernel(const SamplerArgs a, __grid_constant__ const PrioDraw pd) {
  sample_gather_crop_body<kFast, kNStep, false, true>(a, nullptr, &pd);
}
template <bool kFast, bool kNStep>
__global__ void __launch_bounds__(kSamplerThreads) sample_gather_crop_sharded_kernel(const SamplerArgs a,
                                                                                     __grid_constant__ const serl_replay_shards sh) {
  sample_gather_crop_body<kFast, kNStep, true>(a, &sh);
}

// ---------------------------------------------------------------------------------------------
// Fast path (row_bytes % 16 == 0): ONE CTA per (row, camera, obs|next) streams its whole frame(s).
// The serial preamble runs once per frame instead of once per band and is spread over two warps (warp 0: Philox index
// draw; warp 1: the threefry crop-key chain, two lanes wide, three evaluations deep); the 32-row bands of a frame are then
// all fetched at once (one TMA bulk copy + mbarrier per band, 48 KiB of shared memory per CTA) and shifted / written back
// in arrival order, so a CTA pays one memory round trip per frame instead of one per band.
// ---------------------------------------------------------------------------------------------
constexpr int kFrameThreads = 256;
constexpr int kMaxBands = 8;             // frames up to 256 rows

// crop offsets for frame g, computed cooperatively by lanes 0/1 of a full warp (all 32 lanes must call)
__device__ inline void crop_offset_warp(const uint32_t* key, const int32_t* expl, int crop_total, int g, int span, int lane,
                                        int* cy, int* cx) {
  if (expl) { *cy = expl[2 * g]; *cx = expl[2 * g + 1]; return; }
  const uint32_t n = (uint32_t)crop_total;
  // level 1: key_g = split(key, n)[g] = (flat[2g], flat[2g+1])
  const uint32_t pos = 2u * (uint32_t)g + (uint32_t)(lane & 1);
  const uint32_t j = pos < n ? pos : pos - n;
  const u32x2 y1 = threefry2x32(u32x2{key[0], key[1]}, j, n + j);
  const uint32_t f = pos < n ? y1.x : y1.y;
  const u32x2 k{__shfl_sync(0xffffffffu, f, 0), __shfl_sync(0xffffffffu, f, 1)};
  // level 2: k1, k2 = split(key_g, 2): flat = [a0, a1, b0, b1] with (a_j, b_j) = TF(key_g, j, 2 + j)
  const u32x2 y2 = threefry2x32(k, (uint32_t)(lane & 1), 2u + (uint32_t)(lane & 1));
  const uint32_t a0 = __shfl_sync(0xffffffffu, y2.x, 0), a1 = __shfl_sync(0xffffffffu, y2.x, 1);
  const uint32_t b0 = __shfl_sync(0xffffffffu, y2.y, 0), b1 = __shfl_sync(0xffffffffu, y2.y, 1);
  // level 3: higher bits = random_bits(k1, (2,)), lower bits = random_bits(k2, (2,))
  const u32x2 y3 = threefry2x32((lane & 1) ? u32x2{b0, b1} : u32x2{a0, a1}, 0u, 1u);
  const uint32_t hb0 = __shfl_sync(0xffffffffu, y3.x, 0), hb1 = __shfl_sync(0xffffffffu, y3.y, 0);
  const uint32_t lb0 = __shfl_sync(0xffffffffu, y3.x, 1), lb1 = __shfl_sync(0xffffffffu, y3.y, 1);
  const uint32_t sp = (uint32_t)span;
  uint32_t mult = 65536u % sp; mult = (mult * mult) % sp;
  *cy = (int)(((hb0 % sp) * mult + (lb0 % sp)) % sp);
  *cx = (int)(((hb1 % sp) * mult + (lb1 % sp)) % sp);
}

// The frame part of sample_frames_body<..., kStacked = true>: output row out_row of (B_total, H, W, T*C) from the window that ends
// at slot widx, frame t shifted by (cy[t], cx[t]).  Per band: thread 0 issues the T frames' source rows (one bulk copy each,
// band_bytes apart in smem) on one mbarrier; each thread then assembles 16 output bytes (pixel x, frame t, channel c in
// order) from the staged rows and stores them with one 128-bit store.
template <bool kShard>
__device__ __forceinline__ void sample_frames_stacked_rows(const SamplerArgs& a, const serl_replay_shards* shards, uint8_t* smem,
                                                           uint64_t* bar, int widx, int which, int cam, int out_row, int band_bytes,
                                                           const int* cy, const int* cx) {
  const serl_replay_view& rv = a.rv;
  const int T = rv.num_stack, H = rv.height, W = rv.width, C = rv.channels;
  const int row_bytes = W * C, TC = T * C, cpo = (W * TC) >> 4;
  const size_t frame_bytes = (size_t)H * row_bytes;
  const int w0 = widx - T + ((widx - T) < 0 ? rv.capacity - T : 0);      // negative window index: numpy semantics (see above)
  uint8_t* out = (which ? a.next_pix[cam] : a.obs_pix[cam]) + (size_t)out_row * H * W * TC;
  const int nb = ceil_div(H, kBandRows);
  for (int band = 0; band < nb; ++band) {
    const int y0 = band * kBandRows, rows = min(kBandRows, H - y0);
    if (threadIdx.x == 0) {
      uint32_t total = 0;
      for (int t = 0; t < T; ++t) {
        const int dy = cy[t] - a.padding;
        total += (uint32_t)(min(max(y0 + rows - 1 + dy, 0), H - 1) - min(max(y0 + dy, 0), H - 1) + 1) * row_bytes;
      }
      mbar_expect_tx(bar, total);
      for (int t = 0; t < T; ++t) {
        const int dy = cy[t] - a.padding;
        const int r_lo = min(max(y0 + dy, 0), H - 1), r_hi = min(max(y0 + rows - 1 + dy, 0), H - 1);
        const uint8_t* fsrc = window_frame<kShard>(rv, shards, cam, w0, w0 + t + which, frame_bytes);
        bulk_g2s(smem + t * band_bytes, fsrc + (size_t)r_lo * row_bytes, (uint32_t)(r_hi - r_lo + 1) * row_bytes, bar);
      }
    }
    mbar_wait(bar, (uint32_t)band & 1u);
    for (int q = threadIdx.x; q < rows * cpo; q += blockDim.x) {
      const int yl = q / cpo, b0 = (q - yl * cpo) * 16;
      int x = b0 / TC, t = (b0 - x * TC) / C, c = b0 - x * TC - t * C;
      // staged source row of frame t for output row y0 + yl, and its byte at output pixel x
      auto src_px = [&](int t, int x) {
        const int dy = cy[t] - a.padding;
        const int r = min(max(y0 + yl + dy, 0), H - 1) - min(max(y0 + dy, 0), H - 1);
        return smem + t * band_bytes + r * row_bytes + min(max(x + cx[t] - a.padding, 0), W - 1) * C;
      };
      const uint8_t* sp = src_px(t, x);
      uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
      for (int b = 0; b < 16; ++b) {
        o[b >> 2] |= (uint32_t)sp[c] << ((b & 3) * 8);
        if (++c == C) {
          c = 0;
          if (++t == T) { t = 0; ++x; }
          if (b < 15) sp = src_px(t, x);
        }
      }
      asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(out + ((size_t)(y0 + yl) * W * TC + b0)),
                   "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
    }
    __syncthreads();                                       // the staged bands are free again for the next band
  }
}

// grid: x = cam*2 + which, y = row i.  kStacked: the outputs are (B_total, H, W, T*C) (serl_batch_out.stacked); the CTA then
// stages one 32-row band of all T frames at a time (T bulk copies on one mbarrier) and composes each output row's 16-byte
// chunks from the T staged bands, since every output chunk interleaves the bytes of several frames.
template <bool kNStep, bool kShard, bool kPrio = false, bool kStacked = false>
__device__ __forceinline__ void sample_frames_body(const SamplerArgs& a, const serl_replay_shards* shards, const PrioDraw* pd = nullptr) {
  pdl_prologue();
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar[kMaxBands];
  __shared__ int s_idx, s_nidx, s_m, s_cy[8], s_cx[8];

  const serl_replay_view& rv = a.rv;
  const int T = rv.num_stack, H = rv.height, W = rv.width, C = rv.channels;
  const int row_bytes = W * C;
  const int which = blockIdx.x & 1, cam = blockIdx.x >> 1;
  const int i = blockIdx.y;
  const int out_row = a.out_row_offset + i;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool leader = (cam == 0 && which == 0);
  const int band_bytes = kBandRows * row_bytes + 32;

  if (threadIdx.x == 0) {
    const int idx = draw_row<kPrio>(a, pd, i);
    s_idx = idx;
    if (idx < 0) atomicOr(a.status, 1);
    if constexpr (kNStep) { if (idx >= 0 && (which || leader)) s_nidx = nstep_window(a, idx, &s_m); }
    for (int b = 0; b < kMaxBands; ++b) mbar_init(&bar[b], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == 1) {
    for (int t = 0; t < T; ++t) {
      const int g = out_row * T + t;
      int cy, cx;
      crop_offset_warp(which ? a.key_next : a.key_obs, which ? a.explicit_off_next : a.explicit_off_obs, a.crop_total, g,
                       2 * a.padding + 1, lane, &cy, &cx);
      if (lane == 0) {
        s_cy[t] = cy; s_cx[t] = cx;
        if (cam == 0) { int32_t* o = which ? a.off_next_out : a.off_obs_out; if (o) { o[2 * g] = cy; o[2 * g + 1] = cx; } }
      }
    }
  }
  __syncthreads();
  const int idx = s_idx;
  if (idx < 0) return;
  const int nidx = kNStep && (which || leader) ? s_nidx : idx;   // slot whose next observation the row carries

  if (leader) {                                            // small fields: one CTA per row
    const int ns = T * rv.state_dim;
    for (int k = threadIdx.x; k < ns; k += blockDim.x) {
      a.obs_state[(size_t)out_row * ns + k] = rv.state[(size_t)idx * ns + k];
      a.next_state[(size_t)out_row * ns + k] = rv.next_state[(size_t)nidx * ns + k];
    }
    for (int k = threadIdx.x; k < rv.action_dim; k += blockDim.x)
      a.actions[(size_t)out_row * rv.action_dim + k] = rv.actions[(size_t)idx * rv.action_dim + k];
    if (threadIdx.x == 0) {
      if constexpr (kNStep) nstep_scalars(a, idx, nidx, s_m, out_row);
      else { a.rewards[out_row] = rv.rewards[idx]; a.masks[out_row] = rv.masks[idx]; a.dones[out_row] = rv.dones[idx]; }
      if (a.idx_out) a.idx_out[out_row] = idx;
      if constexpr (kPrio) { if (pd->prio_out) pd->prio_out[out_row] = pd->tree[idx]; }
    }
  }

  if constexpr (kStacked) {
    sample_frames_stacked_rows<kShard>(a, shards, smem, &bar[0], which ? nidx : idx, which, cam, out_row, band_bytes, s_cy, s_cx);
    return;
  }
  const size_t frame_bytes = (size_t)H * row_bytes;
  const int nb = ceil_div(H, kBandRows);                   // <= kMaxBands, all in flight at once
  const int cpr = row_bytes >> 4;
  for (int t = 0; t < T; ++t) {
    const int cy = s_cy[t], cx = s_cx[t];
    const int dy = cy - a.padding, sh = (cx - a.padding) * C;
    if (threadIdx.x == 0) {                                // one TMA bulk copy per band, each with its own mbarrier
      const int widx = which ? nidx : idx;
      const int w0 = widx - T + ((widx - T) < 0 ? rv.capacity - T : 0);              // negative window index: numpy semantics (see sample_gather_crop_kernel)
      const uint8_t* fsrc = window_frame<kShard>(rv, shards, cam, w0, w0 + t + which, frame_bytes);
      for (int band = 0; band < nb; ++band) {
        const int y0 = band * kBandRows, rows = min(kBandRows, H - y0);
        const int r_lo = min(max(y0 + dy, 0), H - 1), r_hi = min(max(y0 + rows - 1 + dy, 0), H - 1);
        const uint32_t nbytes = (uint32_t)(r_hi - r_lo + 1) * row_bytes;
        mbar_expect_tx(&bar[band], nbytes);
        bulk_g2s(smem + band * band_bytes, fsrc + (size_t)r_lo * row_bytes, nbytes, &bar[band]);
      }
    }
    const int g = out_row * T + t;
    for (int band = 0; band < nb; ++band) {
      mbar_wait(&bar[band], (uint32_t)t & 1u);
      const int y0 = band * kBandRows, rows = min(kBandRows, H - y0);
      const int r_lo = min(max(y0 + dy, 0), H - 1);
      const uint8_t* sb = smem + band * band_bytes;
      uint8_t* dst = (which ? a.next_pix[cam] : a.obs_pix[cam]) + ((size_t)g * H + y0) * row_bytes;
      // interior chunks: a row-shifted copy with ONE aligned 128-bit shared load per lane.  A warp takes whole rows; lane l
      // loads the aligned 16-byte chunk (l + kq) of the source row (conflict-free: consecutive lanes, consecutive chunks),
      // gets the next chunk from lane l+1 by shuffle, and funnels the two by the byte shift (uniform per frame).  Round 1
      // read five 32-bit words per lane at a 16-byte lane stride: 4-way bank conflicts on 85 % of the shared wavefronts
      // (profiles/r01_ncu_sampler_stem_full.md).  The <= 1 chunk per row that touches the clamped edge is handled by the
      // compact bytewise loop below.
      {
        const int kqg = (sh >= 0) ? (sh >> 4) : -((-sh + 15) >> 4);   // floor(sh / 16)
        const int bsh = sh - 16 * kqg;                         // 0..15
        const int wsft = bsh >> 2, bits = (bsh & 3) * 8;
        const uint4* s128 = reinterpret_cast<const uint4*>(sb);
        const int cpr4 = row_bytes >> 4;
        for (int yl = warp; yl < rows; yl += (kFrameThreads >> 5)) {
          const int r = min(max(y0 + yl + dy, 0), H - 1) - r_lo;
          for (int j0 = 0; j0 < cpr; j0 += 31) {              // 31 output chunks per pass (lane 31 only supplies its neighbour)
            const int jj = j0 + lane, c = jj + kqg;
            uint4 A = make_uint4(0u, 0u, 0u, 0u);
            if (c >= 0 && c < cpr4) A = s128[r * cpr4 + c];
            uint4 Bn;
            Bn.x = __shfl_down_sync(0xffffffffu, A.x, 1); Bn.y = __shfl_down_sync(0xffffffffu, A.y, 1);
            Bn.z = __shfl_down_sync(0xffffffffu, A.z, 1); Bn.w = __shfl_down_sync(0xffffffffu, A.w, 1);
            const int a0 = jj * 16 + sh;
            if (lane < 31 && jj < cpr && a0 >= 0 && a0 + 16 <= row_bytes) {
              uint32_t w0, w1, w2, w3, w4;                     // the five words starting at word offset wsft of (A, Bn)
              switch (wsft) {
                case 0: w0 = A.x; w1 = A.y; w2 = A.z; w3 = A.w; w4 = Bn.x; break;
                case 1: w0 = A.y; w1 = A.z; w2 = A.w; w3 = Bn.x; w4 = Bn.y; break;
                case 2: w0 = A.z; w1 = A.w; w2 = Bn.x; w3 = Bn.y; w4 = Bn.z; break;
                default: w0 = A.w; w1 = Bn.x; w2 = Bn.y; w3 = Bn.z; w4 = Bn.w; break;
              }
              asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst + (size_t)yl * row_bytes + jj * 16),
                           "r"(__funnelshift_r(w0, w1, bits)), "r"(__funnelshift_r(w1, w2, bits)), "r"(__funnelshift_r(w2, w3, bits)),
                           "r"(__funnelshift_r(w3, w4, bits)) : "memory");
            }
          }
        }
      }
      const int ne_l = sh < 0 ? min(cpr, (-sh + 15) >> 4) : 0, ne_r = sh > 0 ? min(cpr - ne_l, (sh + 15) >> 4) : 0;
      const int ne = ne_l + ne_r;
      for (int e = threadIdx.x; e < rows * ne; e += blockDim.x) {
        const int yl = e / ne, k = e - yl * ne;
        const int jj = k < ne_l ? k : cpr - ne_r + (k - ne_l);
        const int r = min(max(y0 + yl + dy, 0), H - 1) - r_lo;
        const int b0 = jj * 16;
        uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
        for (int b = 0; b < 16; ++b) {
          const int ob = b0 + b;
          const int x = (C == 3 && ob < 65536) ? (int)(((uint32_t)ob * 43691u) >> 17) : ob / C;
          const int ch = ob - x * C;
          const int xs = min(max(x + cx - a.padding, 0), W - 1);
          o[b >> 2] |= (uint32_t)sb[r * row_bytes + xs * C + ch] << ((b & 3) * 8);
        }
        asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst + (size_t)yl * row_bytes + b0),
                     "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
      }
    }
    __syncthreads();                                       // every band buffer is free again for the next stacked frame
  }
}

__global__ void __launch_bounds__(kFrameThreads) sample_frames_kernel(const SamplerArgs a) { sample_frames_body<false, false>(a, nullptr); }
__global__ void __launch_bounds__(kFrameThreads) sample_frames_nstep_kernel(const SamplerArgs a) { sample_frames_body<true, false>(a, nullptr); }
template <bool kNStep>
__global__ void __launch_bounds__(kFrameThreads) sample_frames_prio_kernel(const SamplerArgs a, __grid_constant__ const PrioDraw pd) {
  sample_frames_body<kNStep, false, true>(a, nullptr, &pd);
}
template <bool kNStep>
__global__ void __launch_bounds__(kFrameThreads) sample_frames_sharded_kernel(const SamplerArgs a, __grid_constant__ const serl_replay_shards sh) {
  sample_frames_body<kNStep, true>(a, &sh);
}

// Channel-stacked outputs (serl_batch_out.stacked, T > 1): every (kNStep, kShard, kPrio) variant takes both the shard table and
// the prioritized draw; each reads only its own.
template <bool kNStep, bool kShard, bool kPrio>
__global__ void __launch_bounds__(kFrameThreads) sample_frames_stacked_kernel(const SamplerArgs a, __grid_constant__ const serl_replay_shards sh,
                                                                              __grid_constant__ const PrioDraw pd) {
  sample_frames_body<kNStep, kShard, kPrio, true>(a, &sh, &pd);
}
template <bool kNStep, bool kShard, bool kPrio>
__global__ void __launch_bounds__(kSamplerThreads) sample_gather_crop_stacked_kernel(const SamplerArgs a, __grid_constant__ const serl_replay_shards sh,
                                                                                    __grid_constant__ const PrioDraw pd) {
  sample_gather_crop_body<false, kNStep, kShard, kPrio, true>(a, &sh, &pd);
}

// ---------------------------------------------------------------------------------------------
// Replay ring writes (insert path).  The ring bookkeeping (cursor, episode-start fillers, validity)
// is host logic mirroring data/memory_efficient_replay_buffer.py:53-89; these kernels apply a batch
// of slot writes staged in device memory.
// ---------------------------------------------------------------------------------------------
struct ScatterArgs {
  serl_replay_view rv;           // frames etc. are written (const_cast on the device side)
  int n;                         // slot writes
  const int32_t* dst_slot;       // (n)
  const int32_t* src_slot;       // (n) >= 0: copy from ring slot; < 0: from staging row k
  const uint8_t* st_frames[SERL_MAX_CAMS];   // (n, frame_bytes)
  const float* st_state; const float* st_next_state; const float* st_actions;
  const float* st_rewards; const float* st_masks; const uint8_t* st_dones; const uint8_t* st_valid;
  long long row_stride;          // 0: every staging field is a packed (n, ...) array; else: byte distance between rows k, k+1
};

// staging row k of a field: packed arrays, or fields interleaved in one record per row (one H2D copy per flush)
template <class T>
__device__ inline const T* st_row(const T* base, int k, size_t packed_elems, long long stride) {
  return stride ? reinterpret_cast<const T*>(reinterpret_cast<const uint8_t*>(base) + (size_t)k * (size_t)stride) : base + (size_t)k * packed_elems;
}

// grid: x = chunk of the frame, y = cam, z = write k.  Ordered writes: launch once per dependency level.
__global__ void __launch_bounds__(256) replay_scatter_kernel(const ScatterArgs a) {
  pdl_prologue();
  const serl_replay_view& rv = a.rv;
  const int k = blockIdx.z, cam = blockIdx.y;
  const int dst = *st_row(a.dst_slot, k, 1, a.row_stride), ss = *st_row(a.src_slot, k, 1, a.row_stride);
  const size_t fb = (size_t)rv.height * rv.width * rv.channels;
  if (cam < rv.num_cams) {
    const uint8_t* s = ss >= 0 ? rv.frames[cam] + (size_t)ss * fb : st_row(a.st_frames[cam], k, fb, a.row_stride);
    uint8_t* d = const_cast<uint8_t*>(rv.frames[cam]) + (size_t)dst * fb;
    if ((fb & 15) == 0 && ((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15) == 0) {
      const uint4* s4 = reinterpret_cast<const uint4*>(s);
      uint4* d4 = reinterpret_cast<uint4*>(d);
      for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < (fb >> 4); q += (size_t)gridDim.x * blockDim.x)
        d4[q] = s4[q];
    } else {
      for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < fb; q += (size_t)gridDim.x * blockDim.x)
        d[q] = s[q];
    }
  }
  if (cam == 0 && blockIdx.x == 0) {
    const int ns = rv.num_stack * rv.state_dim;
    float* st = const_cast<float*>(rv.state); float* nst = const_cast<float*>(rv.next_state);
    float* ac = const_cast<float*>(rv.actions);
    const float* s_st = st_row(a.st_state, k, ns, a.row_stride); const float* s_nst = st_row(a.st_next_state, k, ns, a.row_stride);
    const float* s_ac = st_row(a.st_actions, k, rv.action_dim, a.row_stride);
    for (int e = threadIdx.x; e < ns; e += blockDim.x) {
      st[(size_t)dst * ns + e] = ss >= 0 ? rv.state[(size_t)ss * ns + e] : s_st[e];
      nst[(size_t)dst * ns + e] = ss >= 0 ? rv.next_state[(size_t)ss * ns + e] : s_nst[e];
    }
    for (int e = threadIdx.x; e < rv.action_dim; e += blockDim.x)
      ac[(size_t)dst * rv.action_dim + e] = ss >= 0 ? rv.actions[(size_t)ss * rv.action_dim + e] : s_ac[e];
    if (threadIdx.x == 0) {
      const_cast<float*>(rv.rewards)[dst] = ss >= 0 ? rv.rewards[ss] : *st_row(a.st_rewards, k, 1, a.row_stride);
      const_cast<float*>(rv.masks)[dst] = ss >= 0 ? rv.masks[ss] : *st_row(a.st_masks, k, 1, a.row_stride);
      const_cast<uint8_t*>(rv.dones)[dst] = ss >= 0 ? rv.dones[ss] : *st_row(a.st_dones, k, 1, a.row_stride);
      const_cast<uint8_t*>(rv.valid)[dst] = *st_row(a.st_valid, k, 1, a.row_stride);
    }
  }
}

// Where rank sh.rank stores slot s (serl_replay_shards): *range = s - lo + halo when lo <= s < hi, *halo = halo - d when
// d = (lo - s) mod capacity is in 1 .. halo; -1 where it does not.  Both apply at world 1 (the halo wraps into the range).
__device__ inline void shard_locals(const serl_replay_shards& sh, int cap, int s, int* range, int* halo) {
  const int lo = sh.rank * sh.slots_per_rank, hi = min(cap, lo + sh.slots_per_rank);
  const int d = ((lo - s) % cap + cap) % cap;
  *range = (s >= lo && s < hi) ? s - lo + sh.halo : -1;
  *halo = (d >= 1 && d <= sh.halo) ? sh.halo - d : -1;
}

__device__ inline void copy_frame(uint8_t* d, const uint8_t* s, size_t fb) {
  if ((fb & 15) == 0 && ((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15) == 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(s);
    uint4* d4 = reinterpret_cast<uint4*>(d);
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < (fb >> 4); q += (size_t)gridDim.x * blockDim.x)
      d4[q] = s4[q];
  } else {
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < fb; q += (size_t)gridDim.x * blockDim.x)
      d[q] = s[q];
  }
}

// Frames of the slot writes, into rank sh.rank's allocation only (the small fields go through replay_scatter_kernel on a
// camera-less view).  A copied slot's source frame is stored on every rank that stores its target (the re-insert at the front
// copies slots capacity - T .. capacity - 1, which rank 0 holds as its wrapped halo).  grid as replay_scatter_kernel.
__global__ void __launch_bounds__(256) replay_scatter_frames_sharded_kernel(const ScatterArgs a, __grid_constant__ const serl_replay_shards sh) {
  pdl_prologue();
  const serl_replay_view& rv = a.rv;
  const int k = blockIdx.z, cam = blockIdx.y;
  const int dst = *st_row(a.dst_slot, k, 1, a.row_stride), ss = *st_row(a.src_slot, k, 1, a.row_stride);
  const size_t fb = (size_t)rv.height * rv.width * rv.channels;
  int dr, dh;
  shard_locals(sh, rv.capacity, dst, &dr, &dh);
  if (dr < 0 && dh < 0) return;
  uint8_t* base = const_cast<uint8_t*>(sh.frames[cam][sh.rank]);
  const uint8_t* s = st_row(a.st_frames[cam], k, fb, a.row_stride);
  if (ss >= 0) {
    int sr, sl;
    shard_locals(sh, rv.capacity, ss, &sr, &sl);
    s = base + (size_t)(sr >= 0 ? sr : sl) * fb;
  }
  if (dr >= 0) copy_frame(base + (size_t)dr * fb, s, fb);
  if (dh >= 0) copy_frame(base + (size_t)dh * fb, s, fb);
}

__global__ void counter_add_kernel(uint64_t* ctr, uint64_t inc) {
  pdl_prologue(); if (threadIdx.x == 0 && blockIdx.x == 0) *ctr += inc; }

__global__ void replay_set_valid_kernel(uint8_t* valid, const int32_t* slots, const uint8_t* vals, int n, int32_t* size_dev, int32_t size) {
  pdl_prologue();
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) valid[slots[k]] = vals[k];
  if (k == 0 && size_dev) *size_dev = size;
}

// ---------------------------------------------------------------------------------------------
// Prioritized replay: the sum tree's writers (layout and semantics in include/serl_b200.h).
// ---------------------------------------------------------------------------------------------
constexpr int kPrioThreads = 1024;

struct PrioSetArgs {
  float* tree; float* max_dev; const uint8_t* ring_valid;
  int capacity, levels; int off[SERL_MAX_TREE_LEVELS];
  const int32_t* slots; const float* td; const uint8_t* valid;
  int n; float alpha, eps;
};

// node j of level l (>= 1) from its children, in ascending order
__device__ inline void prio_recompute(float* tree, const int* off, int l, int j) {
  const float* ch = tree + off[l - 1];
  const int c1 = min(SERL_PRIO_FANOUT * j + SERL_PRIO_FANOUT, off[l] - off[l - 1]);
  float s = 0.f;
  for (int c = SERL_PRIO_FANOUT * j; c < c1; ++c) s = __fadd_rn(s, ch[c]);
  tree[off[l] + j] = s;
}

// ONE CTA.  Last entry wins without atomics: entry k writes its leaf only when no later entry names the same slot.  Then
// level by level every written leaf's ancestor is recomputed from its children (entries sharing an ancestor recompute it
// to the same value).  __syncthreads orders each level's reads after the writes below it.
__global__ void __launch_bounds__(kPrioThreads) priority_set_kernel(const PrioSetArgs a) {
  pdl_prologue();
  __shared__ int s_slot[SERL_PRIO_SET_MAX];
  __shared__ float s_max[kPrioThreads / 32];
  const float m0 = *a.max_dev;
  for (int k = threadIdx.x; k < a.n; k += blockDim.x) s_slot[k] = a.slots[k];
  __syncthreads();
  float mx = 0.f;
  for (int k = threadIdx.x; k < a.n; k += blockDim.x) {
    const int slot = s_slot[k];
    if (slot < 0 || slot >= a.capacity) continue;
    bool last = true;
    for (int q = k + 1; q < a.n && last; ++q) last = s_slot[q] != slot || (a.td && !isfinite(a.td[q]));   // skipped entries do not count
    if (!last) continue;
    float p;
    if (a.td) {
      const float td = a.td[k];
      if (!isfinite(td)) continue;                       // a non-finite TD error would poison every ancestor up to the root
      p = (a.ring_valid && !a.ring_valid[slot]) ? 0.f : powf(__fadd_rn(fabsf(td), a.eps), a.alpha);
    } else {
      p = a.valid[k] ? m0 : 0.f;
    }
    a.tree[slot] = p;
    mx = fmaxf(mx, p);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0 && a.td) {
    float m = m0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, s_max[w]);
    *a.max_dev = m;
  }
  for (int l = 1; l < a.levels; ++l) {
    for (int k = threadIdx.x; k < a.n; k += blockDim.x)
      if (s_slot[k] >= 0 && s_slot[k] < a.capacity) prio_recompute(a.tree, a.off, l, s_slot[k] >> (5 * l));
    __syncthreads();
  }
}

// every node of level l from level l - 1 (one launch per level)
__global__ void priority_rebuild_kernel(const PrioSetArgs a, int l, int count) {
  pdl_prologue();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < count) prio_recompute(a.tree, a.off, l, j);
}

// ONE CTA: p_min over the part's rows with p > 0, then w = (p_min / p)^beta (0 for a row of priority 0)
__global__ void __launch_bounds__(kPrioThreads) priority_weights_kernel(const float* prio, int n, const float* beta_dev, float* w) {
  pdl_prologue();
  __shared__ float s_min[kPrioThreads / 32];
  float mn = INFINITY;
  for (int k = threadIdx.x; k < n; k += blockDim.x) if (prio[k] > 0.f) mn = fminf(mn, prio[k]);
  for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if ((threadIdx.x & 31) == 0) s_min[threadIdx.x >> 5] = mn;
  __syncthreads();
  mn = s_min[0];
  for (int q = 1; q < (int)(blockDim.x >> 5); ++q) mn = fminf(mn, s_min[q]);
  const float beta = *beta_dev;
  for (int k = threadIdx.x; k < n; k += blockDim.x) w[k] = prio[k] > 0.f ? powf(__fdiv_rn(mn, prio[k]), beta) : 0.f;
}

}  // namespace serl

using namespace serl;

static int check_view(const serl_replay_view* rv) {
  if (!rv || rv->num_cams < 0 || rv->num_cams > SERL_MAX_CAMS || rv->num_stack < 1 || rv->size < 0 ||
      rv->size > rv->capacity || rv->height < 1 || rv->width < 1 || rv->channels < 1) {
    set_last_error("serl_replay: invalid replay view");
    return SERL_ERR_INVALID;
  }
  return SERL_OK;
}

static int check_request(const serl_replay_view* rv, const serl_sample_request* rq, const serl_batch_out* out, const char* fn) {
  if (!rq || !out || rq->batch < 1 || rq->crop_total < (rq->out_row_offset + rq->batch) * rv->num_stack) {
    set_last_error("%s: invalid request (batch=%d crop_total=%d)", fn, rq ? rq->batch : -1, rq ? rq->crop_total : -1);
    return SERL_ERR_INVALID;
  }
  if (!rq->explicit_idx && rv->size <= rv->num_stack) {
    set_last_error("%s: buffer holds %d slots, need > num_stack", fn, rv->size);
    return SERL_ERR_INVALID;
  }
  if (rv->num_cams > 0 && (!rq->key_obs || !rq->key_next) && (!rq->explicit_off_obs || !rq->explicit_off_next)) {
    set_last_error("%s: need crop keys or explicit offsets", fn);
    return SERL_ERR_INVALID;
  }
  return SERL_OK;
}

static SamplerArgs sampler_args(const serl_replay_view* rv, const serl_sample_request* rq, const serl_batch_out* out) {
  SamplerArgs a{};
  a.rv = *rv;
  a.seed = rq->seed; a.step = rq->step; a.step_dev = rq->step_dev; a.size_dev = rq->size_dev; a.lane_offset = rq->lane_offset; a.explicit_idx = rq->explicit_idx;
  a.key_obs = rq->key_obs; a.key_next = rq->key_next;
  a.explicit_off_obs = rq->explicit_off_obs; a.explicit_off_next = rq->explicit_off_next;
  a.crop_total = rq->crop_total; a.out_row_offset = rq->out_row_offset; a.padding = rq->padding;
  for (int c = 0; c < rv->num_cams; ++c) { a.obs_pix[c] = out->obs_pix[c]; a.next_pix[c] = out->next_pix[c]; }
  a.obs_state = out->obs_state; a.next_state = out->next_state; a.actions = out->actions;
  a.rewards = out->rewards; a.masks = out->masks; a.dones = out->dones; a.idx_out = out->idx;
  a.off_obs_out = out->off_obs; a.off_next_out = out->off_next; a.status = out->status; a.batch = rq->batch;
  return a;
}

// The sampler kernels of one (kNStep, kShard, kPrio) triple; the sharded kernels take the shard table as their last parameter.
// Prioritized draws run on unsharded rings only.
template <bool kNStep, bool kShard, bool kPrio = false> struct SamplerKernels;
template <bool kNStep> struct SamplerKernels<kNStep, false, true> {
  static constexpr auto frames = sample_frames_prio_kernel<kNStep>;
  static constexpr auto banded = sample_gather_crop_prio_kernel<true, kNStep>;
  static constexpr auto bytewise = sample_gather_crop_prio_kernel<false, kNStep>;
  static constexpr const char* frames_n = kNStep ? "sample_frames_prio_kernel<true>" : "sample_frames_prio_kernel<false>";
  static constexpr const char* banded_n = kNStep ? "sample_gather_crop_prio_kernel<true, true>" : "sample_gather_crop_prio_kernel<true, false>";
  static constexpr const char* byte_n = kNStep ? "sample_gather_crop_prio_kernel<false, true>" : "sample_gather_crop_prio_kernel<false, false>";
};
template <bool kNStep> struct SamplerKernels<kNStep, false, false> {
  static constexpr auto frames = kNStep ? sample_frames_nstep_kernel : sample_frames_kernel;
  static constexpr auto banded = kNStep ? sample_gather_crop_nstep_kernel<true> : sample_gather_crop_kernel<true>;
  static constexpr auto bytewise = kNStep ? sample_gather_crop_nstep_kernel<false> : sample_gather_crop_kernel<false>;
  static constexpr const char* frames_n = kNStep ? "sample_frames_nstep_kernel" : "sample_frames_kernel";
  static constexpr const char* banded_n = kNStep ? "sample_gather_crop_nstep_kernel<true>" : "sample_gather_crop_kernel<true>";
  static constexpr const char* byte_n = kNStep ? "sample_gather_crop_nstep_kernel<false>" : "sample_gather_crop_kernel<false>";
};
template <bool kNStep> struct SamplerKernels<kNStep, true, false> {
  static constexpr auto frames = sample_frames_sharded_kernel<kNStep>;
  static constexpr auto banded = sample_gather_crop_sharded_kernel<true, kNStep>;
  static constexpr auto bytewise = sample_gather_crop_sharded_kernel<false, kNStep>;
  static constexpr const char* frames_n = kNStep ? "sample_frames_sharded_kernel<true>" : "sample_frames_sharded_kernel<false>";
  static constexpr const char* banded_n = kNStep ? "sample_gather_crop_sharded_kernel<true, true>" : "sample_gather_crop_sharded_kernel<true, false>";
  static constexpr const char* byte_n = kNStep ? "sample_gather_crop_sharded_kernel<false, true>" : "sample_gather_crop_sharded_kernel<false, false>";
};

template <bool kShard, bool kPrio = false, class K>
static void launch_sampler(K kern, dim3 grid, dim3 block, size_t smem, cudaStream_t st, const SamplerArgs& a,
                           const serl_replay_shards* sh, const PrioDraw* pd) {
  if constexpr (kShard) launch_k(kern, grid, block, smem, st, a, *sh);
  else if constexpr (kPrio) launch_k(kern, grid, block, smem, st, a, *pd);
  else launch_k(kern, grid, block, smem, st, a);
}

// Picks the kernel from the frame geometry (see the kernels above).  kNStep selects the n-step instantiations; kShard the ones
// that read frames through the shard table `sh`; kPrio the prioritized draw.  Function-local statics are per instantiation, so
// each kernel keeps its own shared-memory opt-in.
// Channel-stacked outputs (T > 1): one CTA per (row, camera, obs|next) when rows are 16-byte multiples and the T staged bands fit
// in shared memory, else the bytewise kernel.
template <bool kNStep, bool kShard, bool kPrio>
static int sample_stacked_launch(const serl_replay_view* rv, const serl_sample_request* rq, const SamplerArgs& a,
                                 const serl_replay_shards* sh, cudaStream_t st, const PrioDraw* pd) {
  const serl_replay_shards shv = sh ? *sh : serl_replay_shards{};
  const PrioDraw pdv = pd ? *pd : PrioDraw{};
  const int row_bytes = rv->width * rv->channels;
  const bool fast = (row_bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(rv->frames[0]) & 15) == 0);
  const size_t smem = (size_t)rv->num_stack * ((size_t)kBandRows * row_bytes + 32);
  static size_t optin = 0, static_smem = 0, configured = 0;
  auto frames_k = sample_frames_stacked_kernel<kNStep, kShard, kPrio>;
  if (fast && !optin) {
    int dev = 0, v = 0;
    cudaFuncAttributes fa{};
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaFuncGetAttributes(&fa, frames_k) != cudaSuccess)
      return check_launch("sample_frames_stacked_kernel");
    optin = (size_t)v; static_smem = fa.sharedSizeBytes;
  }
  if (fast && rv->num_stack <= 8 && smem + static_smem <= optin) {
    if (smem > configured) {
      if (cudaFuncSetAttribute(frames_k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return check_launch("cudaFuncSetAttribute(sample_frames_stacked)");
      configured = smem;
    }
    launch_k(frames_k, dim3(rv->num_cams * 2, rq->batch), kFrameThreads, smem, st, a, shv, pdv);
    return check_launch("sample_frames_stacked_kernel");
  }
  launch_k(sample_gather_crop_stacked_kernel<kNStep, kShard, kPrio>, dim3(ceil_div(rv->height, kBandRows), rv->num_cams * 2 * rv->num_stack, rq->batch),
           kSamplerThreads, 0, st, a, shv, pdv);
  return check_launch("sample_gather_crop_stacked_kernel");
}

template <bool kNStep, bool kShard, bool kPrio = false>
static int sample_crop_launch(const serl_replay_view* rv, const serl_sample_request* rq, const SamplerArgs& a,
                              const serl_replay_shards* sh, cudaStream_t st, const PrioDraw* pd = nullptr, bool stacked = false) {
  if (stacked && rv->num_stack > 1 && rv->num_cams > 0) return sample_stacked_launch<kNStep, kShard, kPrio>(rv, rq, a, sh, st, pd);
  using Ks = SamplerKernels<kNStep, kShard, kPrio>;
  auto frames_k = Ks::frames;
  auto banded_k = Ks::banded;
  auto byte_k = Ks::bytewise;
  const char* frames_n = Ks::frames_n;
  const char* banded_n = Ks::banded_n;
  const char* byte_n = Ks::byte_n;

  const int row_bytes = rv->width * rv->channels;
  const bool fast = rv->num_cams > 0 && (row_bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(rv->frames[0]) & 15) == 0);
  dim3 grid(ceil_div(rv->height, kBandRows), rv->num_cams * 2 * rv->num_stack, rq->batch);
  if (rv->num_cams == 0) grid = dim3(1, 1, rq->batch);
  if (fast && rv->num_stack <= 8 && ceil_div(rv->height, kBandRows) <= kMaxBands &&
      (size_t)ceil_div(rv->height, kBandRows) * ((size_t)kBandRows * row_bytes + 32) <= 96 * 1024) {
    const size_t smem = (size_t)ceil_div(rv->height, kBandRows) * ((size_t)kBandRows * row_bytes + 32);
    static size_t configured = 0;
    if (smem > configured) {
      if (cudaFuncSetAttribute(frames_k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return check_launch("cudaFuncSetAttribute(sample_frames)");
      configured = smem;
    }
    dim3 fgrid(rv->num_cams * 2, rq->batch);
    launch_sampler<kShard, kPrio>(frames_k, fgrid, kFrameThreads, smem, st, a, sh, pd);
    return check_launch(frames_n);
  } else if (fast) {
    // one CTA per 32-row band: the band's rows + 32 bytes of slack for the shift's fifth word, opted in past the 48 KiB
    // default (a 1536-byte row already needs more).  Rows too wide for the device's opt-in limit (W*C >~ 7,260 bytes on
    // sm_90) go to the bytewise kernel below.
    const size_t smem = (size_t)kBandRows * row_bytes + 32;
    static size_t optin = 0, static_smem = 0;
    if (!optin) {
      int dev = 0, v = 0;
      cudaFuncAttributes fa{};
      if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
          cudaFuncGetAttributes(&fa, banded_k) != cudaSuccess)
        return check_launch(banded_n);
      optin = (size_t)v; static_smem = fa.sharedSizeBytes;
    }
    if (smem + static_smem <= optin) {
      static size_t configured = 0;
      if (smem > configured) {
        if (cudaFuncSetAttribute(banded_k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return check_launch("cudaFuncSetAttribute(sample_gather_crop<true>)");
        configured = smem;
      }
      launch_sampler<kShard, kPrio>(banded_k, grid, kSamplerThreads, smem, st, a, sh, pd);
      return check_launch(banded_n);
    }
  }
  launch_sampler<kShard, kPrio>(byte_k, grid, kSamplerThreads, 0, st, a, sh, pd);
  return check_launch(byte_n);
}

extern "C" int serl_replay_sample_crop(const serl_replay_view* rv, const serl_sample_request* rq,
                                       const serl_batch_out* out, void* stream) {
  if (int e = check_view(rv)) return e;
  if (int e = check_request(rv, rq, out, "serl_replay_sample_crop")) return e;
  return sample_crop_launch<false, false>(rv, rq, sampler_args(rv, rq, out), nullptr, static_cast<cudaStream_t>(stream), nullptr, out->stacked);
}

static int check_nstep(const serl_nstep_desc* ns, const char* fn) {
  if (!ns || ns->n < 1 || ns->n > SERL_MAX_NSTEP || !ns->head_dev || !(ns->discount == ns->discount)) {
    set_last_error("%s: invalid n-step descriptor (n=%d, need 1..%d, a discount and head_dev)", fn, ns ? ns->n : -1, SERL_MAX_NSTEP);
    return SERL_ERR_INVALID;
  }
  return SERL_OK;
}

static void set_nstep(SamplerArgs& a, const serl_nstep_desc* ns) {
  a.n_step = ns->n; a.discount = ns->discount; a.head_dev = ns->head_dev; a.m_out = ns->m_out; a.next_idx_out = ns->next_idx_out;
}

extern "C" int serl_replay_sample_crop_nstep(const serl_replay_view* rv, const serl_sample_request* rq, const serl_nstep_desc* ns,
                                             const serl_batch_out* out, void* stream) {
  if (int e = check_view(rv)) return e;
  if (int e = check_request(rv, rq, out, "serl_replay_sample_crop_nstep")) return e;
  if (int e = check_nstep(ns, "serl_replay_sample_crop_nstep")) return e;
  SamplerArgs a = sampler_args(rv, rq, out);
  set_nstep(a, ns);
  return sample_crop_launch<true, false>(rv, rq, a, nullptr, static_cast<cudaStream_t>(stream), nullptr, out->stacked);
}

// A shard table the kernels can follow: every rank's range non-empty, every allocation present for every camera, and a
// halo of T slots (the window a row reads is w0 .. w0 + T).
static int check_shards(const serl_replay_view* rv, const serl_replay_shards* sh, const char* fn) {
  bool ok = sh && rv->num_cams > 0 && sh->world >= 1 && sh->world <= SERL_MAX_SHARD_RANKS && sh->rank >= 0 && sh->rank < sh->world &&
            sh->halo == rv->num_stack && sh->slots_per_rank == (rv->capacity + sh->world - 1) / sh->world &&
            (sh->world - 1) * sh->slots_per_rank < rv->capacity;
  for (int c = 0; ok && c < rv->num_cams; ++c)
    for (int r = 0; r < sh->world; ++r) ok = ok && sh->frames[c][r] != nullptr;
  if (!ok) {
    set_last_error("%s: invalid shard table (world=%d rank=%d slots_per_rank=%d halo=%d for capacity %d, T %d)", fn, sh ? sh->world : -1,
                   sh ? sh->rank : -1, sh ? sh->slots_per_rank : -1, sh ? sh->halo : -1, rv->capacity, rv->num_stack);
    return SERL_ERR_INVALID;
  }
  return SERL_OK;
}

extern "C" int serl_replay_sample_crop_sharded(const serl_replay_view* rv, const serl_replay_shards* sh, const serl_sample_request* rq,
                                               const serl_batch_out* out, void* stream) {
  if (int e = check_view(rv)) return e;
  if (int e = check_shards(rv, sh, "serl_replay_sample_crop_sharded")) return e;
  if (int e = check_request(rv, rq, out, "serl_replay_sample_crop_sharded")) return e;
  return sample_crop_launch<false, true>(rv, rq, sampler_args(rv, rq, out), sh, static_cast<cudaStream_t>(stream), nullptr, out->stacked);
}

extern "C" int serl_replay_sample_crop_nstep_sharded(const serl_replay_view* rv, const serl_replay_shards* sh, const serl_sample_request* rq,
                                                     const serl_nstep_desc* ns, const serl_batch_out* out, void* stream) {
  if (int e = check_view(rv)) return e;
  if (int e = check_shards(rv, sh, "serl_replay_sample_crop_nstep_sharded")) return e;
  if (int e = check_request(rv, rq, out, "serl_replay_sample_crop_nstep_sharded")) return e;
  if (int e = check_nstep(ns, "serl_replay_sample_crop_nstep_sharded")) return e;
  SamplerArgs a = sampler_args(rv, rq, out);
  set_nstep(a, ns);
  return sample_crop_launch<true, true>(rv, rq, a, sh, static_cast<cudaStream_t>(stream), nullptr, out->stacked);
}

static int check_tree(const serl_priority_tree* t, int capacity, const char* fn) {
  if (!t || !t->nodes || !t->max_dev || t->capacity < 1 || (capacity >= 0 && t->capacity != capacity)) {
    set_last_error("%s: invalid priority tree (capacity %d, ring capacity %d)", fn, t ? t->capacity : -1, capacity);
    return SERL_ERR_INVALID;
  }
  return SERL_OK;
}

extern "C" int serl_replay_sample_crop_prio(const serl_replay_view* rv, const serl_sample_request* rq, const serl_priority_tree* t,
                                            const serl_nstep_desc* ns, const serl_batch_out* out, float* prio_out, void* stream) {
  if (int e = check_view(rv)) return e;
  if (int e = check_request(rv, rq, out, "serl_replay_sample_crop_prio")) return e;
  if (int e = check_tree(t, rv->capacity, "serl_replay_sample_crop_prio")) return e;
  if (ns) { if (int e = check_nstep(ns, "serl_replay_sample_crop_prio")) return e; }
  SamplerArgs a = sampler_args(rv, rq, out);
  PrioDraw pd{};
  pd.tree = t->nodes; pd.levels = prio_tree_layout(t->capacity, pd.off); pd.prio_out = prio_out;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!ns) return sample_crop_launch<false, false, true>(rv, rq, a, nullptr, st, &pd, out->stacked);
  set_nstep(a, ns);
  return sample_crop_launch<true, false, true>(rv, rq, a, nullptr, st, &pd, out->stacked);
}

static PrioSetArgs prio_args(const serl_priority_tree* t) {
  PrioSetArgs a{};
  a.tree = t->nodes; a.max_dev = t->max_dev; a.ring_valid = t->valid; a.capacity = t->capacity; a.levels = prio_tree_layout(t->capacity, a.off);
  return a;
}

extern "C" int serl_replay_priority_set(const serl_priority_tree* t, const int32_t* slots, const float* td, const uint8_t* valid, int n,
                                        float alpha, float eps, void* stream) {
  if (int e = check_tree(t, -1, "serl_replay_priority_set")) return e;
  if (n < 0 || n > SERL_PRIO_SET_MAX || (n > 0 && (!slots || (!td && !valid))) || (td && !(alpha >= 0.f && eps >= 0.f))) {
    set_last_error("serl_replay_priority_set: invalid arguments (n=%d, max %d; alpha=%g eps=%g)", n, SERL_PRIO_SET_MAX, alpha, eps);
    return SERL_ERR_INVALID;
  }
  if (n == 0) return SERL_OK;
  PrioSetArgs a = prio_args(t);
  a.slots = slots; a.td = td; a.valid = valid; a.n = n; a.alpha = alpha; a.eps = eps;
  launch_k(priority_set_kernel, 1, kPrioThreads, 0, static_cast<cudaStream_t>(stream), a);
  return check_launch("priority_set_kernel");
}

extern "C" int serl_replay_priority_rebuild(const serl_priority_tree* t, void* stream) {
  if (int e = check_tree(t, -1, "serl_replay_priority_rebuild")) return e;
  const PrioSetArgs a = prio_args(t);
  for (int l = 1; l < a.levels; ++l) {
    const int cnt = l + 1 < a.levels ? a.off[l + 1] - a.off[l] : 1;
    launch_k(priority_rebuild_kernel, ceil_div(cnt, 256), 256, 0, static_cast<cudaStream_t>(stream), a, l, cnt);
    if (int e = check_launch("priority_rebuild_kernel")) return e;
  }
  return SERL_OK;
}

extern "C" int serl_replay_priority_weights(const float* prio, int n, const float* beta_dev, float* w, void* stream) {
  if (n < 1 || !prio || !beta_dev || !w) { set_last_error("serl_replay_priority_weights: invalid arguments (n=%d)", n); return SERL_ERR_INVALID; }
  launch_k(priority_weights_kernel, 1, kPrioThreads, 0, static_cast<cudaStream_t>(stream), prio, n, beta_dev, w);
  return check_launch("priority_weights_kernel");
}

static ScatterArgs scatter_args(const serl_replay_view* rv, const serl_scatter_request* rq) {
  ScatterArgs a{};
  a.rv = *rv; a.n = rq->n; a.dst_slot = rq->dst_slot; a.src_slot = rq->src_slot;
  for (int c = 0; c < rv->num_cams; ++c) a.st_frames[c] = rq->frames[c];
  a.st_state = rq->state; a.st_next_state = rq->next_state; a.st_actions = rq->actions;
  a.st_rewards = rq->rewards; a.st_masks = rq->masks; a.st_dones = rq->dones; a.st_valid = rq->valid;
  a.row_stride = rq->row_stride;
  return a;
}

static dim3 scatter_grid(const serl_replay_view* rv, const serl_scatter_request* rq) {
  const size_t fb = (size_t)rv->height * rv->width * rv->channels;
  int chunks = (int)((fb / 16 + 255) / 256); if (chunks < 1) chunks = 1; if (chunks > 16) chunks = 16;
  return dim3(chunks, rv->num_cams > 0 ? rv->num_cams : 1, rq->n);
}

extern "C" int serl_replay_scatter_sharded(const serl_replay_view* rv, const serl_replay_shards* sh, const serl_scatter_request* rq,
                                           void* stream) {
  if (int e = check_view(rv)) return e;
  if (int e = check_shards(rv, sh, "serl_replay_scatter_sharded")) return e;
  if (!rq || rq->n < 0) { set_last_error("serl_replay_scatter_sharded: invalid request"); return SERL_ERR_INVALID; }
  if (rq->n == 0) return SERL_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  serl_replay_view fields = *rv;                         // small fields: every rank writes every slot
  fields.num_cams = 0;
  launch_k(replay_scatter_kernel, dim3(1, 1, rq->n), 256, 0, st, scatter_args(&fields, rq));
  if (int e = check_launch("replay_scatter_kernel")) return e;
  launch_k(replay_scatter_frames_sharded_kernel, scatter_grid(rv, rq), 256, 0, st, scatter_args(rv, rq), *sh);
  return check_launch("replay_scatter_frames_sharded_kernel");
}

extern "C" int serl_replay_scatter(const serl_replay_view* rv, const serl_scatter_request* rq, void* stream) {
  if (int e = check_view(rv)) return e;
  if (!rq || rq->n < 0) { set_last_error("serl_replay_scatter: invalid request"); return SERL_ERR_INVALID; }
  if (rq->n == 0) return SERL_OK;
  launch_k(replay_scatter_kernel, scatter_grid(rv, rq), 256, 0, static_cast<cudaStream_t>(stream), scatter_args(rv, rq));
  return check_launch("replay_scatter_kernel");
}

extern "C" int serl_replay_set_valid(uint8_t* valid, const int32_t* slots, const uint8_t* vals, int n, void* stream) {
  if (n <= 0) return SERL_OK;
  launch_k(replay_set_valid_kernel, ceil_div(n, 128), 128, 0, static_cast<cudaStream_t>(stream), valid, slots, vals, n, nullptr, 0);
  return check_launch("replay_set_valid_kernel");
}

extern "C" int serl_replay_commit(uint8_t* valid, const int32_t* slots, const uint8_t* vals, int n, int32_t* size_dev, int32_t size, void* stream) {
  if (n < 0 || !size_dev) { set_last_error("serl_replay_commit: invalid arguments"); return SERL_ERR_INVALID; }
  launch_k(replay_set_valid_kernel, n > 0 ? ceil_div(n, 128) : 1, 128, 0, static_cast<cudaStream_t>(stream), valid, slots, vals, n, size_dev, size);
  return check_launch("replay_set_valid_kernel");
}

extern "C" int serl_counter_add(uint64_t* counter, uint64_t inc, void* stream) {
  launch_k(counter_add_kernel, 1, 32, 0, static_cast<cudaStream_t>(stream), counter, inc);
  return check_launch("counter_add_kernel");
}

// Host-side mirrors of the integer RNG specs (no GPU needed): used by CPU tests to pin the device
// functions (same __host__ __device__ code) against oracle/jax_prng.py and oracle/replay.py.
extern "C" int serl_host_crop_offsets(const uint32_t key[2], int n_frames, int padding, int32_t* out) {
  for (int g = 0; g < n_frames; ++g) {
    u32x2 k = jax_split_at(u32x2{key[0], key[1]}, (uint32_t)n_frames, (uint32_t)g);
    int cy, cx; jax_randint2(k, (uint32_t)(2 * padding + 1), &cy, &cx);
    out[2 * g] = cy; out[2 * g + 1] = cx;
  }
  return SERL_OK;
}

extern "C" int serl_host_draw_indices(uint64_t seed, uint64_t step, uint32_t lane_offset, int batch, int size,
                                      const uint8_t* valid, int32_t* out) {
  if (size < 1) return SERL_ERR_INVALID;
  const uint32_t thresh = (uint32_t)((0x100000000ull - (uint32_t)size) % (uint32_t)size);
  for (int i = 0; i < batch; ++i) {
    out[i] = -1;
    for (int att = 0; att < kMaxDrawAttempts; ++att) {
      u32x4 r = philox4x32_10(u32x4{lane_offset + (uint32_t)i, (uint32_t)att, (uint32_t)step, (uint32_t)(step >> 32)},
                              (uint32_t)seed, (uint32_t)(seed >> 32));
      uint64_t m = (uint64_t)r.x * (uint32_t)size;
      if ((uint32_t)m < thresh) continue;
      uint32_t idx = (uint32_t)(m >> 32);
      if (valid[idx]) { out[i] = (int)idx; break; }
    }
  }
  return SERL_OK;
}

extern "C" int serl_host_draw_prio(const float* nodes_host, const uint8_t* valid_host, int capacity, uint64_t seed, uint64_t step,
                                   uint32_t lane_offset, int batch, int32_t* out) {
  if (!nodes_host || !valid_host || capacity < 1 || batch < 1) return SERL_ERR_INVALID;
  int off[SERL_MAX_TREE_LEVELS];
  const int levels = prio_tree_layout(capacity, off);
  for (int b = 0; b < batch; ++b) {
    out[b] = -1;
    for (int att = 0; att < kMaxDrawAttempts; ++att) {
      u32x4 r = philox4x32_10(u32x4{lane_offset + (uint32_t)b, (uint32_t)att, (uint32_t)step, (uint32_t)(step >> 32)},
                              (uint32_t)seed, (uint32_t)(seed >> 32));
      float p;
      const int idx = prio_descend(nodes_host, off, levels, b, batch, r.x, &p);
      if (idx >= 0 && p > 0.f && valid_host[idx]) { out[b] = idx; break; }
    }
  }
  return SERL_OK;
}

extern "C" int serl_host_threefry_split(const uint32_t key[2], int n, uint32_t* out) {
  for (int i = 0; i < n; ++i) { u32x2 k = jax_split_at(u32x2{key[0], key[1]}, (uint32_t)n, (uint32_t)i); out[2 * i] = k.x; out[2 * i + 1] = k.y; }
  return SERL_OK;
}

extern "C" int serl_host_random_bits(const uint32_t key[2], int size, uint32_t* out) {
  for (int j = 0; j < size; ++j) out[j] = jax_random_bits_at(u32x2{key[0], key[1]}, (uint32_t)size, (uint32_t)j);
  return SERL_OK;
}

// ---- CUDA IPC of frame allocations (frame-sharded replay) ----------------------------------------------------------------
static_assert(sizeof(cudaIpcMemHandle_t) == SERL_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t size");

typedef int (*AddressRangeFn)(unsigned long long* base, size_t* size, unsigned long long ptr);   // cuMemGetAddressRange_v2

extern "C" int serl_ipc_export(const void* ptr, void* handle_host, uint64_t* offset_host) {
  cudaIpcMemHandle_t h;
  if (!ptr || !handle_host || !offset_host) { set_last_error("serl_ipc_export: null pointer"); return SERL_ERR_INVALID; }
  static AddressRangeFn range = nullptr;
  if (!range) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q{};
    if (cudaGetDriverEntryPointByVersion("cuMemGetAddressRange", &fn, 12000, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess || !fn) {
      set_last_error("serl_ipc_export: the driver has no cuMemGetAddressRange"); return SERL_ERR_CUDA;
    }
    range = reinterpret_cast<AddressRangeFn>(fn);
  }
  unsigned long long base = 0;
  size_t bytes = 0;
  if (int rc = range(&base, &bytes, reinterpret_cast<unsigned long long>(ptr))) {
    set_last_error("serl_ipc_export: cuMemGetAddressRange failed (%d)", rc); return SERL_ERR_CUDA;
  }
  if (cudaError_t e = cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base))) {
    set_last_error("serl_ipc_export: cudaIpcGetMemHandle: %s", cudaGetErrorString(e)); return SERL_ERR_CUDA;
  }
  memcpy(handle_host, &h, sizeof(h));
  *offset_host = reinterpret_cast<unsigned long long>(ptr) - base;
  return SERL_OK;
}

extern "C" int serl_ipc_open(const void* handle_host, void** base_host) {
  cudaIpcMemHandle_t h;
  if (!handle_host || !base_host) { set_last_error("serl_ipc_open: null pointer"); return SERL_ERR_INVALID; }
  memcpy(&h, handle_host, sizeof(h));
  if (cudaError_t e = cudaIpcOpenMemHandle(base_host, h, cudaIpcMemLazyEnablePeerAccess)) {
    set_last_error("serl_ipc_open: cudaIpcOpenMemHandle: %s", cudaGetErrorString(e)); return SERL_ERR_CUDA;
  }
  return SERL_OK;
}

extern "C" int serl_ipc_close(void* base) {
  if (cudaError_t e = cudaIpcCloseMemHandle(base)) {
    set_last_error("serl_ipc_close: cudaIpcCloseMemHandle: %s", cudaGetErrorString(e)); return SERL_ERR_CUDA;
  }
  return SERL_OK;
}

extern "C" int serl_can_access_peer(int device, int peer_device) {
  if (device == peer_device) return 1;
  int ok = 0;
  if (cudaError_t e = cudaDeviceCanAccessPeer(&ok, device, peer_device)) {
    set_last_error("serl_can_access_peer(%d, %d): %s", device, peer_device, cudaGetErrorString(e)); return SERL_ERR_CUDA;
  }
  return ok ? 1 : 0;
}

extern "C" int serl_copy_async(void* dst, const void* src, size_t bytes, void* stream) {
  if (cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream))) {
    set_last_error("serl_copy_async: %s", cudaGetErrorString(e)); return SERL_ERR_CUDA;
  }
  return SERL_OK;
}
