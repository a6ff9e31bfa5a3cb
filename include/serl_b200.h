/* libserl_b200 - C ABI of the H100 (sm_90a) DrQ/SAC learner hot path.
 *
 * The reference (rail-berkeley/serl) has no FFI: its boundary is the Python API of `serl_launcher`
 * (SURVEY.md §8b).  This header is the C-ABI underneath this repo's Python mirror of that API
 * (serl_b200/): plain pointers and sizes, an explicit CUDA stream (cudaStream_t passed as void*),
 * no torch types, no allocation inside the library (callers own all buffers / workspaces).
 * Every function returns 0 on success or a negative SERL_ERR_* code; serl_last_error() gives the
 * message for the calling thread.  All pointers are DEVICE pointers unless a name says `host`.
 *
 * Citations are relative to /root/reference/serl_launcher/serl_launcher.
 */
#ifndef SERL_B200_H_
#define SERL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SERL_MAX_CAMS 4

/* ---- library ------------------------------------------------------------------------------- */
const char* serl_last_error(void);
int serl_version(void);                       /* ABI version, bumped on signature changes */
unsigned long long serl_launch_count(void);   /* kernels this library has enqueued in this process (graph capture included) */
int serl_device_sm_count(int device);         /* host query used to size persistent grids */
int serl_balanced_grid(int items, int sms);   /* CTAs of a persistent one-CTA-per-SM kernel over `items` work items: the smallest grid with as few waves as min(items, sms) CTAs */
/* Work units a persistent launch of the 16-bit frozen trunk keeps resident at once, as its entry point sizes its grid: a pass
 * over `work` units runs ceil(work / units) rounds on ceil(work / rounds) units.  The units are images (4-CTA clusters) for
 * SERL_TRUNK_STEM and SERL_TRUNK_RES32, images (CTA pairs) for SERL_TRUNK_RES16, and CTAs over items of
 * ceil(N / images per item) x channel slices for the others.  fmt: SERL_FMT_FP16 / SERL_FMT_BF16. */
enum { SERL_TRUNK_STEM = 0, SERL_TRUNK_RES32, SERL_TRUNK_RES16, SERL_TRUNK_HEAD16, SERL_TRUNK_HEAD8, SERL_TRUNK_RES8, SERL_TRUNK_HEAD4,
       SERL_TRUNK_RES4 };
int serl_trunk_resident_units(int launch, int fmt);

/* ---- replay ring in HBM ---------------------------------------------------------------------
 * Storage layout of data/replay_buffer.py:41-66 + data/memory_efficient_replay_buffer.py:13-51:
 * ONE camera frame per slot (frame dedup), per-slot scalars, a validity byte per slot. */
typedef struct serl_replay_view {
  const uint8_t* frames[SERL_MAX_CAMS];  /* (capacity, H, W, C) uint8 per camera                   */
  const float* state;                    /* (capacity, T*S) observations.state                      */
  const float* next_state;               /* (capacity, T*S) next_observations.state                 */
  const float* actions;                  /* (capacity, A)                                           */
  const float* rewards;                  /* (capacity,)                                             */
  const float* masks;                    /* (capacity,)                                             */
  const uint8_t* dones;                  /* (capacity,)                                             */
  const uint8_t* valid;                  /* (capacity,) _is_correct_index                           */
  int32_t num_cams, height, width, channels, num_stack /*T*/, state_dim /*S*/, action_dim /*A*/;
  int32_t capacity, size;                /* size = len(buffer): draws are uniform over [0, size)    */
} serl_replay_view;

typedef struct serl_sample_request {
  uint64_t seed, step;           /* Philox key / counter words of the index draw (repo spec)         */
  const uint64_t* step_dev;      /* optional device counter overriding `step` (CUDA-graph replay)     */
  const int32_t* size_dev;       /* optional device fill level overriding rv->size                    */
  uint32_t lane_offset;          /* Philox lane of output row 0                                      */
  int32_t batch;                 /* rows drawn by this call                                          */
  const int32_t* explicit_idx;   /* optional (batch): gather these slots instead of drawing          */
  const uint32_t* key_obs;       /* device uint32[2]: JAX key; frame g uses split(key, crop_total)[g] */
  const uint32_t* key_next;
  const int32_t* explicit_off_obs;   /* optional (crop_total, 2) [cy, cx] overriding the keys        */
  const int32_t* explicit_off_next;
  int32_t crop_total;            /* frames in the whole (possibly concatenated) batch = B_total * T   */
  int32_t out_row_offset;        /* first output row written by this call (RLPD: demo half offset)    */
  int32_t padding;               /* DrQ pad (4): offsets in [0, 2*padding]                            */
} serl_sample_request;

typedef struct serl_batch_out {
  uint8_t* obs_pix[SERL_MAX_CAMS];   /* (B_total, T, H, W, C) shifted observation frames             */
  uint8_t* next_pix[SERL_MAX_CAMS];  /* (B_total, T, H, W, C) shifted next-observation frames         */
  float* obs_state; float* next_state;   /* (B_total, T*S)                                           */
  float* actions; float* rewards; float* masks; uint8_t* dones;
  int32_t* idx;                      /* optional (B_total) drawn slots                                */
  int32_t* off_obs; int32_t* off_next;   /* optional (B_total*T, 2) applied offsets                   */
  int32_t* status;                   /* device int32, OR-ed with 1 if a draw found no valid slot      */
  int32_t stacked;                   /* 1: obs_pix / next_pix are (B_total, H, W, T*C) instead, the T frames of a row
                                        stacked on the channel axis oldest first (EncodingWrapper's enable_stacking
                                        rearrange "B T H W C -> B H W (T C)"); the same bytes as 0 when T = 1            */
} serl_batch_out;

/* Replaces MemoryEfficientReplayBuffer.sample (memory_efficient_replay_buffer.py:91-164) +
 * ReplayBuffer.get_iterator's device_put (replay_buffer.py:77-90) + _unpack (utils/train_utils.py:44-66)
 * + batched_random_crop (vision/data_augmentations.py:7-36, agents/continuous/drq.py:244-253). */
int serl_replay_sample_crop(const serl_replay_view* rv, const serl_sample_request* rq,
                            const serl_batch_out* out, void* stream);

/* n-step returns.  Drawn slot i (same draw, same crops as serl_replay_sample_crop) carries the window of the largest m <= n
 * such that slots i .. i+m-1 (mod capacity) are written (at or behind the newest slot, head-1) and valid, and none of
 * i .. i+m-2 has dones = 1:
 *   rewards = sum_{k<m} discount^k r[i+k]   (fp32: g = 1, R = r[i]; for k = 1..m-1: g = g*discount, R = R + g*r[i+k]; no FMA)
 *   masks = g * masks[i+m-1],  dones = dones[i+m-1],  next observation (frames + state) = slot i+m-1's, with the row's
 *   next-observation crop offsets.
 * Observations, actions and the observation crop are slot i's.  n = 1 reproduces serl_replay_sample_crop bit for bit. */
#define SERL_MAX_NSTEP 16
typedef struct serl_nstep_desc {
  int32_t n;                     /* window bound, 1..SERL_MAX_NSTEP                                   */
  float discount;
  const int32_t* head_dev;       /* device int32: the ring's insert index (read on the device: graph replays see new inserts) */
  int32_t* m_out;                /* optional (B_total) window length m of each row                    */
  int32_t* next_idx_out;         /* optional (B_total) slot i+m-1 whose next observation the row holds */
} serl_nstep_desc;

int serl_replay_sample_crop_nstep(const serl_replay_view* rv, const serl_sample_request* rq, const serl_nstep_desc* ns,
                                  const serl_batch_out* out, void* stream);

typedef struct serl_scatter_request {
  int32_t n;                         /* slot writes, applied independently (no ordering inside a call) */
  const int32_t* dst_slot;           /* (n)                                                            */
  const int32_t* src_slot;           /* (n)  >= 0: copy from that ring slot; < 0: from staging row k    */
  const uint8_t* frames[SERL_MAX_CAMS];  /* staging (n, H, W, C)                                       */
  const float* state; const float* next_state; const float* actions;
  const float* rewards; const float* masks; const uint8_t* dones;
  const uint8_t* valid;              /* (n) validity byte to store                                     */
  int64_t row_stride;                /* 0: the fields above are packed (n, ...) arrays; else they point into row 0 of an
                                      * interleaved staging record and row k lies k*row_stride BYTES further (the whole
                                      * staged batch then moves host->device as ONE copy)                          */
} serl_scatter_request;

/* Device side of MemoryEfficientReplayBuffer.insert (memory_efficient_replay_buffer.py:53-89,
 * replay_buffer.py:71-75): applies slot writes staged by the host ring logic. */
int serl_replay_scatter(const serl_replay_view* rv, const serl_scatter_request* rq, void* stream);
int serl_counter_add(uint64_t* counter, uint64_t inc, void* stream);   /* device-resident step counters */
int serl_replay_set_valid(uint8_t* valid, const int32_t* slots, const uint8_t* vals, int n, void* stream);
/* same + publishes the ring's new size to its device-resident copy (read by graph-replayed sampling launches) */
int serl_replay_commit(uint8_t* valid, const int32_t* slots, const uint8_t* vals, int n, int32_t* size_dev, int32_t size, void* stream);

/* ---- prioritized replay (proportional, Schaul et al. 2016) -------------------------------------------
 * Sum tree over a ring's `capacity` slots, fan-out 32, every level in ONE float array, leaves first:
 *   count[0] = capacity, count[l] = ceil(count[l-1] / 32) until a level of 1 node (the root; capacity 1: the leaf is the root);
 *   offset[0] = 0, offset[l] = offset[l-1] + count[l-1]; nodes = offset[L-1] + 1 floats.
 * Leaf i is slot i's priority p_i (0 while the slot is not valid).  Node j of level l >= 1 is the fp32 sum, from 0 in ascending
 * order, of children 32j .. min(32j+31, count[l-1]-1) of level l-1, and is RECOMPUTED from its children whenever one changes, so
 * the tree is a pure function of its leaves.  max_dev holds the running maximum m (1.0 in a new ring) given to new slots.
 *
 * Draw of row b of a call of B = rq->batch rows (stratified, proportional): attempt a takes word x of the same Philox block as
 * the uniform draw, counter (lane_offset + b, a, step), and
 *   u = fl(fl(fl(b + fl(x) * 2^-32) / B) * root)                                   (fl: fp32 round-to-nearest; x*2^-32 is exact)
 * then descends from the root: over a node's children in order, with running prefix s (fl(s + child)), it takes the first
 * child whose new prefix exceeds u and sets u = fl(u - s) with s the prefix before it; when none does, the last child with a
 * non-zero sum (same subtraction); a node whose children are all 0 fails the attempt.  A leaf of 0 or a slot that is not valid
 * fails the attempt too; after the same attempt budget as the uniform draw the row sets status.  explicit_idx skips the draw.
 * Writers of one tree (ring flushes, priority updates) and its draws must run in stream order: two priority writes running
 * concurrently could recompute a shared ancestor from a child the other has not written yet. */
#define SERL_PRIO_FANOUT 32
#define SERL_MAX_TREE_LEVELS 8
typedef struct serl_priority_tree {
  float* nodes;                  /* (nodes) the tree above                                               */
  float* max_dev;                /* device float: running maximum priority m                             */
  const uint8_t* valid;          /* optional (capacity) ring validity: a TD write to a slot that is not valid writes 0 */
  int32_t capacity;              /* leaves                                                               */
} serl_priority_tree;

/* serl_replay_sample_crop (ns == NULL) / _nstep (ns != NULL) with the draw above; the same gathers and crops for the drawn
 * slots.  An n-step row's window starts at its drawn slot.  prio_out: optional (B_total) leaf p of each row's slot. */
int serl_replay_sample_crop_prio(const serl_replay_view* rv, const serl_sample_request* rq, const serl_priority_tree* t,
                                 const serl_nstep_desc* ns, const serl_batch_out* out, float* prio_out, void* stream);
/* Sets leaves slots[0..n) and recomputes their ancestors level by level.  td != NULL: p_k = powf(|td_k| + eps, alpha) (0 where
 * t->valid says the slot is not valid; an entry with a non-finite td is skipped) and m = max(m, written p).  td == NULL:
 * p_k = valid[k] ? m : 0 (a ring flush).  A slot named twice takes its LAST entry.
 * Entries naming a slot outside [0, capacity) are skipped.  n <= SERL_PRIO_SET_MAX per call (later calls override earlier
 * ones, so longer lists go in order, in pieces). */
#define SERL_PRIO_SET_MAX 4096
int serl_replay_priority_set(const serl_priority_tree* t, const int32_t* slots, const float* td, const uint8_t* valid, int n,
                             float alpha, float eps, void* stream);
/* Recomputes every interior node from the leaves (after the leaves were written directly, e.g. by a load). */
int serl_replay_priority_rebuild(const serl_priority_tree* t, void* stream);
/* Importance weights of one part's n drawn rows: w_k = powf(fl(p_min / p_k), beta), p_min = the smallest non-zero p_k, beta
 * read from beta_dev (device float); a row with p_k = 0 (an explicit index naming a slot of priority 0) gets w_k = 0. */
int serl_replay_priority_weights(const float* prio, int n, const float* beta_dev, float* w, void* stream);
/* Host mirror of the draw (nodes_host: the whole tree in host memory); CPU tests pin it against oracle/per.py. */
int serl_host_draw_prio(const float* nodes_host, const uint8_t* valid_host, int capacity, uint64_t seed, uint64_t step,
                        uint32_t lane_offset, int batch, int32_t* out);

/* ---- frame-sharded replay (data-parallel learner) ------------------------------------------------
 * Only the frames are sharded; every other field of the view stays a full replica on every rank.  Rank r of `world` owns
 * slots [lo_r, hi_r), lo_r = r * slots_per_rank, hi_r = min(lo_r + slots_per_rank, capacity), and also stores the `halo`
 * slots in front of lo_r, (lo_r - halo .. lo_r - 1) mod capacity.  Its frame allocation holds slot s at local index
 * (s - lo_r + halo) mod capacity, so frames[cam][r] points at slot lo_r - halo.  The T + 1 frames a row reads (window
 * w0 .. w0 + T, see the sampler) are read from the owner of w0 + T, where they are contiguous.  frames[cam][r] may be a
 * peer's allocation mapped into this process (serl_ipc_open). */
#define SERL_MAX_SHARD_RANKS 8
typedef struct serl_replay_shards {
  const uint8_t* frames[SERL_MAX_CAMS][SERL_MAX_SHARD_RANKS];  /* per camera, per rank: that rank's frame allocation */
  int32_t slots_per_rank;        /* ceil(capacity / world)                                             */
  int32_t halo;                  /* slots stored in front of lo_r: the frame stack T                    */
  int32_t world, rank;           /* world <= SERL_MAX_SHARD_RANKS; rank = the calling rank (scatter)    */
} serl_replay_shards;

/* serl_replay_sample_crop / _nstep with every frame read from its owner's allocation: the same batch, bit for bit. */
int serl_replay_sample_crop_sharded(const serl_replay_view* rv, const serl_replay_shards* sh, const serl_sample_request* rq,
                                    const serl_batch_out* out, void* stream);
int serl_replay_sample_crop_nstep_sharded(const serl_replay_view* rv, const serl_replay_shards* sh, const serl_sample_request* rq,
                                          const serl_nstep_desc* ns, const serl_batch_out* out, void* stream);
/* serl_replay_scatter into rank sh->rank's frame allocation: a frame write lands only where its slot is in the rank's range or
 * halo, and a slot copy (src_slot >= 0) reads the source frame from the same allocation. */
int serl_replay_scatter_sharded(const serl_replay_view* rv, const serl_replay_shards* sh, const serl_scatter_request* rq, void* stream);

/* CUDA IPC of one device allocation between processes (cudaIpcGetMemHandle / cudaIpcOpenMemHandle with
 * cudaIpcMemLazyEnablePeerAccess / cudaIpcCloseMemHandle).  handle_host: host buffer of SERL_IPC_HANDLE_BYTES.  A handle
 * names the whole allocation that holds `ptr` (a caching allocator may have carved `ptr` out of a larger one), so export also
 * returns ptr's byte offset into it: the peer's pointer is the base serl_ipc_open returns plus that offset. */
#define SERL_IPC_HANDLE_BYTES 64
int serl_ipc_export(const void* ptr, void* handle_host, uint64_t* offset_host);
int serl_ipc_open(const void* handle_host, void** base_host);
int serl_ipc_close(void* base);
int serl_can_access_peer(int device, int peer_device);   /* 1: device can map peer_device's memory (same device: 1), 0: not */
int serl_copy_async(void* dst, const void* src, size_t bytes, void* stream);   /* cudaMemcpyAsync(cudaMemcpyDefault) */

/* ---- JAX-compatible key schedule and random fills ---------------------------------------------
 * Key slots written by serl_rng_schedule (uint32[2] each), following SACAgent.update's split order
 * (agents/continuous/sac.py:137,152,197,224,288; common/common.py:198-200; drq.py:307-308). */
enum {
  SERL_KEY_CROP_OBS = 0, SERL_KEY_CROP_NEXT = 1, SERL_KEY_CRITIC_NEXT = 2, SERL_KEY_CRITIC_SUBSAMPLE = 3,
  SERL_KEY_ACTOR_DROPOUT = 4, SERL_KEY_ACTOR_SAMPLE = 5, SERL_KEY_TEMP_NEXT = 6, SERL_NUM_KEYS = 8
};
int serl_rng_schedule(uint32_t* rng_state, uint32_t* keys, int do_aug, int do_update, void* stream);
/* Critic-MLP dropout keys of an update (critic / policy network_kwargs dropout_rate > 0), written to slots past SERL_NUM_KEYS
 * (keys holds SERL_NUM_KEYS_MLP slots): c1 (target critic), c2 = split(c1)[0] (online critic under critic_subsample_size; c1
 * without) and the actor loss's critic_rng (sac.py:137-176,197).  Reads rng_state BEFORE serl_rng_schedule advances it, with the
 * same do_aug; the policy passes' MLP masks use the slots serl_rng_schedule writes (DESIGN.md section 4). */
enum { SERL_KEY_MLP_CRITIC_TARGET = 8, SERL_KEY_MLP_CRITIC_SUBSAMPLED = 9, SERL_KEY_MLP_ACTOR_CRITIC = 10, SERL_NUM_KEYS_MLP = 12 };
int serl_mlp_dropout_keys(const uint32_t* rng_state, uint32_t* keys, int do_aug, void* stream);
int serl_host_mlp_dropout_keys(const uint32_t* rng, uint32_t* keys, int do_aug);
/* BCAgent.update's key chain (common/common.py:198-200 with one loss, agents/continuous/bc.py:47): new_rng, k = split(rng);
 * key = split(k)[1] (the step's dropout key); rng_state = new_rng. */
int serl_bc_key_chain(uint32_t* rng_state, uint32_t* key, void* stream);
int serl_host_bc_key_chain(uint32_t* rng_host, uint32_t* key_host);
int serl_normal_fill(const uint32_t* key, float* out, int n, void* stream);            /* jax.random.normal   */
int serl_dropout_mask_fill(const uint32_t* key, uint32_t fold, float keep, uint8_t* mask, int n, void* stream);
int serl_subsample_idx(const uint32_t* key, int ensemble, int32_t* out /*n*/, int n, void* stream); /* randint(key,(n,),0,E), sac.py:153-158 */

/* Host mirrors of the integer RNG specs (same code compiled for the host; usable without a GPU). */
int serl_host_rng_schedule(uint32_t* rng_state_host, uint32_t* keys_host, int do_aug, int do_update);
int serl_host_crop_offsets(const uint32_t key_host[2], int n_frames, int padding, int32_t* out_host);
int serl_host_draw_indices(uint64_t seed, uint64_t step, uint32_t lane_offset, int batch, int size,
                           const uint8_t* valid_host, int32_t* out_host);
int serl_host_threefry_split(const uint32_t key_host[2], int n, uint32_t* out_host);
int serl_host_random_bits(const uint32_t key_host[2], int size, uint32_t* out_host);

/* ---- frozen ResNet-10 trunk, fp32 build (vision/resnet_v1.py:217-286,129-156) ------------------ */
/* NHWC conv, HWIO weights, explicit low/high zero padding.  x_is_u8: x is uint8 and the ImageNet
 * normalisation (x/255 - mean)/std of resnet_v1.py:222-224 is fused into the operand load. */
int serl_conv2d_nhwc_f32(const void* x, int x_is_u8, const float* w, float* y, int N, int Hi, int Wi, int Ci,
                         int Co, int kh, int kw, int stride, int pad_lo, int pad_hi, void* stream);
/* GroupNorm (flax statistics), optional residual add and ReLU; y may alias x. */
int serl_groupnorm_nhwc_f32(const float* x, float* y, const float* scale, const float* bias, const float* residual,
                            int N, int HW, int C, int groups, float eps, int relu, void* stream);
int serl_maxpool3x3s2_nhwc_f32(const float* x, float* y, int N, int Hi, int Wi, int C, void* stream);

/* ---- frozen ResNet-10 trunk, 16-bit build on the wgmma tensor cores (same layers as above) -------- */
/* operand format of the kind::f16 MMAs: bf16, or fp16 (same throughput, 3 more mantissa bits; packs saturate) */
enum { SERL_FMT_BF16 = 0, SERL_FMT_FP16 = 1 };
/* uint8 crops (N,H,W,3) -> normalised 16-bit, 2x2 space-to-depth, zero padded: xs (N, H/2+3, W/2+3, 16)
 * (12 real channels (p,q,c) + 4 zero channels, so four taps are one aligned 128-byte operand row) */
int serl_trunk_stem_prep_h16(const uint8_t* x, void* xs, int N, int H, int W, int fmt, void* stream);
/* The unfused stem conv_init (7x7/2 as a 4x4/1 conv over the space-to-depth image): raw 16-bit output + GroupNorm sums.  Not on
 * the product path: with serl_gn_finalize and serl_maxpool_affine_h16 it is the reference the fused stem below equals bit for
 * bit.  A descriptor with stem == 0 or an operand transform returns SERL_ERR_UNSUPPORTED. */
typedef struct serl_conv_tc_desc {
  const void* x;           /* 16-bit space-to-depth image (N,Hi,Wi,16) from serl_trunk_stem_prep_h16 (Ci ignored)  */
  const void* w;           /* 16-bit [64][4 x 64], K-major (48 valid per row), from the stem weight packing          */
  void* y;                 /* 16-bit (N,Ho,Wo,64) raw convolution output (pre-GroupNorm)                              */
  float* stats;            /* (N,4,2) fp32 sum / sum-of-squares per GroupNorm group, accumulated (pre-zero it)       */
  const float* in_a;       /* must be null                                                                            */
  const float* in_b;
  int32_t* error;          /* device int32, OR-ed with 2 if a pipeline barrier timed out                             */
  int32_t N, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad_lo, stem, fmt;
} serl_conv_tc_desc;
int serl_conv2d_tc_h16(const serl_conv_tc_desc* d, void* stream);
/* conv_init (7x7/2 as a 4x4/1 conv over the space-to-depth image) FUSED with the 3x3/2 SAME max-pool that follows its
 * GroupNorm + ReLU (vision/resnet_v1.py:247-261).  relu(a*x+b) is monotone in x with the sign of the frozen GroupNorm
 * scale, so the pool runs on the raw sign-adjusted conv output inside the epilogue and the 64x64 map never reaches HBM.
 * xs (N,67,67,16) from serl_trunk_stem_prep_h16; w = packed stem weights; pooled (N,32,32,64); side (N,4,32,64);
 * stats (N,4,2) GroupNorm sums of the raw conv output; neg_mask bit c = (scale[c] < 0).
 * serl_pool_finish_h16 then writes y = relu(|a| * pooled' + b) with (a, b) from serl_gn_finalize. */
typedef struct serl_stem_pool_desc {
  const void* xs; const void* w; void* pooled; void* side; float* stats; int32_t* error;
  uint64_t neg_mask;
  int32_t N, fmt;
} serl_stem_pool_desc;
int serl_stem_conv_pool_tc_h16(const serl_stem_pool_desc* d, void* stream);
int serl_pool_finish_h16(const void* pooled, const void* side, const float* a, const float* b, void* y, int N, int fmt, void* stream);
/* "_gn" consumers: take the conv epilogue's GroupNorm sums (N,4,2) + the frozen scale / bias instead of a finalized (a, b)
 * table and derive the affine in registers (same arithmetic as serl_gn_finalize) - no finalize launch in the chain. */
int serl_pool_finish_gn_h16(const void* pooled, const void* side, const float* stats, const float* gamma, const float* beta, void* y,
                            int N, float eps, int fmt, void* stream);
/* (N,4,2) sums -> per-(image, channel) affine a = rstd*gamma, b = beta - mean*a (flax GroupNorm statistics) */
int serl_gn_finalize(const float* stats, const float* gamma, const float* beta, float* out_a, float* out_b, int N, int C,
                     int HW, float eps, void* stream);
int serl_maxpool_affine_h16(const void* x, const float* a, const float* b, void* y, int N, int Hi, int Wi, int C, int fmt, void* stream);

/* ---- dense algebra for the trainable heads (fp32) ---------------------------------------------- */
typedef struct serl_gemm_desc {
  const float* A; const float* B; float* C; const float* bias;
  float* workspace; size_t workspace_bytes;     /* split-K / batch-reduce partials */
  int32_t M, N, K, Z;
  int64_t sAz, sAm, sAk, sBz, sBk, sBn, sCz, sBiasZ;
  int32_t ldc;
  int32_t accumulate;                           /* C += result                                     */
  int32_t reduce_z;                             /* single C = sum over z                           */
} serl_gemm_desc;
int serl_gemm_f32(const serl_gemm_desc* d, void* stream);
/* Same contract on the tensor cores: fp32 operands split into TF32 hi + lo parts, three wgmma (tf32) products
 * per k-step accumulated in fp32 registers ("3xTF32": fp32-class accuracy, ~2^-22 per product).  Heads of the 16-bit builds. */
int serl_gemm_tf32x3(const serl_gemm_desc* d, void* stream);

/* Heads of the 16-bit builds, round 2: fp32 GEMM on the tensor cores (wgmma, 3xTF32 split; operands staged from the fp32
 * tensors in either layout: X @ W, dZ @ W^T and X^T @ dZ of a Dense layer all read the row-major arrays in place) with fused epilogues.
 * Replaces, per launch, Dense (+ bias) [+ LayerNorm + tanh [+ value head | + policy heads + tanh-Gaussian sample]] of
 * networks/mlp.py:22-31, networks/actor_critic_nets.py:57-73,178-227,230-272, vision/resnet_v1.py:371-374.
 * C[z](m, n) = sum_k A[z](m, k) B[z](k, n); element strides in floats; per operand one of its two strides must be 1 and the
 * other a multiple of 4, base pointers 16-byte aligned (TMA), z stride 0 = the operand is shared by the Z members.
 * Up to SERL_TGEMM_MAX_PROBLEMS problems (same M, N, K, operand layouts and epilogue) per launch. */
#define SERL_TGEMM_MAX_PROBLEMS 6
#define SERL_TGEMM_EPI_STORE 0            /* C = acc + bias (+ C)                                                        */
#define SERL_TGEMM_EPI_LN_TANH 1          /* N == 256: C = tanh(LayerNorm(acc + bias) * scale + ln_bias); optional xhat, rstd */
#define SERL_TGEMM_EPI_LN_TANH_HEAD 2     /* ... and head_out[m, :head_n] = C[m, :] @ head_w (256, head_n) + head_b        */
#define SERL_TGEMM_EPI_PARTIAL 4          /* k-split partial products left in the workspace [(member * splits + s)][M][N] for serl_enc_finish */
#define SERL_TGEMM_EPI_LN_TANH_POLICY 3   /* ... two heads (means, log-stds) -> clipped std, u = mu + std * noise, act = tanh(u), logp */
typedef struct serl_tgemm_problem {
  const float* A; const float* B;
  int64_t sAz, sAm, sAk, sBz, sBk, sBn;
  int32_t Z;
  float* C; int64_t sCz; int32_t ldc;            /* may be NULL for the LayerNorm epilogues (activation not kept)          */
  const float* bias; int64_t sBiasZ;
  const float* ln_scale; const float* ln_bias; int64_t sLnZ;
  float* xhat; float* rstd; int64_t sXhatZ, sRstdZ;   /* optional saves for the backward pass: xhat (M, 256), rstd (M)     */
  const float* head_w; const float* head_b; int64_t sHeadWz, sHeadBz;
  float* head_out; int64_t sHeadOutZ; int32_t ld_head;  /* HEAD: (M, head_n) with row stride ld_head; POLICY: means (M, A)   */
  const float* head_w2; const float* head_b2; float* head_out2;   /* POLICY: log-std head and its raw output (M, A)        */
  const float* noise; float* act; int32_t ld_act; float* logp; float* u_out; float* std_out;   /* POLICY (Z == 1)          */
} serl_tgemm_problem;
typedef struct serl_tgemm_desc {
  const serl_tgemm_problem* problems; int32_t num_problems;   /* HOST array                                                */
  int32_t M, N, K;
  int32_t epilogue, head_n;
  int32_t accumulate, reduce_z, splits;          /* splits: 0 = automatic k-split (one problem per launch when > 1)        */
  float ln_eps, std_min, std_max; int32_t deterministic;
  float* workspace; size_t workspace_bytes;      /* k-split / reduce_z partials                                           */
  int32_t* error;                                /* device int32, OR-ed with 32 if a pipeline barrier timed out             */
} serl_tgemm_desc;
int serl_tgemm_tf32(const serl_tgemm_desc* d, void* stream);
/* serl_tgemm_tf32 with the MLP's Dropout in a LayerNorm epilogue (LN_TANH, LN_TANH_HEAD, LN_TANH_POLICY): masks is a HOST array of
 * one 16-byte aligned (M, 256) uint8 keep mask per problem, shared by the problem's Z members; z' = mask ? (acc + bias) * inv_keep
 * : 0 ahead of the LayerNorm statistics, and xhat / rstd are saved for z'. */
int serl_tgemm_tf32_masked(const serl_tgemm_desc* d, const uint8_t* const* masks, float inv_keep, void* stream);

/* Batched companions of serl_tgemm_tf32 (csrc/heads_fused.cu): one launch over every problem of a step. */
#define SERL_HEADS_MAX_PROBLEMS 12
typedef struct serl_sle_problem {             /* SpatialLearnedEmbeddings (+ Dropout keep mask), vision/resnet_v1.py:81-116,352 */
  const float* feat; const float* kernel; const uint8_t* keep_mask; float* out; int32_t ld_out;
} serl_sle_problem;
int serl_sle_fwd_multi(const serl_sle_problem* problems /*host*/, int num_problems, float keep, int N, int P, int C, int F, void* stream);
typedef struct serl_sle_bwd_problem {         /* SLE kernel gradient: dkernel[p,c,f] = sum_n feat[n,p,c] * dout[n, c*8+f]              */
  const float* feat; const float* dout; int32_t ld_dout; float* dkernel;
} serl_sle_bwd_problem;
int serl_sle_bwd_multi(const serl_sle_bwd_problem* problems /*host*/, int num_problems, float* workspace, size_t workspace_bytes,
                       int N, int P, int C, int F, void* stream);
typedef struct serl_enc_finish_problem {      /* out = tanh(LayerNorm(z + bias) * scale + ln_bias), z from k-split partials or a small dense */
  const float* partials; int32_t S;           /* (S, rows, D) partial products of serl_tgemm_tf32, or NULL                      */
  const float* x; int32_t ld_x; const float* w; int32_t K;   /* else z = x (rows, K) @ w (K, D): the proprio Dense, encoding.py:65 */
  const float* bias; const float* ln_scale; const float* ln_bias;
  float* out; int32_t ld_out; float* xhat; float* rstd; int32_t D;   /* D <= 256                                                  */
} serl_enc_finish_problem;
int serl_enc_finish(const serl_enc_finish_problem* problems /*host*/, int num_problems, int rows, float eps, void* stream);
typedef struct serl_ln_bwd_problem {          /* LayerNorm + tanh backward; upstream gradient dt (+ dt2), or dq[row] * head_w[group][d] */
  const float* dt; int32_t ld_dt; const float* dt2; int32_t ld_dt2; const float* dq; const float* head_w; int64_t head_w_stride;
  const float* t; int32_t ld_t; const float* xhat; const float* rstd; const float* scale; int32_t rows_per_group; int64_t group_stride;
  float* dz; float* dy; int32_t R, D;
  int32_t dt_parts; int64_t dt_part_stride;   /* > 1: dt is the sum of dt_parts arrays (ensemble partials of serl_tgemm_tf32's PARTIAL epilogue) */
} serl_ln_bwd_problem;
int serl_layernorm_tanh_bwd_multi(const serl_ln_bwd_problem* problems /*host*/, int num_problems, void* stream);
/* The backward of a masked LayerNorm epilogue: dz of row r of problem i *= masks[i][(r % mask_rows) * D + d] ? inv_keep : 0. */
int serl_layernorm_tanh_bwd_multi_masked(const serl_ln_bwd_problem* problems /*host*/, int num_problems, const uint8_t* const* masks /*host*/,
                                         int mask_rows, float inv_keep, void* stream);
#define SERL_SMALL_GRAD_MAX_JOBS 12
#define SERL_SMALL_GRAD_COLSUM 0              /* out_a[g][d] = sum_r x[g*rows + r][d]                     (bias gradients)         */
#define SERL_SMALL_GRAD_LN 1                  /* out_a = sum_r x*y (scale), out_b = sum_r x (bias)        (x = dy, y = xhat)        */
#define SERL_SMALL_GRAD_HEAD 2                /* out_a[g][d] = sum_r x[r][d] * y[r], out_b[g] = sum_r y[r] (x = h, y = dq: value head) */
typedef struct serl_small_grad_job {
  int32_t kind; const float* x; int64_t ld_x; const float* y; int64_t ld_y; float* out_a; float* out_b; int32_t groups, rows, D;
} serl_small_grad_job;
int serl_small_grads(const serl_small_grad_job* jobs /*host*/, int num_jobs, void* stream);

/* SpatialLearnedEmbeddings (vision/resnet_v1.py:81-116) + Dropout (resnet_v1.py:352) */
int serl_sle_fwd(const float* feat, const float* kernel, const uint8_t* keep_mask, float keep, float* out,
                 int N, int P, int C, int F, int ld_out, void* stream);
int serl_sle_bwd_kernel_grad(const float* feat, const float* dout, float* dkernel, float* workspace, size_t workspace_bytes,
                             int N, int P, int C, int F, int ld_dout, void* stream);
/* LayerNorm(eps, fast variance) + tanh, rows grouped for vmapped (ensemble) parameters (networks/mlp.py:26-31) */
int serl_layernorm_tanh_fwd(const float* z, int ld_z, const float* scale, const float* bias, int rows_per_group, int group_stride,
                            float* out, int ld_out, float* xhat, float* rstd, int R, int D, float eps, void* stream);
int serl_layernorm_tanh_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* xhat, const float* rstd,
                            const float* scale, int rows_per_group, int group_stride, float* dz, float* dy,
                            float* dscale, float* dbias, int R, int D, void* stream);
int serl_layernorm_param_grad(const float* dy, const float* xhat, float* dscale, float* dbias, int rows_per_group, int R, int D,
                              void* stream);   /* dscale/dbias half of serl_layernorm_tanh_bwd (when it was called with NULLs) */
/* MLP layer activations (networks/mlp.py:10-32, flax.linen names): leaky_relu slope 0.01, gelu approximate=True */
#define SERL_ACT_TANH 0
#define SERL_ACT_RELU 1
#define SERL_ACT_SWISH 2          /* = silu */
#define SERL_ACT_LEAKY_RELU 3
#define SERL_ACT_GELU 4
/* [LayerNorm +] activation, the general form of serl_layernorm_tanh_fwd / _bwd (layer_norm = 0: out = act(z), scale / bias /
 * xhat / rstd unused).  The backward needs the pre-activation: tanh reads its output t; the other activations recompute it
 * from xhat / scale / bias with LayerNorm and read `pre` (the forward's z, row stride ld_pre) without.  With LayerNorm dy is
 * written for serl_layernorm_param_grad; without it dz = dy and dy is unused. */
int serl_layernorm_act_fwd(const float* z, int ld_z, const float* scale, const float* bias, int rows_per_group, int group_stride,
                           float* out, int ld_out, float* xhat, float* rstd, int R, int D, float eps, int act, int layer_norm,
                           void* stream);
int serl_layernorm_act_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* pre, int ld_pre, const float* xhat,
                           const float* rstd, const float* scale, const float* bias, int rows_per_group, int group_stride,
                           float* dz, float* dy, int R, int D, int act, int layer_norm, void* stream);
/* The same layers with the MLP's Dropout ahead of the LayerNorm / activation (networks/mlp.py:26-31): z' = mask ? z * inv_keep : 0,
 * mask (R, D) keep bytes from serl_dropout_mask_fill, inv_keep = 1 / (1 - dropout_rate).  Without LayerNorm z' is written back to
 * z, so the backward's `pre` is the activation's real input.  The backward multiplies dz by mask * inv_keep. */
int serl_ln_act_dropout_fwd(float* z, int ld_z, const float* scale, const float* bias, int rows_per_group, int group_stride,
                            const uint8_t* mask, float inv_keep, float* out, int ld_out, float* xhat, float* rstd, int R, int D, float eps,
                            int act, int layer_norm, void* stream);
int serl_ln_act_dropout_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* pre, int ld_pre, const float* xhat,
                            const float* rstd, const float* scale, const float* bias, int rows_per_group, int group_stride,
                            const uint8_t* mask, float inv_keep, float* dz, float* dy, int R, int D, int act, int layer_norm, void* stream);
/* The two above with mask row period mask_rows: row r reads mask row r % mask_rows, so an ensemble's E*B member-major rows share
 * one (B, D) mask (mask_rows = B; flax's nn.vmap broadcasts the dropout rng over the members, actor_critic_nets.py:156-164). */
int serl_ln_act_dropout_rows_fwd(float* z, int ld_z, const float* scale, const float* bias, int rows_per_group, int group_stride,
                                 const uint8_t* mask, int mask_rows, float inv_keep, float* out, int ld_out, float* xhat, float* rstd,
                                 int R, int D, float eps, int act, int layer_norm, void* stream);
int serl_ln_act_dropout_rows_bwd(const float* dt, int ld_dt, const float* t, int ld_t, const float* pre, int ld_pre, const float* xhat,
                                 const float* rstd, const float* scale, const float* bias, int rows_per_group, int group_stride,
                                 const uint8_t* mask, int mask_rows, float inv_keep, float* dz, float* dy, int R, int D, int act,
                                 int layer_norm, void* stream);
int serl_colsum_f32(const float* x, float* out, int groups, int rows, int D, long long ld, int accumulate, void* stream);
int serl_copy2d_f32(const float* src, long long ld_src, float* dst, long long ld_dst, int R, int D, void* stream);
int serl_fill_f32(float* x, float v, int n, void* stream);

/* ---- SAC losses (agents/continuous/sac.py:118-234, networks/actor_critic_nets.py:230-272) -------- */
int serl_tanh_gaussian_fwd(const float* mu, const float* log_std, const float* eps, float std_min, float std_max,
                           float* act, int ld_act, float* logp, float* u_out, float* std_out, int B, int A,
                           int deterministic, void* stream);
int serl_critic_loss(const float* q, const float* q_next, const int32_t* sub, int n_sub, const float* rewards,
                     const float* masks, const float* logp_next, const float* lagrange, int backup_entropy, float gamma,
                     float grad_scale, float* target_q, float* dq, float* info /*3*/, int E, int B, void* stream);
/* serl_critic_loss with importance weights w (B) (prioritized replay): loss = sum_{e,b} w_b (Q - y)^2 / (E*B),
 * dQ = 2 w_b (Q - y) / (E*B) * grad_scale, and delta (B) = the row's TD error (sum_e |Q[e,b] - y_b|, e ascending) / E.
 * w = 1 reproduces serl_critic_loss's target_q, dQ and info bit for bit. */
int serl_critic_loss_weighted(const float* q, const float* q_next, const int32_t* sub, int n_sub, const float* rewards,
                              const float* masks, const float* logp_next, const float* lagrange, int backup_entropy, float gamma,
                              float grad_scale, const float* w, float* target_q, float* dq, float* delta, float* info /*3*/, int E,
                              int B, void* stream);
int serl_actor_loss(const float* q, const float* logp, const float* lagrange, const float* da, int ld_da, const float* act,
                    int ld_act, const float* std, const float* log_std, const float* eps, float std_min, float std_max,
                    float grad_scale, float* dmu, float* dlogstd, float* info /*3*/, int E, int B, int A, void* stream);
/* Policy std parameterisations (networks/actor_critic_nets.py:190-210), then clip(std, std_min, std_max):
 *   EXP:      std = exp(x),      x = Dense_1 output (row stride A)
 *   SOFTPLUS: std = softplus(x), x = Dense_1 output (row stride A);  d x = d std * sigmoid(x)
 *   UNIFORM:  std = exp(x),      x = the (A,) log_stds leaf, broadcast to every row (row stride 0): the actor-loss kernel writes
 *             the per-row gradient (B, A) and the caller sums its columns into the leaf's gradient.
 *   FIXED:    std = x,           x = a constant (A,) device vector (Policy's fixed_std), row stride 0: no parameter, so the BC loss
 *             writes no std gradient (dx may be NULL).  serl_tanh_gaussian_fwd_std and serl_bc_loss_std take it; the SAC actor
 *             loss does not.
 * serl_tanh_gaussian_fwd / serl_actor_loss are the EXP forms with ld_x = A. */
#define SERL_STD_EXP 0
#define SERL_STD_SOFTPLUS 1
#define SERL_STD_UNIFORM 2
#define SERL_STD_FIXED 4      /* 3 is not assigned */
int serl_tanh_gaussian_fwd_std(const float* mu, const float* x, int ld_x, int std_param, const float* eps, float std_min, float std_max,
                               float* act, int ld_act, float* logp, float* u_out, float* std_out, int B, int A,
                               int deterministic, void* stream);
int serl_actor_loss_std(const float* q, const float* logp, const float* lagrange, const float* da, int ld_da, const float* act,
                        int ld_act, const float* std, const float* x, int ld_x, int std_param, const float* eps, float std_min,
                        float std_max, float grad_scale, float* dmu, float* dx, float* info /*3*/, int E, int B, int A, void* stream);
/* Behaviour cloning (agents/continuous/bc.py:36-76, launcher policy utils/launcher.py:26-47: Dense -> tanh, no LayerNorm):
 * element-wise tanh forward / backward, and loss = -mean_b log N(a_b; mu_b, diag(clip(exp(log_std_b))^2)) with its gradients
 * w.r.t. mu / log_std (scaled by grad_scale / B) and info = {actor_loss, mse} * grad_scale. */
int serl_tanh_fwd(const float* z, float* out, int n, void* stream);
int serl_tanh_bwd(const float* dt, const float* t, float* dz, int n, void* stream);
int serl_bc_loss(const float* mu, const float* log_std, const float* actions, float std_min, float std_max, float grad_scale,
                 float* dmu, float* dlogstd, float* info /*2*/, int B, int A, void* stream);
/* serl_bc_loss for every std head (SERL_STD_*: x is the head's output with row stride ld_x, 0 exactly for "uniform" / "fixed") and with
 * tanh_squash != 0 the tanh-squashed Gaussian: log_prob(a) = N(atanh a; mu, std) - sum 2 (log 2 - u - softplus(-2u)), u = atanh a,
 * mse against the mode tanh(mu).  dx = d loss / d x per row (the "uniform" leaf gradient is its column sum).  A std exactly on a
 * clip bound passes no gradient.  <exp, no squash> is serl_bc_loss bit for bit. */
int serl_bc_loss_std(const float* mu, const float* x, int ld_x, int std_param, int tanh_squash, const float* actions, float std_min,
                     float std_max, float grad_scale, float* dmu, float* dx, float* info /*2*/, int B, int A, void* stream);
int serl_temperature_loss(const float* logp, const float* lagrange, float target_entropy, float grad_scale,
                          float* dlagrange, float* info /*1*/, int B, void* stream);

/* ---- forward-only passes of the agent's public API (agents/continuous/sac.py:33-116) ---- */
/* Multi-action critic, first layer (networks/actor_critic_nets.py:33-46: one Q per (state, candidate action)).  W0 of member e
 * is [W_enc; W_act] ((F + A) x H row-major); P (E, B, H) = enc @ W_enc + b0 comes from the GEMMs.  For every member e, state b
 * and candidate n (row r = (e*B + b)*N + n of z / out, E*B*N rows of H):
 *   z[r, :] = P[e, b, :] + sum_{k < A} a[b, n, k] * W_act[e][k, :]   (k ascending, fp32 fma)
 *   out[r, :] = act(LayerNorm_e(z[r, :]))  (layer_norm = 0: act(z)); scale / bias (E, H).
 * w_act: address of W_act[0] (row F of member 0's W0), member stride w_act_z floats.  1 <= A <= 32. */
int serl_critic_multi_action_fwd(const float* P, const float* actions, const float* w_act, long long w_act_z, const float* scale,
                                 const float* bias, float* z, float* out, int E, int B, int N, int A, int H, float eps, int act,
                                 int layer_norm, void* stream);
/* Log-probability of given actions x (B, A) under tanh(N(mu, diag(std^2))) (std: the clipped std), one thread per row, fixed
 * order over the A dimensions: u = atanh(x); logp = sum_i [-0.5 ((u-mu)/std)^2 - log std - 0.5 log 2pi]
 * - sum_i 2 (log 2 - u - softplus(-2u)).  No clipping of x: |x| = 1 gives an infinite u, as distrax's Tanh bijector does. */
int serl_tanh_normal_log_prob(const float* mu, const float* std, const float* x, float* logp, int B, int A, void* stream);
/* GeqLagrangeMultiplier (networks/lagrange.py:9-78): out[i] = softplus(lagrange) * (lhs[i] - rhs), or softplus(lagrange) for
 * every i when lhs is NULL. */
int serl_lagrange_penalty(const float* lagrange, const float* lhs, float rhs, float* out, int n, void* stream);

/* ---- binary reward classifier (networks/reward_classifier.py:16-28; train_step of the examples'
 *      train_reward_classifier.py, async_cable_route_drq: lines 121-137) ---------------------------------------------- */
/* z (R, D = 256): Dense output incl. bias.  mask (R, D) optional Dropout keep mask: z' = where(mask, z / keep, 0).  Then
 * h = relu(LayerNorm(z'; eps, fast variance) * scale + bias) and logit[r] = h[r] . w + b[0] (the Dense(1) head, w (D)).
 * h, xhat (R, D) and rstd (R) are optional saves for the backward pass. */
int serl_layernorm_relu_head_fwd(const float* z, const uint8_t* mask, float keep, const float* scale, const float* bias,
                                 const float* w, const float* b, float* h, float* xhat, float* rstd, float* logit,
                                 int R, int D, float eps, void* stream);
/* Backward of the above from dlogit (R): dh = dlogit (x) w, through relu, LayerNorm and the dropout mask.  dy (R, D) =
 * gradient w.r.t. the LayerNorm output (for its scale / bias gradients; optional), dz (R, D) = gradient w.r.t. z. */
int serl_layernorm_relu_head_bwd(const float* dlogit, const float* w, const float* h, const float* xhat, const float* rstd,
                                 const float* scale, const uint8_t* mask, float keep, float* dy, float* dz, int R, int D,
                                 void* stream);
/* loss = mean_b [max(x,0) - x y + log1p(exp(-|x|))] of logits_train, dlogit = (sigmoid(x) - y) * grad_scale / B,
 * accuracy = mean_b [(float)(sigmoid(logits_eval) >= 0.5) == y]; info = {loss, accuracy}.  One CTA, deterministic. */
int serl_bce_logits_loss(const float* logits_train, const float* logits_eval, const float* labels, float grad_scale,
                         float* dlogit, float* info /*2*/, int B, void* stream);
/* Dropout backward in place: dx = mask ? dx / keep : 0 (the SLE output gradient before serl_sle_bwd_multi when the pass
 * that produced it ran with dropout). */
int serl_dropout_bwd_f32(float* dx, const uint8_t* mask, float keep, int n, void* stream);

/* ---- VICE reward classifier (agents/continuous/vice.py:357-600; csrc/vice.cu) -------------------------------------------
 * draws: per camera c, keys[6c..6c+6) = (k0, k1, k_eps): lam[c] = uniform(k0), perm[c] (N) = permutation(k1, N) in `rounds`
 * sort rounds, eps[c] (N/2) = uniform(k_eps, (N/2,)).  N <= 2048, one CTA per camera. */
int serl_vice_draws(const uint32_t* keys, int ncams, int N, int rounds, float* lam, int* perm, float* eps, void* stream);
/* out rows [0, N) = lam f + (1 - lam) f[perm], rows [N, 3N/2) = eps mix[i] + (1 - eps) mix[N/2 + i]; (rows, D) per camera. */
int serl_vice_mix(const float* feats, long long in_stride, const float* lam, const int* perm, const float* eps, float* out,
                  long long out_stride, int ncams, int N, int D, void* stream);
/* smoothed-label mixup BCE of N logits with the last camera's lam / perm: info[0] = loss, dlogit = d loss / d logit * grad_scale */
int serl_vice_bce(const float* logits, const float* lam, const int* perm, float grad_scale, float* dlogit, float* info, int N,
                  void* stream);
/* [dropout] -> LayerNorm -> act (tanh | leaky_relu) [-> Dense(1)] on rows [R0, R), D 256 | 512; tangent = 1: tangent rows whose
 * primal partner is r - pair_off (zdot is replaced by its masked value, y gets ydot). */
int serl_vice_ln_act_fwd(float* z, int ld_z, const float* pre_bias, const uint8_t* mask, int ld_mask, float keep, const float* scale,
                         const float* bias, float* y, int ld_y, float* xhat, float* rstd, const float* head_w, const float* head_b,
                         float* logit, int R0, int R, int pair_off, int tangent, int D, int act, float eps, void* stream);
/* reverse of the above over primal rows [R0, R); rows >= R - R_pair also carry their tangent row r + R_pair (second order). */
int serl_vice_ln_act_bwd(const float* dy, int ld_dy, const float* dlogit, float dlogit_const, const float* head_w, float tan_seed,
                         const float* xhat, const float* rstd, const float* z, int ld_z, const uint8_t* mask, int ld_mask, float keep,
                         const float* scale, const float* bias, const float* y, int ld_y, float* dz, int ld_dz, float* dscale_rows,
                         float* dbias_rows, float* dw_rows, int R0, int R, int R_pair, int D, int act, void* stream);
/* dx[r, p, c] = sum_f ds[r, c*8 + f] kernel[p, c, f] (SpatialLearnedEmbeddings input gradient) */
int serl_vice_sle_input_grad(const float* ds, int ld_ds, const float* kernel, float* dx, int R, int P, int C, void* stream);
/* keep masks bernoulli(fold_in(key, fold), keep, (rows, n)), or one (n,) row repeated on every row (broadcast = 1) */
int serl_vice_mask_fill(const uint32_t* key, int fold, float keep, uint8_t* out, int rows, int n, int broadcast, void* stream);
/* per (camera, row) |g| = sqrt(sum(g^2 + 1e-6)) -> norms, v = coef (|g| - 1) / |g| g */
int serl_vice_gp_rows(const float* g, long long g_stride, float* v, long long v_stride, float coef, float* norms, int ncams, int B,
                      int D, void* stream);
/* info[1] = s mean |g|, info[2] = s mean((|g| - 1)^2), info[3] = info[0] + gp_weight info[2]; s = info_scale (1/world under data
 * parallelism, as serl_vice_bce scales info[0]: one SUM all-reduce of gradient + infos gives the mean) */
int serl_vice_gp_finish(const float* norms, int M, float gp_weight, float info_scale, float* info, void* stream);
/* rewards = (sigmoid(logit) >= 0.5) in fp32 (threshold = 0: sigmoid(logit)), mean_out (optional) = mean(rewards) */
int serl_vice_reward(const float* logit, float* rewards, float* mean_out, int B, int threshold, void* stream);

/* Stride-1 3x3 convolution + GroupNorm(4 groups) [+ residual] [+ ReLU] in one kernel (vision/resnet_v1.py:129-156: the
   ResNetBlock body after / including each 3x3 conv).  An image's fp32 accumulators stay on chip until its statistics are
   complete, so no raw conv output and no normalisation pass ever touch HBM:
       y = [relu]( GN(conv3x3(x, w); gamma, beta) [+ res | + GN_res(res)] )
   x (N,H,W,Ci), res / y (N,H,W,Co) 16-bit NHWC; w packed [Co][9*Ci] K-major ((kh,kw,ci) order); out_f32 (N,H,W,Co) replaces y
   for the last block.  res_stats (N,4,2) + res_gamma/res_beta: the residual is a RAW projection-conv output whose own
   GroupNorm is applied on the fly.  Shapes: the four ResNet-10 block shapes at 128x128 input (H=W in {32,16,8,4}, Ci=Co). */
typedef struct serl_conv3x3_res_desc {
  const void* x; const void* w; void* y; float* out_f32; const void* res;
  const float* gamma; const float* beta;
  const float* res_stats; const float* res_gamma; const float* res_beta;
  int32_t* error;
  int32_t N, H, W, Ci, Co, relu, fmt;
  float eps;
} serl_conv3x3_res_desc;
int serl_conv3x3_res_h16(const serl_conv3x3_res_desc* d, void* stream);

/* Head of ResNetBlock_1..3 (vision/resnet_v1.py:139-154), GroupNorm fused into the convs: x (N,2Wo,2Wo,Ci) ->
       y = relu(GN(conv3x3 stride 2 SAME(x, w); gamma, beta))            (N,Wo,Wo,Co), Co = 2 Ci
       r = GN(conv1x1 stride 2(x, w_proj); gamma_proj, beta_proj)        (N,Wo,Wo,Co)   (the block's residual branch, normalised)
   w packed [Co][9*Ci], w_proj [Co][Ci], K-major 16-bit.  Wo in {16, 8, 4} (Co = 128, 256, 512). */
typedef struct serl_conv3x3s2_res_desc {
  const void* x; const void* w; const void* w_proj; void* y; void* r;
  const float* gamma; const float* beta; const float* gamma_proj; const float* beta_proj;
  int32_t* error;
  int32_t N, Wo, Ci, Co, fmt;
  float eps;
} serl_conv3x3s2_res_desc;
int serl_conv3x3s2_res_h16(const serl_conv3x3s2_res_desc* d, void* stream);

/* ---- optimizer (common/common.py:124-168, common/optimizers.py:6-56) --------------------------- */
typedef struct serl_adam_desc {
  float* params; float* target; float* m; float* v; const float* grad;
  int32_t n;
  int32_t seg_end[3];        /* flat layout: group 0 = critic tx, 1 = actor tx, 2 = temperature tx */
  int32_t live[3];           /* network updated this call (else its gradient is zero)             */
  int32_t* counts;           /* device int32[3]: optax counts, incremented by the call            */
  float lr[3]; int32_t warmup[3];
  float b1, b2, eps, tau;
  int32_t polyak;            /* soft target update after the step                                 */
  float* lr_out;             /* optional device float[3]                                          */
  /* Flat-buffer extras (serl_b200/params.py): `n` counts parameter slots only; indices in
     [seg_end[0], seg_end[0] + gap) hold no parameter (info scalars of the gradient buffer) and are
     skipped.  Leaves in [aux_lo, aux_hi) are updated by TWO transforms (reference
     common/common.py:136-168: the proprio encoder gets gradients from the critic loss AND from the
     actor loss, common/encoding.py:48-70): group 0 through grad/m/v[i] and group 1 (the actor tx)
     through grad/m/v[i + aux_off]; the two updates are summed before they are applied.            */
  int32_t gap, aux_lo, aux_hi, aux_off;
} serl_adam_desc;
int serl_adam_polyak(const serl_adam_desc* d, void* stream);

/* Per-tx options of common/optimizers.py:6-56 beyond learning rate and linear warm-up.
   clip[g] > 0: optax.clip_by_global_norm(clip[g]) ahead of tx g's Adam - the update sees g unchanged if
   norm < clip, else (g / norm) * clip, with `norm` read from norms[g] (serl_grad_global_norms).
   decay_steps[g] > 0: warmup_cosine_decay_schedule(0, lr, warmup, decay_steps, end_value=0) instead of the
   linear warm-up then constant; needs decay_steps > warmup.                                              */
typedef struct serl_adam_opts {
  float clip[3];             /* <= 0: no clipping                                                  */
  int32_t decay_steps[3];    /* <= 0: no cosine decay                                              */
  const float* norms;        /* device float[3]; required when some live tx clips                  */
} serl_adam_opts;
#define SERL_GRAD_NORM_CTAS 256   /* fixed grid of the norm pass: the summation order never depends on the device */
/* norms[g] = sqrt(sum of grad^2 over what tx g sees), for every live g with want[g] != 0 (else 0):
   g = 0: [0, seg_end[0]); g = 1: [seg_end[0] + gap, seg_end[1]) and the actor-tx twin slots
   [aux_lo + aux_off, aux_hi + aux_off); g = 2: [seg_end[1], seg_end[2]).  The info gap is in no norm.
   Fixed-order per-CTA float64 partials in `partials` (SERL_GRAD_NORM_CTAS * 3 doubles), then a
   fixed-order final sum: bitwise reproducible, no atomics.  Two launches.                               */
int serl_grad_global_norms(const serl_adam_desc* d, const int32_t want[3], double* partials, float* norms, void* stream);
/* serl_adam_polyak with the options above (the descriptor's lr / warmup / counts keep their meaning).    */
int serl_adam_polyak_opts(const serl_adam_desc* d, const serl_adam_opts* o, void* stream);

/* ---- DrQ "small" encoder (small_conv.cu): 3x3 / stride-2 VALID convs, fp32 CUDA-core implicit GEMMs ------
   Layouts: x (N,H,W,Ci) NHWC, uint8 (scaled by 1/255) when x_is_u8, else fp32; w (3,3,Ci,Co) HWIO; b (Co);
   y / dz (N,Ho,Wo,Co) with Ho = (H-3)/2+1.  Co % 4 == 0.  No atomics: bitwise reproducible.
   tc == 0: CUDA-core fp32 FMAs (the fp32 build); tc != 0: tensor cores, wgmma tf32 with 3xTF32 splitting
   (fp32-class products; the fp16 / bf16 builds).                                                          */
/* y = relu(conv(x, w) + b). */
int serl_sconv_fwd(const void* x, int x_is_u8, const float* w, const float* b, float* y, int N, int H, int W, int Ci, int Co,
                   int tc, void* stream);
/* dx = conv_transpose(dz, w) * (x > 0): the previous layer's pre-activation gradient, x its (post-ReLU) output.
   Ci % 4 == 0. */
int serl_sconv_dgrad(const float* dz, const float* w, const float* x, float* dx, int N, int H, int W, int Ci, int Co, int tc,
                     void* stream);
/* dw = sum over pixels of x-patch (x) dz, db = sum over pixels of dz: split-K over the N*Ho*Wo pixels in about
   `splits` fixed ranges (partials in workspace: ceil(K / ceil(K / splits, 16)) * (9Ci+1) * Co floats), then a
   fixed-order reduction.  Two launches. */
int serl_sconv_wgrad(const void* x, int x_is_u8, const float* dz, float* dw, float* db, float* workspace, long long workspace_bytes,
                     int splits, int N, int H, int W, int Ci, int Co, int tc, void* stream);
/* out[n][c] = mean over P positions of y[n][p][c]. */
int serl_sconv_mean_fwd(const float* y, float* out, int N, int P, int C, void* stream);
/* dz[n][p][c] = dout[n*ld + c] / P where y[n][p][c] > 0, else 0 (mean backward through the last ReLU). */
int serl_sconv_mean_bwd(const float* dout, int ld, const float* y, float* dz, int N, int P, int C, void* stream);

/* ---- DrQ "resnet" encoder training (resnet_train.cu): a trainable ResNet-10's backward and its 16-bit-build convs ----
   Convs: x (N,H,W,Ci) fp32 NHWC with Ci % 4 == 0; w (kh,kw,Cw,Co) HWIO with Cw <= Ci (Cw < Ci: the input's extra channels
   are zero padding, as in the stem's 4-channel copy); dz / y (N,Ho,Wo,Co), Ho = (H + pad_lo + pad_hi - kh) / stride + 1;
   Co % 4 == 0.  Implicit GEMMs over a 4-stage cp.async ring.  tc == 0: CUDA-core fp32 FMAs (the fp32 build); tc != 0:
   wgmma tf32 with 3xTF32 splitting (fp32-class products; the fp16 / bf16 builds).  No atomics: bitwise reproducible.     */
/* y = conv(x, w) (no bias). */
int serl_rconv_fwd(const float* x, const float* w, float* y, int N, int H, int W, int Ci, int Cw, int Co, int kh, int kw, int stride,
                   int pad_lo, int pad_hi, int tc, void* stream);
/* dx (+)= conv_transpose(dz, w) (accumulate != 0: added to dx), per parity class of (iy % stride, ix % stride) over its
   taps only.  H % stride == W % stride == 0. */
int serl_rconv_dgrad(const float* dz, const float* w, float* dx, int N, int H, int W, int Ci, int Co, int kh, int kw, int stride,
                     int pad_lo, int pad_hi, int accumulate, int tc, void* stream);
/* *floats = the split-K partials serl_rconv_wgrad needs for a shape. */
int serl_rconv_wgrad_workspace(int N, int H, int W, int Ci, int Co, int kh, int kw, int stride, int pad_lo, int pad_hi,
                               long long* floats);
/* dw (kh,kw,Cw,Co) = sum over pixels of x-patch (x) dz: fixed split-K ranges (a function of the shape), then a
   fixed-order reduction.  Two launches. */
int serl_rconv_wgrad(const float* x, const float* dz, float* dw, float* workspace, long long workspace_bytes, int N, int H, int W,
                     int Ci, int Cw, int Co, int kh, int kw, int stride, int pad_lo, int pad_hi, int tc, void* stream);
/* y (N,H,W,4) fp32 = ((x / 255 - mean) / std, 0) of x (N,H,W,3) uint8 (ImageNet mean / std, as serl_conv2d_nhwc_f32). */
int serl_rconv_stem_prep(const uint8_t* x, float* y, int N, int H, int W, void* stream);
/* y (N,H,W,Cp) fp32, Cp = 4 * ceil(Ci / 4), of a frame stack x (N,H,W,Ci) uint8 (Ci = 3T): channel c normalised with the
 * statistics of channel c mod 3, channels Ci .. Cp-1 zero. */
int serl_rconv_stem_prep_stacked(const uint8_t* x, float* y, int N, int H, int W, int Ci, void* stream);
/* Backward of serl_groupnorm_nhwc_f32 (y = [relu](GN(x) [+ residual])): dx, dres = the residual's gradient (nullable),
   dscale / dbias (C).  y: the forward's output (its > 0 is the ReLU mask; relu != 0).  workspace: 2 N C + 2 N groups
   floats.  Statistics recomputed as the forward computes them; fixed-order sums.  Three launches. */
int serl_groupnorm_bwd_nhwc(const float* x, const float* y, const float* dy, const float* scale, float* dx, float* dres,
                            float* dscale, float* dbias, float* workspace, int N, int HW, int C, int groups, float eps, int relu,
                            void* stream);
/* Backward of serl_maxpool3x3s2_nhwc_f32 as a gather from the saved input x: each window's gradient goes to its first
   maximal element in row-major window order. */
int serl_maxpool3x3s2_bwd_nhwc(const float* x, const float* dy, float* dx, int N, int H, int W, int C, void* stream);

/* ---- image augmentations (augment.cu): vision/data_augmentations.py on n NHWC images -------------------------------------
   keys: uint32 pairs, one per image (jax.vmap's form) unless a function says otherwise; every draw, decision and key split is
   derived on the device (threefry2x32), so no call reads anything back to the host.  One launch per call.                  */
/* dst = the edge-padded crop of src at randint(key_i, (2,), 0, 2 padding + 1) per image: any element type (pix_bytes bytes per
   pixel).  split_n > 0 (== n): key_i = split(keys[0:2], n)[i] (batched_random_crop); split_n == 0: keys holds n keys. */
int serl_aug_crop(const void* src, void* dst, const uint32_t* keys, int split_n, int n, int H, int W, int pix_bytes, int padding,
                  void* stream);
/* color_transform's options: op k = brightness, contrast, saturation, hue draws uniform(lo[k], hi[k]) (the float32 bounds jax
   builds from the strengths); bit k of `enabled`: that strength is > 0. */
typedef struct {
  float lo[4], hi[4];
  int enabled, shuffle;
  float apply_prob, jitter_prob, gray_prob;
} serl_color_desc;
#define SERL_COLOR_DRAWS 12          /* per image: apply, jitter, grayscale, order[4], drawn parameter of op 0..3, 0 */
/* dst = color_transform(src) per image, float32 (n, H, W, 3); draws (nullable) = SERL_COLOR_DRAWS floats per image. */
int serl_aug_color(const float* src, float* dst, const uint32_t* keys, float* draws, int n, int H, int W, const serl_color_desc* desc,
                   void* stream);
#define SERL_BLUR_MAX_RADIUS 96      /* (32 + 2 radius) rows of 256 floats of shared memory per CTA */
/* dst = gaussian_blur(src) per image, float32 (n, H, W, C), taps of radius `radius`; draws (nullable) = apply, sigma per image. */
int serl_aug_blur(const float* src, float* dst, const uint32_t* keys, float* draws, int n, int H, int W, int C, int radius,
                  float sigma_min, float sigma_max, float apply_prob, void* stream);
/* dst = random_flip(src) per image, float32 (n, H, W, C). */
int serl_aug_flip(const float* src, float* dst, const uint32_t* keys, int n, int H, int W, int C, void* stream);
/* dst = solarize(src) per image, float32 (n, H, W, C). */
int serl_aug_solarize(const float* src, float* dst, const uint32_t* keys, int n, int H, int W, int C, float threshold, float apply_prob,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SERL_B200_H_ */
