/*
 * rainbow_b200.h -- C ABI of the H100-native (sm_90a) Rainbow learner hot path.
 *
 * The reference (Kaixhin/Rainbow @ 1745b184) has no FFI/plugin layer: its hot
 * path is Python (memory.py, agent.py, model.py).  This header is the drop-in
 * boundary a maintainer of the reference would bind with ctypes/cffi from
 * those three files (INTEGRATION.md shows the stubs).  Each entry point names
 * the reference lines it replaces.
 *
 * Conventions
 *   - C linkage, plain pointers and sizes, no torch / C++ types.
 *   - Every pointer is a DEVICE pointer owned by the caller (e.g.
 *     tensor.data_ptr()) unless a parameter is documented "host".
 *   - Every call enqueues work on `stream` (a cudaStream_t passed as void*)
 *     and returns immediately; nothing synchronises, allocates or frees.
 *     All calls are CUDA-graph capturable.
 *   - Return value: RB_OK (0) or a negative errno-style code; the text of the
 *     last error of the calling thread is available from rb_last_error().
 *   - Device-side conditions (rejected sample batch, bad index) are reported
 *     through the `status` words written by the kernel, never by a sync.
 *
 * Data layout in HBM (structure of arrays; reference Transition_dtype is an
 * array of 7069-byte structs, memory.py:7):
 *   tree         float32[tree_start + size]   heap order, root at tree[0],
 *                children 2i+1 / 2i+2, leaves from tree_start = 2^ceil(log2 size)-1
 *                (memory.py:17-18).  For 128-byte-aligned level loads allocate
 *                one pad float in front so that (tree - 1) is 128 B aligned.
 *   frames       uint8[size][7056]            last frame of each transition
 *   timestep     int32[size]                  in-episode step (0 = episode start)
 *   action       int32[size]
 *   reward       float32[size]
 *   nonterminal  uint8[size]
 *   ring_state   int64[5]  {head (next write slot), full (0/1), t_episode, appended_total, launch ticket of
 *                          rb_append / rb_append_batch (zero between launches)}
 *   running_max  float32[1] largest exponentiated priority seen (memory.py:20,48)
 *   rng_counter  uint64[1]  Philox draw counter, advanced by the kernels themselves
 *                           (so a replayed CUDA graph draws fresh numbers)
 */
#ifndef RAINBOW_B200_H
#define RAINBOW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RB_ABI_VERSION 3

#define RB_OK 0
#define RB_ERR_INVAL (-22)       /* bad argument (EINVAL) */
#define RB_ERR_RANGE (-34)       /* size outside supported range (ERANGE) */
#define RB_ERR_CUDA (-5)         /* CUDA runtime reported an error (EIO) */

#define RB_FRAME_BYTES 7056      /* 84*84 */
#define RB_MAX_WINDOW 64         /* history + multi_step */
#define RB_MAX_ATOMS 128
#define RB_MAX_NOISY_LAYERS 8
#define RB_MAX_PEERS 8           /* ranks of one NVLink domain handled by rb_peer_clip_adam */
#define RB_APPEND_BATCH 8        /* transitions per rb_append_batch launch */
#define RB_NONTERMINAL_FINAL 2   /* nonterminal byte of a final-observation record (rb_append_batch_trunc) */
#define RB_MAX_SHIFT_PAD 16      /* largest pad of rb_gather_shift */
#define RB_MAX_AUG_COPIES 8      /* most copies of a state (M) or next state (K) in rb_gather_aug */
#define RB_MAX_RESET_SEGMENTS 32 /* most parameter tensors one rb_param_reset call covers */
#define RB_MAX_ANNEAL_STEPS 65536 /* longest horizon schedule (T) of rb_horizon_advance */
#define RB_MAX_REDO_LAYERS 8     /* most scored layers of rb_redo_mask / rb_redo_recycle */
#define RB_MAX_REDO_BLOCKS 4     /* most incoming, and most outgoing, parameter blocks of one scored layer */
#define RB_REDO_RECORD_WORDS (2 + 2 * RB_MAX_REDO_LAYERS) /* int64 words of rb_redo_mask's record */

/* status words written by rb_tree_sample (int32[4]): status[0] = 1 if the batch now in the output buffers passed the
 * whole-batch validity test (memory.py:131), 0 otherwise; status[1] = draws used; status[2] = number of device-RNG
 * batches so far that were still invalid after max_attempts draws (cumulative; the caller zero-initialises it once).
 * A rejected batch has all its importance weights set to 0 (its loss gradient is exactly zero), and status[0] can be
 * handed as the `gate` of rb_clip_adam / rb_tree_update so neither the parameters nor the priorities are touched --
 * the device-side counterpart of the reference's redraw-until-valid loop (memory.py:128-132), without a host sync. */

typedef void* rb_stream_t; /* cudaStream_t */

/* kernel ids for the optional timing hooks (rb_profile_*) */
enum {
  RB_K_TREE_UPDATE = 0, RB_K_TREE_FIND, RB_K_TREE_SAMPLE, RB_K_GATHER, RB_K_ITER_STATES, RB_K_APPEND, RB_K_C51,
  RB_K_NOISY_RESAMPLE, RB_K_NOISY_COMPOSE, RB_K_SQNORM, RB_K_CLIP_ADAM, RB_K_HEAD_FC1, RB_K_HEAD_FC2, RB_K_HEAD_LOGITS,
  RB_K_HEAD_WGRAD2, RB_K_HEAD_DH, RB_K_HEAD_BWD1, RB_K_NOISE_FACTORS, RB_K_C51_DUELING, RB_K_BIAS_GRAD, RB_K_Q_VALUES,
  RB_K_HEAD_REDUCE1, RB_K_CONV_WGRAD, RB_K_HEAD_BWD1_WGRAD, RB_K_HEAD_BWD1_DX, RB_K_LEARN_STATS, RB_K_GATHER_SHIFT,
  RB_K_GATHER_AUG, RB_K_C51_DUELING_AVG, RB_K_TARGET_EMA, RB_K_PARAM_RESET, RB_KERNEL_COUNT
};

int rb_abi_version(void);
const char* rb_last_error(void);

/* Diagnostics (no reference counterpart): when enabled, every kernel launch is bracketed by CUDA events
 * on its stream (do not enable during CUDA-graph capture).  rb_profile_collect synchronises on the
 * recorded events of one kernel id, returns their summed duration and count, and clears them. */
int rb_profile_enable(int on);
int rb_profile_collect(int kernel_id, double* total_ms, int* launches);

/* memory.py:157-159 ReplayMemory.update_priorities -> :44-48 SegmentTree.update
 * (-> :28-33 _propagate -> :23-25 _update_nodes).
 * leaf[tree_idx[k]] = raw_priority[k]^omega (duplicates: last k wins), parents recomputed
 * level by level as fl32(left+right) up to the root, running_max = max(running_max, max_k leaf).
 * omega_is_applied != 0 means raw_priority already holds exponentiated values (SegmentTree.update).
 * status[0] is set to 1 if any tree_idx lies outside the leaf range (nothing is written for it).
 * gate (optional device int32, may be NULL): when *gate == 0 the launch does nothing (rejected sample batch). */
int rb_tree_update(float* tree, int64_t tree_start, int64_t size, const int64_t* tree_idx,
                   const float* raw_priority, float omega, int omega_is_applied, int B, float* running_max,
                   int32_t* status, const int32_t* gate, rb_stream_t stream);

/* memory.py:79-82 SegmentTree.find (-> :64-76 _retrieve): float64 residual against float32 nodes,
 * strict '>' goes right, child indices clipped to the last element on the leaf level. */
int rb_tree_find(const float* tree, int64_t tree_start, int64_t size, const double* values, int B, float* probs,
                 int64_t* data_idx, int64_t* tree_idx, rb_stream_t stream);

/* memory.py:148-154 ReplayMemory.sample head + :124-132 _get_samples_from_segments:
 * p_total = tree[0]; seg = fl32(p_total/B); v_k = seg*u_k + k*seg (float64); find; whole-batch
 * validity test (memory.py:131) with redraw; importance weights (count*p/p_total)^-beta / max.
 *   u01 != NULL : parity mode.  u01 is float64[u01_attempts][B] of unit uniforms (what
 *                 RandomState.uniform consumes); attempt a uses row a; at most u01_attempts tries.
 *   u01 == NULL : device Philox4x32-10 keyed by `seed`, counter *rng_counter (advanced by the
 *                 number of draws); at most max_attempts tries.
 * beta_dev (optional, may be NULL) overrides `beta` with a device scalar (graph replay). */
int rb_tree_sample(const float* tree, int64_t tree_start, int64_t size, const int64_t* ring_state, int n,
                   int history, const double* u01, int u01_attempts, uint64_t seed, uint64_t* rng_counter, int B,
                   float beta, const float* beta_dev, int max_attempts, float* probs, int64_t* data_idx,
                   int64_t* tree_idx, float* weights, int32_t* status, rb_stream_t stream);

/* memory.py:111-121 _get_transitions + :134-145 (tail of _get_samples_from_segments) + :85-86 get:
 * window of history+n records around each data_idx (indices mod size), episode-boundary blanking,
 * states = u8/255 [B,history,84,84], next_states (window shifted by n), actions int64[B],
 * returns = sum_k gamma_pow[k]*reward[B], nonterminals float32[B] (of the last window record). */
int rb_gather(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
              const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n,
              const float* gamma_pow, float* states, float* next_states, int64_t* actions, float* returns,
              float* nonterminals, rb_stream_t stream);

/* rb_gather with random-shift augmentation of the observations (DrQ, Kostrikov et al. 2020; no reference counterpart):
 * every observation -- each sample's state and its next state -- is edge-padded by `pad` pixels and cropped back to
 * 84 x 84 at its own integer offset (oy, ox), each uniform in [0, 2 pad], the same for all of its history frames:
 *   out[c][y][x] = in[c][clamp(y + oy - pad, 0, 83)][clamp(x + ox - pad, 0, 83)]
 * where `in` is what rb_gather writes (blanking included).  actions, returns and nonterminals are rb_gather's, bitwise.
 * Offsets: one Philox4x32-10 call per sample b with key `seed` and counter (c_lo, c_hi, b, 0x53484654), c = *rng_counter
 * as the kernel reads it (rb_tree_sample has just advanced it, so each batch and each graph replay draws afresh; this call
 * does not advance it); words x, y give the state's (oy, ox), z, w the next state's; offset = (word * (2 pad + 1)) >> 32.
 * shifts (required): int32[2][B][2] (side: 0 = state, 1 = next state; sample; (oy, ox)) receives the offsets used.
 * RB_ERR_RANGE: pad outside [1, RB_MAX_SHIFT_PAD], plus every check of rb_gather; RB_ERR_INVAL: a NULL pointer.  A refused
 * call launches nothing. */
int rb_gather_shift(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                    const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n,
                    const float* gamma_pow, float* states, float* next_states, int64_t* actions, float* returns,
                    float* nonterminals, int pad, uint64_t seed, const uint64_t* rng_counter, int32_t* shifts,
                    rb_stream_t stream);

/* rb_gather_shift generalised to DrQ's K / M copies (Kostrikov et al. 2020, Algorithm 1) and SPR's intensity augmentation
 * (Schwarzer et al. 2021); no reference counterpart.  Every sample's state is written m_copies = M times and its next state
 * k_copies = K times, copy-major: states float32[M*B][history][84][84] (rows [jB, (j+1)B) hold copy j), next_states
 * float32[K*B][...] the same way.  Each copy of each observation has its own shift offset (as rb_gather_shift; none when
 * pad == 0) and its own intensity multiplier, the same for all of its history frames:
 *   out[c][y][x] = fl32(in[c][clamp(y + oy - pad, 0, 83)][clamp(x + ox - pad, 0, 83)] * mult)
 *   mult = fmaf(intensity, clamp(N(0, 1), -2, 2), 1)     (intensity == 0: mult = 1 and no multiply is done)
 * where `in` is what rb_gather writes.  actions, returns and nonterminals are rb_gather's, bitwise.
 * Draws, key `seed`, c = *rng_counter as the kernel reads it (not advanced by this call), for sample b and copy j:
 *   offsets    Philox4x32-10 counter (c_lo, c_hi, b, 0x53484654 + j): x, y -> the state's (oy, ox), z, w -> the next
 *              state's, offset = (word * (2 pad + 1)) >> 32 -- copy 0's are rb_gather_shift's;
 *   multiplier Philox4x32-10 counter (c_lo, c_hi, b, 0x494E5453 + j) through Box-Muller: the first normal of (x, y) is the
 *              state's, the first of (z, w) the next state's.
 * shifts int32[2][copies][B][2] and scales float32[2][copies][B] (side: 0 = state, 1 = next state; copy; sample), copies =
 * max(M, K), receive the draws (offsets 0 when pad == 0, multipliers 1 when intensity == 0); side 0 copies >= M and side 1
 * copies >= K are drawn but not applied.
 * RB_ERR_RANGE: pad outside [0, RB_MAX_SHIFT_PAD], intensity outside [0, 0.5] or not finite, m_copies or k_copies outside
 * [1, RB_MAX_AUG_COPIES], plus every check of rb_gather; RB_ERR_INVAL: a NULL pointer, or pad 0 with intensity 0 and
 * M = K = 1 (that is rb_gather).  A refused call launches nothing. */
int rb_gather_aug(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                  const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n,
                  const float* gamma_pow, float* states, float* next_states, int64_t* actions, float* returns,
                  float* nonterminals, int pad, float intensity, int m_copies, int k_copies, uint64_t seed,
                  const uint64_t* rng_counter, int32_t* shifts, float* scales, rb_stream_t stream);

/* An annealed update horizon (BBF, Schwarzer et al. 2023; no reference counterpart): one row per update step u of the
 * schedule, built on the host.  n = n_u (>= 1), gamma_n = fl32(gamma_u ** n_u), gamma_pow[k] = fl32(gamma_u ** k) for
 * k < n_u and 0 beyond.  A table holds T + 1 rows, u = 0 .. T. */
typedef struct rb_horizon {
  int32_t n;
  float gamma_n;
  float gamma_pow[RB_MAX_WINDOW];
} rb_horizon;

/* One thread: *current = table[min(*counter, T)] (a negative counter reads row 0), then *counter += 1 (int64, device).
 * The update graph's first node when the horizon is annealed; it has no profiling id (time it with events around the
 * launch).  RB_ERR_INVAL: a NULL pointer; RB_ERR_RANGE: T outside
 * [1, RB_MAX_ANNEAL_STEPS].  A refused call launches nothing. */
int rb_horizon_advance(const rb_horizon* table, int T, int64_t* counter, rb_horizon* current, rb_stream_t stream);

/* rb_gather, rb_gather_shift and rb_gather_aug with the horizon read from the device row *current (as
 * rb_horizon_advance left it) instead of the arguments n and gamma_pow.  n_max sizes the window: the replay must have
 * been sampled for n_max (rb_tree_sample with n = n_max), and the row's n is clamped into [1, n_max].  With n_t, gamma_pow
 * and gamma_n of the row, every output is bitwise what the fixed-horizon kernel writes with n = n_t and that gamma_pow,
 * except nonterminals, which come in discount form: fl32(nonterminal * gamma_n), i.e. gamma_n or +0.  A loss kernel
 * (rb_c51_*) launched on them with gamma_n = 1 computes what it computes on 0 / 1 nonterminals with the row's gamma_n.
 * The augmentation arguments select the kernel as the Python sampler does: pad 0, intensity 0 and M = K = 1 gathers like
 * rb_gather (rng_counter, shifts and scales may be NULL); pad > 0 with intensity 0 and M = K = 1 like rb_gather_shift
 * (shifts int32[2][B][2]; scales may be NULL); anything else like rb_gather_aug, with its layouts and its draws.
 * RB_ERR_RANGE: pad outside [0, RB_MAX_SHIFT_PAD], intensity outside [0, 0.5] or NaN, copies outside
 * [1, RB_MAX_AUG_COPIES], plus every check of rb_gather with n = n_max; RB_ERR_INVAL: a NULL pointer the selected kernel
 * needs.  A refused call launches nothing.  Profiled under the id of the gather it stands for (RB_K_GATHER,
 * RB_K_GATHER_SHIFT or RB_K_GATHER_AUG). */
int rb_gather_horizon(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                      const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n_max,
                      const rb_horizon* current, float* states, float* next_states, int64_t* actions, float* returns,
                      float* nonterminals, int pad, float intensity, int m_copies, int k_copies, uint64_t seed,
                      const uint64_t* rng_counter, int32_t* shifts, float* scales, rb_stream_t stream);

/* Bootstrapping through time-limit truncations (no reference counterpart).  rb_gather_horizon's arguments, checks,
 * kernel choice, layouts and draws, and the same outputs for every sample whose records idx + 1 .. idx + n_t - 1 hold no
 * final-observation record (nonterminal byte RB_NONTERMINAL_FINAL, written by rb_append_batch_trunc).  A sample whose
 * first such record is idx + k, k < n_t, is cut there: every output is bitwise what rb_gather_horizon writes for it with a
 * row of n = k, gamma_pow[0 .. k - 1] of *current and gamma_n = current->gamma_pow[k] -- the return of k steps, the next
 * state stacked back from the final observation, and the nonterminal fl32(nonterminal * gamma^k) for a loss launched with
 * gamma_n = 1.  A fixed horizon passes a constant row (n, fl32(gamma ** n), fl32(gamma ** k)).  The rows built by
 * rainbow_b200.horizon hold fl32(gamma ** k) at every k < n, which is the gamma_n of a horizon of k steps.  Refusals as
 * rb_gather_horizon's, named rb_gather_trunc. */
int rb_gather_trunc(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                    const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n_max,
                    const rb_horizon* current, float* states, float* next_states, int64_t* actions, float* returns,
                    float* nonterminals, int pad, float intensity, int m_copies, int k_copies, uint64_t seed,
                    const uint64_t* rng_counter, int32_t* shifts, float* scales, rb_stream_t stream);

/* memory.py:166-178 ReplayMemory.__next__, batched: states for current_idx = first .. first+count-1,
 * backward-only blanking, negative indices wrap.  out is float32[count][history][84*84]. */
int rb_iter_states(const uint8_t* frames, const int32_t* timestep, int64_t size, int64_t first, int count,
                   int history, float* out, rb_stream_t stream);

/* memory.py:105-108 ReplayMemory.append -> :56-61 SegmentTree.append (-> :51-54, :36-41):
 * quantise the newest frame (f32*255, truncating cast), store the record at ring_state.head with
 * timestep = ring_state.t_episode, set its leaf to *running_max and walk to the root, advance the
 * head, set full on wrap, t_episode = terminal ? 0 : t_episode+1.
 * state_last_frame: float32[84*84] device pointer (state[-1]).  The same launch as rb_append_batch with k = 1. */
int rb_append(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep, int32_t* action,
              float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max,
              const float* state_last_frame, int32_t action_value, float reward_value, int terminal,
              rb_stream_t stream);

/* k consecutive rb_append calls in ONE launch (actor side batching, SURVEY.md 8(f).2): HOST arrays of length k --
 * last_frames[j] points at the j-th newest frame (float32[84*84], DEVICE memory or PINNED HOST memory, read in place),
 * actions / rewards / terminals its fields.  Result is identical to k rb_append calls in order.  1 <= k <= RB_APPEND_BATCH.
 * (ReplayMemory(defer_appends=True) uses it.) */
int rb_append_batch(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep, int32_t* action,
                    float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max,
                    const float* const* last_frames, const int32_t* actions, const float* rewards, const int32_t* terminals,
                    int k, rb_stream_t stream);

/* rb_append_batch that can also store final-observation records: terminals[j] == RB_NONTERMINAL_FINAL stores record j with
 * action 0 and reward 0 (actions[j] and rewards[j] are not read), the timestep that continues its episode, nonterminal
 * byte RB_NONTERMINAL_FINAL and leaf 0 -- never sampled, and the running max unchanged -- and the next record starts an
 * episode (timestep 0), as after a terminal.  Other terminals[j] as in rb_append_batch, with the same result.  A time
 * limit's last step is the pair (s_T-1, a, r, 0), (final observation, -, -, RB_NONTERMINAL_FINAL).  Refusals as
 * rb_append_batch's, named rb_append_batch_trunc. */
int rb_append_batch_trunc(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep,
                          int32_t* action, float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max,
                          const float* const* last_frames, const int32_t* actions, const float* rewards,
                          const int32_t* terminals, int k, rb_stream_t stream);

/* Bytes of device scratch rb_append_bulk needs for k records (0 for k <= 0). */
int rb_append_bulk_scratch_bytes(int64_t k);

/* k consecutive appends of already-quantised records in one call (a dataset fill): the result is bitwise that of k
 * rb_append_batch_trunc records in order -- frames, timestep, action, reward, nonterminal, every tree node, the running
 * max (unchanged) and ring_state[0..3].  new_frames: uint8[k][84*84], device or pinned host memory, copied into slots
 * head, head + 1, ... (mod size) by the copy engine (split in two at the wrap); head must be ring_state[0] as the stream
 * will find it (the host mirror of the ring's head).  actions int32[k], rewards float32[k] and flags uint8[k] are device
 * arrays: flag 0 = nonterminal, RB_NONTERMINAL_FINAL = a final-observation record (action 0, reward 0, leaf 0; actions[j]
 * and rewards[j] are not read), any other value = terminal.  Timesteps continue ring_state[2] until the first nonzero
 * flag.  scratch: device memory of at least rb_append_bulk_scratch_bytes(k) bytes, used by this call only.
 * RB_ERR_INVAL: a NULL pointer or an odd size; RB_ERR_RANGE: k outside [1, size], head outside [0, size), a tree deeper
 * than 30 levels or scratch_bytes too small.  A refused call launches nothing.  Profiled under RB_K_APPEND. */
int rb_append_bulk(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep, int32_t* action,
                   float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max, int64_t head,
                   const uint8_t* new_frames, const int32_t* actions, const float* rewards, const uint8_t* flags,
                   int64_t k, void* scratch, int64_t scratch_bytes, rb_stream_t stream);

/* agent.py:66-96 Agent.learn minus the three network bodies, given PRE-softmax logits [B,A,Z]
 * (model.py:75 `q`; the softmax / log_softmax of model.py:76-79 are folded in):
 * double-DQN argmax with the online net, target distribution, Tz clamp, l/u projection with the
 * reference's fix-ups and accumulation order, loss_i = -sum m*logp (the TD priority of
 * agent.py:100), and d(mean_i w_i*loss_i)/dq_online_s.  m_out / astar_out may be NULL. */
int rb_c51_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                     const int64_t* actions, const float* returns, const float* nonterminals,
                     const float* weights, const float* support, float vmin, float vmax, float delta_z,
                     float gamma_n, int B, int A, int Z, float* loss, float* grad_q_online_s, float* m_out,
                     int64_t* astar_out, rb_stream_t stream);
/* rb_c51_loss_grad under value rescaling (Pohlen et al. 2018; DESIGN.md §16): the logits are a distribution over the
 * support in h units, h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x.  support_q[Z] = fl32(h^-1(support)) (return units)
 * replaces the support in the double-DQN arg-max, and the target atoms are Tz_j = h(fl32(r + fl32(s support_q_j))),
 * s = fl32(nonterminal gamma_n), clamped to [vmin, vmax] (h units) and projected as rb_c51_loss_grad projects them.
 * RB_ERR_INVAL also for a NULL support_q and eps outside [0, 1] or NaN.  A refused call writes nothing.  Profiled under
 * RB_K_C51. */
int rb_c51_vt_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                        const float* returns, const float* nonterminals, const float* weights, const float* support,
                        float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z, float* loss,
                        float* grad_q_online_s, float* m_out, int64_t* astar_out, const float* support_q, float eps,
                        rb_stream_t stream);

/* model.py:82-85 DQN.reset_noise -> :36-40 NoisyLinear.reset_noise -> :32-34 _scale_noise, all
 * layers of one net in one launch.  HOST arrays (length n_layers): weight_eps[l] -> float32[out][in],
 * bias_eps[l] -> float32[out], in_features, out_features.
 *   x_in / x_out != NULL : parity mode, raw standard normals, concatenated over layers in layer
 *                          order (eps_in of layer 0, of layer 1, ... / eps_out likewise).
 *   NULL                 : device Philox + Box-Muller keyed by seed and *rng_counter (+1 per call). */
int rb_noisy_resample(float* const* weight_eps, float* const* bias_eps, const int* in_features,
                      const int* out_features, int n_layers, const float* x_in, const float* x_out, uint64_t seed,
                      uint64_t* rng_counter, rb_stream_t stream);

/* Materialise weight_epsilon / bias_epsilon (model.py:39-40) from ALREADY SCALED factor vectors
 * f(eps_in) / f(eps_out) (concatenated over layers like x_in / x_out above): eps_w = f_out (outer) f_in. */
int rb_noisy_outer(float* const* weight_eps, float* const* bias_eps, const int* in_features, const int* out_features,
                   int n_layers, const float* f_in, const float* f_out, rb_stream_t stream);

/* model.py:36-38 for every NoisyLinear of a net, WITHOUT the outer product: f_in[n_in] / f_out[n_out] receive
 * f(eps_in) / f(eps_out) of all layers back to back (layer order).  Same Philox indexing as
 * rb_noisy_resample: rb_noise_factors + rb_noisy_outer == rb_noisy_resample for equal seed and counter.
 * x_in / x_out: optional injected raw normals (parity).  *rng_counter += 1 in Philox mode. */
int rb_noise_factors(float* f_in, int n_in, float* f_out, int n_out, const float* x_in, const float* x_out, uint64_t seed,
                     uint64_t* rng_counter, rb_stream_t stream);

/* ---- fused factorised-noise dueling head (small batches) -----------------------------------------------
 * model.py:69-75 minus the conv body:  h_s = relu(x W1_s^T + b1_s), z_s = h_s W2_s^T + b2_s for the value (s=0) and
 * advantage (s=1) streams, W = mu + sigma * (eps_out (outer) eps_in) composed on the fly from the factor vectors
 * (model.py:39-44) -- weight_epsilon never has to exist in memory.  All pointers are device pointers; the eight
 * eps_* pointers are either all given (training mode) or all NULL (eval mode, model.py:45-46).
 * Requirements: conv_features % 32 == 0, hidden % 64 == 0. */
typedef struct rb_head_params {
  const float* w1_mu[2];    const float* w1_sigma[2];   /* [hidden][conv_features]        fc_h_v, fc_h_a */
  const float* b1_mu[2];    const float* b1_sigma[2];   /* [hidden] */
  const float* w2_mu[2];    const float* w2_sigma[2];   /* [atoms][hidden], [actions*atoms][hidden]   fc_z_v, fc_z_a */
  const float* b2_mu[2];    const float* b2_sigma[2];
  const float* eps_in1[2];  const float* eps_out1[2];   /* f(eps): [conv_features], [hidden] */
  const float* eps_in2[2];  const float* eps_out2[2];   /* [hidden], [atoms] / [actions*atoms] */
  int conv_features, hidden, atoms, actions;
} rb_head_params;

typedef struct rb_head_grads {   /* gradients are OVERWRITTEN (not accumulated) */
  float* w1_mu[2]; float* w1_sigma[2]; float* b1_mu[2]; float* b1_sigma[2];
  float* w2_mu[2]; float* w2_sigma[2]; float* b2_mu[2]; float* b2_sigma[2];
} rb_head_grads;

/* split-K factors used by the head kernels: scratch part1 is float32[s1][M][2*hidden], part2 float32[s2][M][atoms*(1+actions)];
 * tickets is int32[rb_head_ticket_count()], zero-initialised ONCE by the caller (the kernels leave it zeroed).
 * s1 is the larger of the two layer-1 implementations' factors (tensor-core kernel, csrc/rb_head_tc.cu; FFMA kernel). */
int rb_head_splits(int conv_features, int hidden, int* s1, int* s2);
int rb_head_ticket_count(void);
/* Whether the fused head takes this shape, without touching the device: RB_OK, or the code rb_head_forward over `rows`
 * rows (rows > 0) and rb_head_backward over `backward_batch` rows (backward_batch > 0, up to 512) would return for it with
 * valid pointers.  rows == 0 / backward_batch == 0 leave that call out.  Both calls check these limits before they launch
 * anything: a refused backward writes nothing. */
int rb_head_supported(int conv_features, int hidden, int atoms, int actions, int rows, int backward_batch);
/* probes / tests only: bit 0 skips the layer-1 launch of rb_head_forward, bit 1 the layer-2 launch, bit 2 forces the FFMA
 * layer-1 kernel instead of the tensor-core one, bit 3 the split-K layer-2 kernel instead of the single-pass one, bit 4
 * makes rb_head_backward run its large-batch layer-1 kernels at every B (0 = normal) */
int rb_head_debug(int flags);

/* Forward over M = m_lo + m_hi rows (x_lo: [m_lo][conv_features], x_hi: [m_hi][conv_features] or NULL).
 * Outputs: h[M][2*hidden] (post-ReLU hidden activations, value stream in columns [0,hidden), advantage stream in
 * [hidden,2*hidden)) and z[M][atoms*(1+actions)] = (z_value | z_advantage), biases included.
 * Layer 1 runs on the tensor cores (TMA + wgmma, error-compensated TF32 = fp32-equivalent results; csrc/rb_head_tc.cu)
 * followed by a fixed-order split-K reduction kernel; shapes that kernel does not cover (m_hi > 0 with m_lo % 8 != 0) and
 * RB_HEAD_TC=0 in the environment use the FFMA kernel whose last-arriving CTA reduces the partials.  Deterministic. */
int rb_head_forward(const rb_head_params* p, const float* x_lo, int m_lo, const float* x_hi, int m_hi, float* part1, float* part2,
                    int32_t* tickets, float* h, float* z, rb_stream_t stream);

/* q[M][actions][atoms] = zv + za - mean_a(za) (model.py:75) from z. */
int rb_head_logits(const float* z, int M, int actions, int atoms, float* q, rb_stream_t stream);

/* Backward for 1 <= B <= 512 rows, hidden <= 1024 and actions * atoms small enough for the dh kernel's shared memory
 * (about 1060; rb_head_supported says which shapes): given dz[B][atoms*(1+actions)] (value block first),
 * x[B][conv_features] and h[B][2*hidden] writes all 16 parameter gradients through `g` and dx[B][conv_features].
 * dh_scratch: float32[(B + Bp) * 2*hidden], Bp = B rounded up to a multiple of 32 (dh [B][2*hidden], then its transpose
 * [2*hidden][Bp] with the columns past B zero, for the layer-1 kernels).
 * Layer 1 has two implementations with the same outputs, and the call picks by B: up to 32 rows one pass over W1 makes
 * the weight gradients and dx together (k_head_bwd1); above that they run as two GEMM-shaped tensor-core launches,
 * weight gradients reduced over the batch, then dx reduced over both streams' rows (k_head_bwd1_wgrad, k_head_bwd1_dx).
 * relu_mask_x != 0 additionally zeroes dx where x <= 0, i.e. folds in the backward of the ReLU that produced the conv
 * features (model.py:59), so dx is the gradient w.r.t. the last conv layer's pre-activation.
 * `parts` selects which of the three launches to enqueue (so a caller can put the independent layer-2 weight
 * gradient on another stream): RB_HEAD_BWD_WGRAD2 (layer-2 parameter gradients), RB_HEAD_BWD_DH (dh_scratch),
 * RB_HEAD_BWD_LAYER1 (layer-1 parameter gradients + dx; needs dh_scratch); RB_HEAD_BWD_ALL = all, in that order. */
#define RB_HEAD_BWD_WGRAD2 1
#define RB_HEAD_BWD_DH 2
#define RB_HEAD_BWD_LAYER1 4
#define RB_HEAD_BWD_ALL 7
int rb_head_backward(const rb_head_params* p, const rb_head_grads* g, const float* x, const float* h, const float* dz, int B,
                     float* dh_scratch, float* dx, int relu_mask_x, int parts, rb_stream_t stream);

/* agent.py:53-55 Agent.act / :110-112 evaluate_q after the network body, for M states at once: from the head output
 * z[M][atoms*(1+actions)] computes q[m][a] = sum_z support_z * softmax_z(zv + za[a] - mean_a za) (model.py:75-79) and its
 * arg-max / max over actions.  q (float32[M][actions]), best_action (int64[M]), best_q (float32[M]) are each optional. */
int rb_q_values(const float* z, int M, int actions, int atoms, const float* support, float* q, int64_t* best_action,
                float* best_q, rb_stream_t stream);

/* Bias gradient of a conv layer (the sum over batch and pixels torch computes in convolution_backward):
 * out[c] = sum_{b,p} grad_out[b][c][p], grad_out float32[B][C][HW] contiguous; B * HW < 2^31 - 256 (else RB_ERR_RANGE). */
int rb_bias_grad(const float* grad_out, int B, int C, int HW, float* out, rb_stream_t stream);

/* Weight gradient of a conv layer whose data gradient is not needed (the network's first layer; the weight half of
 * torch's convolution_backward there): out[oc][ic][ky][kx] = sum_{b,y,x} grad_out[b][oc][y][x] * input[b][ic][y*stride+ky][x*stride+kx]
 * for a square K x K kernel without padding (K in {3, 4, 5, 8}; IC * K * ceil(OC/4) <= 256).  grad_out float32
 * [B][OC][OH][OW], input float32 [B][IC][IH][IW] (OH = (IH-K)/stride + 1), out float32 [OC][IC][K][K] (overwritten),
 * bias_out (optional, may be NULL) float32 [OC] = sum_{b,y,x} grad_out (the layer's bias gradient, from the same pass),
 * partials: scratch of rb_conv_wgrad_scratch_elems(...) floats.  Two launches, fixed summation order (deterministic).
 * rb_conv_wgrad_scratch_elems returns 0 where the count does not fit in int, and rb_conv_wgrad refuses that B with
 * RB_ERR_RANGE. */
int rb_conv_wgrad_scratch_elems(int B, int IC, int IH, int OC, int K, int stride);
int rb_conv_wgrad(const float* grad_out, const float* input, int B, int IC, int IH, int IW, int OC, int K, int stride,
                  float* partials, float* out, float* bias_out, rb_stream_t stream);

/* rb_c51_loss_grad fed by the fused heads: z_online has 2B rows (s then s'), z_target B rows (s');
 * returns loss[B] and dz[B][atoms*(1+actions)] = d mean(w*loss) / d (z_value | z_advantage) of the online(s) rows
 * (the dueling combination model.py:75 and its backward are folded in). */
int rb_c51_dueling_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                             const float* returns, const float* nonterminals, const float* weights, const float* support,
                             float vmin, float vmax, float delta_z, float gamma_n, int B, float* loss, float* dz, float* m_out,
                             int64_t* astar_out, rb_stream_t stream);
/* rb_c51_dueling_loss_grad under value rescaling: the arg-max and the target atoms as rb_c51_vt_loss_grad forms them,
 * with its refusals.  Profiled under RB_K_C51_DUELING. */
int rb_c51_dueling_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                                const float* returns, const float* nonterminals, const float* weights, const float* support,
                                float vmin, float vmax, float delta_z, float gamma_n, int B, float* loss, float* dz,
                                float* m_out, int64_t* astar_out, const float* support_q, float eps, rb_stream_t stream);

/* rb_c51_dueling_loss_grad with DrQ's averaging over K target copies and M online copies (Kostrikov et al. 2020,
 * Algorithm 1).  z_online has (M + K) B rows: copy j of s at row jB + i, then copy k of s' at row (M + k) B + i; z_target
 * K B rows, copy k of s' at row kB + i.  For sample i: a*_k is the double-DQN arg-max on online(s'_k) (first maximum wins)
 * and m_k the projection of target(s'_k) at a*_k; m = (sum_k m_k, fp32 in k order) / K; loss_j = -sum m log p_j(a) for
 * online(s_j); loss[i] = (sum_j loss_j) / M.  dz[M B][atoms*(1+actions)]: row jB + i is the gradient of online(s_j) with
 * weight / (M B) in place of weight / B.  m_out [B][atoms] (optional) receives m, astar_out [K][B] (optional) a*_k.
 * At M = K = 1 every output equals rb_c51_dueling_loss_grad's, bitwise.  RB_ERR_RANGE: M or K outside
 * [1, RB_MAX_AUG_COPIES], plus rb_c51_dueling_loss_grad's limits with M + 2K staged rows.  A refused call writes nothing. */
int rb_c51_dueling_avg_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                 const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                                 const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int M,
                                 int K, float* loss, float* dz, float* m_out, int64_t* astar_out, rb_stream_t stream);
/* rb_c51_dueling_avg_loss_grad under value rescaling: every m_k projected as rb_c51_vt_loss_grad projects, averaged on the
 * h-space grid; rb_c51_vt_loss_grad's refusals.  At M = K = 1 every output equals rb_c51_dueling_vt_loss_grad's, bitwise.
 * Profiled under RB_K_C51_DUELING_AVG. */
int rb_c51_dueling_avg_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                    const int64_t* actions, const float* returns, const float* nonterminals,
                                    const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                    float gamma_n, int B, int M, int K, float* loss, float* dz, float* m_out,
                                    int64_t* astar_out, const float* support_q, float eps, rb_stream_t stream);

/* Quantile regression (QR-DQN, Dabney et al. 2018) in place of the categorical projection: atoms = N quantiles per action
 * (2 <= N <= RB_MAX_ATOMS) at the midpoints tau_i = (2i + 1) / (2N); no support.  For sample b with taken action a:
 *   theta_i = q_online(s, a)_i (the dueling combination model.py:75 without a softmax),
 *   a* = argmax_a (1/N) sum_j q_online(s', a)_j (double DQN; the first maximum wins),
 *   T_j = r + fl32(nonterminal * gamma_n) q_target(s', a*)_j,  u_ij = T_j - theta_i,
 *   loss_b = sum_i (1/N) sum_j |tau_i - [u_ij < 0]| H_kappa(u_ij) / kappa,  H_kappa(u) = u^2 / 2 if |u| <= kappa, else
 *            kappa (|u| - kappa / 2)   (the TD priority), and the gradient of (1/B) sum_b w_b loss_b:
 *   g_i = -(w_b / B) (1/N) sum_j |tau_i - [u_ij < 0]| clamp(u_ij, -kappa, kappa) / kappa.
 * rb_qr_dueling_loss_grad takes the fused heads' rows like rb_c51_dueling_loss_grad (z_online 2B rows, s then s';
 * z_target B rows) and writes loss[B] and dz[B][atoms*(1+actions)] (dz_v = g, dz_a[a'] = g ([a' == a] - 1/A));
 * rb_qr_loss_grad takes plain quantile rows [B][A][N] like rb_c51_loss_grad and writes grad[B][A][N] (g at the taken
 * action, 0 elsewhere).  Optional outputs: theta_out [B][N] receives the T rows, astar_out [B] a*.  kappa must be finite
 * and > 0.  Sums run in a fixed order (eager launches and graph replays agree bitwise).  RB_ERR_INVAL: a NULL required
 * pointer, B, actions <= 0, atoms < 2 or a bad kappa; RB_ERR_RANGE: atoms > RB_MAX_ATOMS or rows too large for shared
 * memory.  A refused call writes nothing.  Profiled under RB_K_C51_DUELING / RB_K_C51, the loss they stand for. */
int rb_qr_dueling_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                            const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n,
                            int B, float* loss, float* dz, float* theta_out, int64_t* astar_out, rb_stream_t stream);
int rb_qr_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                    const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n, int B,
                    int A, int N, float* loss, float* grad_q_online_s, float* theta_out, int64_t* astar_out,
                    rb_stream_t stream);
/* rb_q_values for quantile heads: q[m][a] = (1/N) sum_j (zv + za[a] - mean_a za)_j and its arg-max (first maximum) / max
 * over actions, from z[M][atoms*(1+actions)].  q, best_action, best_q are each optional (not all NULL). */
int rb_qr_q_values(const float* z, int M, int actions, int atoms, float* q, int64_t* best_action, float* best_q,
                   rb_stream_t stream);
/* The quantile entries under value rescaling (DESIGN.md §16): the quantiles are in h units.  x_j = h^-1(q_target(s', a*)_j),
 * T_j = h(fl32(r + fl32(s x_j))), a* = argmax_a (1/N) sum_j h^-1(q_online(s', a)_j) (first maximum wins); theta, u, the
 * loss, the gradient and theta_out (= T) are in h units.  rb_qr_vt_q_values: q[m][a] = (1/N) sum_j h^-1(q_j) (return
 * units).  RB_ERR_INVAL also for eps outside [0, 1] or NaN.  A refused call writes nothing.  Profiled as their siblings. */
int rb_qr_dueling_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                               const float* returns, const float* nonterminals, const float* weights, float kappa,
                               float gamma_n, int B, float* loss, float* dz, float* theta_out, int64_t* astar_out, float eps,
                               rb_stream_t stream);
int rb_qr_vt_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                       const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n,
                       int B, int A, int N, float* loss, float* grad_q_online_s, float* theta_out, int64_t* astar_out,
                       float eps, rb_stream_t stream);
int rb_qr_vt_q_values(const float* z, int M, int actions, int atoms, float* q, int64_t* best_action, float* best_q,
                      float eps, rb_stream_t stream);

/* rb_qr_dueling_loss_grad with DrQ's averaging over K target copies and M online copies, rows as
 * rb_c51_dueling_avg_loss_grad takes them: z_online has (M + K) B rows, copy j of s at row jB + i, then copy k of s' at
 * row (M + k) B + i; z_target K B rows, copy k of s' at row kB + i.  For sample i:
 *   a*_k = argmax_a (1/N) sum_n q_online(s'_k, a)_n (first maximum wins),
 *   T_k,n = rb_qr_dueling_loss_grad's target row from target(s'_k) at a*_k,
 *   Tbar_n = (sum_k T_k,n, fp32 in k order) / K, rounded once: the quantile-wise average of the K target quantile
 *            functions (its mean is DrQ's averaged target value), not the mixture of their K N samples,
 *   loss_j, g_j = rb_qr_dueling_loss_grad's loss and gradient row of online(s_j) at the taken action against Tbar, with
 *            weight / (M B) in place of weight / B,
 *   loss[i] = (sum_j loss_j, fp32 in j order) / M (also the priority).
 * dz[M B][atoms*(1+actions)]: row jB + i is g_j through the dueling backward.  theta_out [B][atoms] (optional) receives
 * Tbar, so rb_learn_stats_batch_qr takes it unchanged; astar_out [K][B] (optional) a*_k.  At M = K = 1 every output
 * equals rb_qr_dueling_loss_grad's, bitwise.  RB_ERR_INVAL: a NULL required pointer, B, actions <= 0, atoms < 2 or a bad
 * kappa; RB_ERR_RANGE: M or K outside [1, RB_MAX_AUG_COPIES], atoms > RB_MAX_ATOMS, or the M + 2K staged rows too large
 * for shared memory.  A refused call writes nothing.  Profiled under RB_K_C51_DUELING_AVG. */
int rb_qr_dueling_avg_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                                float kappa, float gamma_n, int B, int M, int K, float* loss, float* dz, float* theta_out,
                                int64_t* astar_out, rb_stream_t stream);
/* rb_qr_dueling_avg_loss_grad under value rescaling: a*_k and T_k as rb_qr_dueling_vt_loss_grad forms them, Tbar averaged
 * in h units; also RB_ERR_INVAL for eps outside [0, 1] or NaN.  At M = K = 1 every output equals
 * rb_qr_dueling_vt_loss_grad's, bitwise.  Profiled under RB_K_C51_DUELING_AVG. */
int rb_qr_dueling_avg_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                   const int64_t* actions, const float* returns, const float* nonterminals,
                                   const float* weights, float kappa, float gamma_n, int B, int M, int K, float* loss,
                                   float* dz, float* theta_out, int64_t* astar_out, float eps, rb_stream_t stream);

/* Munchausen targets for the quantile loss (M-RL, Vieillard, Pietquin & Geist 2020; DESIGN.md §17): the target net's
 * softmax policy replaces the double-DQN arg-max, and a clipped log-policy bonus joins the return.  With
 * q(x, a) = (1/N) sum_j q_target(x, a)_j (the dueling combination, then the mean over quantiles) and, per row q[A],
 *   m = max_a q_a,  S = sum_a exp((q_a - m) / temperature) (in action order),  pi_a = exp((q_a - m) / temperature) / S,
 *   l_a = (q_a - m) - temperature log S   (temperature ln pi_a, <= 0),
 * sample i with taken action a has
 *   b   = alpha max(l_a(s), clip)                                                (target row of s),
 *   c_j = sum_a' pi_a'(s') (q_target(s', a')_j - l_a'(s'))  (in action order),
 *   T_j = fl32(r + b) + fl32(fl32(nonterminal * gamma_n) c_j),
 * and theta, the loss (also the priority) and the gradient are rb_qr_dueling_loss_grad's against T.  There is no arg-max.
 * expf / logf run at full precision.
 * rb_qr_dueling_munchausen_loss_grad: z_online has B rows (s only; the online s' rows feed nothing), z_target 2B rows,
 * s at row i then s' at row B + i; writes loss[B] and dz[B][atoms*(1+actions)].  rb_qr_munchausen_loss_grad: plain
 * quantile rows [B][A][N] of online(s), target(s) and target(s'); writes grad[B][A][N] (g at the taken action, 0
 * elsewhere).  Optional outputs: theta_out [B][N] receives T (rb_learn_stats_batch_qr takes it unchanged), bonus_out [B]
 * receives b.  RB_ERR_INVAL: rb_qr_dueling_loss_grad's, plus alpha outside [0, 1], temperature not finite or below
 * FLT_MIN, clip not finite or >= 0 (NaN refused); RB_ERR_RANGE: atoms > RB_MAX_ATOMS or rows too large for shared memory.
 * A refused call writes nothing.  Sums run in a fixed order (eager launches and graph replays agree bitwise).  Profiled
 * under RB_K_C51_DUELING / RB_K_C51. */
int rb_qr_dueling_munchausen_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                       const int64_t* actions, const float* returns, const float* nonterminals,
                                       const float* weights, float kappa, float gamma_n, float alpha, float temperature,
                                       float clip, int B, float* loss, float* dz, float* theta_out, float* bonus_out,
                                       rb_stream_t stream);
int rb_qr_munchausen_loss_grad(const float* q_online_s, const float* q_target_s, const float* q_target_ns,
                               const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                               float kappa, float gamma_n, float alpha, float temperature, float clip, int B, int A, int N,
                               float* loss, float* grad_q_online_s, float* theta_out, float* bonus_out, rb_stream_t stream);

/* Risk-sensitive selection (distortion risk measures, Dabney et al. 2018 §5; DESIGN.md §18): the double-DQN arg-max and
 * the greedy values read the return distribution through a distortion beta: [0, 1] -> [0, 1] in place of its mean,
 *   RB_RISK_CVAR  beta(t) = min(t / eta, 1),          eta in (0, 1]  (1: the mean);
 *   RB_RISK_WANG  beta(t) = Phi(Phi^-1(t) - eta),     eta finite     (< 0 risk-averse, 0 the mean, > 0 risk-seeking),
 * beta(t) being the weight of the levels [0, t]: the inverses of IQN's level maps eta tau and Phi(Phi^-1(tau) + eta).
 * Quantile rows: Q_beta = sum_j (beta((j+1)/N) - beta(j/N)) theta_j, quantile j standing for the levels [j/N, (j+1)/N]
 * in index order.  Categorical rows: p = softmax over atoms, F_k = sum_{k' <= k} p_k' (F_{Z-1} = 1),
 * Q_beta = sum_k (beta(F_k) - beta(F_{k-1})) support_k with F_{-1} = 0; the support must be non-decreasing (the agent's
 * linspace is).  DESIGN.md §18 states the fp32 operation order.
 * Each entry below is its parent's (the name without _risk) with Q_beta in place of the mean, and the parent's arguments
 * plus risk_kind and risk_eta: in the loss entries Q_beta of online(s') picks a* (the first maximum wins), and everything
 * after it -- the projection or the quantile loss, the loss, the gradient, m_out / theta_out and astar_out -- is the
 * parent's for that a*; rb_q_values_risk / rb_qr_q_values_risk write Q_beta per action, its arg-max and its max.
 * RB_ERR_INVAL: the parent's refusals, plus a kind other than RB_RISK_CVAR / RB_RISK_WANG, a CVaR eta outside (0, 1] or a
 * Wang eta that is not finite (NaN refused).  A refused call writes nothing.  Profiled under the parent's kernel id. */
#define RB_RISK_CVAR 1
#define RB_RISK_WANG 2
int rb_c51_risk_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                          const float* returns, const float* nonterminals, const float* weights, const float* support,
                          float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z, float* loss,
                          float* grad_q_online_s, float* m_out, int64_t* astar_out, int risk_kind, float risk_eta,
                          rb_stream_t stream);
int rb_c51_dueling_risk_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                  const int64_t* actions, const float* returns, const float* nonterminals,
                                  const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                  float gamma_n, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                  int risk_kind, float risk_eta, rb_stream_t stream);
int rb_qr_dueling_risk_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                 const int64_t* actions, const float* returns, const float* nonterminals,
                                 const float* weights, float kappa, float gamma_n, int B, float* loss, float* dz,
                                 float* theta_out, int64_t* astar_out, int risk_kind, float risk_eta, rb_stream_t stream);
int rb_qr_risk_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                         const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n,
                         int B, int A, int N, float* loss, float* grad_q_online_s, float* theta_out, int64_t* astar_out,
                         int risk_kind, float risk_eta, rb_stream_t stream);
int rb_q_values_risk(const float* z, int M, int actions, int atoms, const float* support, float* q, int64_t* best_action,
                     float* best_q, int risk_kind, float risk_eta, rb_stream_t stream);
int rb_qr_q_values_risk(const float* z, int M, int actions, int atoms, float* q, int64_t* best_action, float* best_q,
                        int risk_kind, float risk_eta, rb_stream_t stream);

/* HL-Gauss targets for the categorical loss (Farebrother et al. 2024, "Stop Regressing"; DESIGN.md §20): cross-entropy
 * against the histogram that N(y, sigma^2) puts on the support's bins, in place of C51's projection.  Per sample:
 *   a*    = the double-DQN arg-max of the expected values of online(s') (first maximum wins), as the parents take it;
 *   ybar  = the expected value of target(s') at a*;  y = clamp(fl32(r + fl32(fl32(nonterminal gamma_n) ybar)), vmin, vmax);
 *   bins  e_k = fl32(support_k - h) for k < Z, e_Z = fl32(support_{Z-1} + h), h = fl32(delta_z / 2): the atoms are the
 *         bin centres;
 *   mass  t_k = fl32(fl32(e_k - y) c), c = fl32(1 / fl32(sqrt(2) sigma)); u_k = 1/2 (erfc(t_k) - erfc(t_{k+1})) when
 *         t_k >= 0, 1/2 (erfc(-t_{k+1}) - erfc(-t_k)) when t_{k+1} <= 0, else 1/2 (erf(t_{k+1}) - erf(t_k));
 *         U = sum_k u_k (per lane over its atoms k = lane + 32 r in r order, then the xor butterfly), m_k = fl32(u_k / U);
 *   loss  -sum_k m_k log p_k(s, a) and the gradient row (w / B)(p sum(m) - m) of the taken action, as the parents form
 *         them against their projection; priorities are this cross-entropy, whose floor is the entropy H(m) > 0.
 * sigma is in return units (the agent passes fl32(ratio * delta_z)).  Each entry takes its parent's arguments (the name
 * without _hlg), sigma after gamma_n, and the optional y_out [B] (y per sample) after astar_out; m_out and astar_out are
 * the parent's.  RB_ERR_INVAL: the parent's refusals, plus a sigma that is not a positive normal fp32 (NaN, +-inf, 0,
 * negatives and subnormals).  A refused call writes nothing.  Profiled under the parent's kernel id. */
int rb_c51_hlg_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                         const float* returns, const float* nonterminals, const float* weights, const float* support,
                         float vmin, float vmax, float delta_z, float gamma_n, float sigma, int B, int A, int Z,
                         float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, float* y_out,
                         rb_stream_t stream);
int rb_c51_dueling_hlg_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                 const int64_t* actions, const float* returns, const float* nonterminals,
                                 const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                 float gamma_n, float sigma, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                 float* y_out, rb_stream_t stream);

/* Two-hot targets for the categorical loss (Farebrother et al. 2024; MuZero, Schrittwieser et al. 2020, Appendix F;
 * DESIGN.md §21): cross-entropy against the scalar double-DQN target y split between its two neighbouring atoms, in place
 * of C51's projection.  Per sample:
 *   a*    = the double-DQN arg-max of the expected values of online(s') (first maximum wins), as the parents take it;
 *   ybar  = the expected value of target(s') at a*;  y = clamp(fl32(r + fl32(fl32(nonterminal gamma_n) ybar)), vmin, vmax);
 *   split b = fl32(fl32(y - vmin) / delta_z), l = floor(b), u = ceil(b), then the projection's fix-ups (u > 0 and l == u:
 *         l -= 1; then l < Z - 1 and l == u: u += 1); m_l = fl32(u - b), m_u = fl32(b - l), every other m_k = 0 (an
 *         index u = Z, where rounding puts b past Z - 1, is dropped as the projection drops it);
 *   loss  -sum_k m_k log p_k(s, a) and the gradient row (w / B)(p sum(m) - m) of the taken action, as the parents form
 *         them; priorities are this cross-entropy, whose floor is the entropy H(m) <= ln 2 (0 when y is on an atom).
 * Each entry takes its parent's arguments (rb_c51_loss_grad / rb_c51_dueling_loss_grad) and the optional y_out [B]
 * (y per sample) after astar_out; m_out and astar_out are the parent's.  RB_ERR_INVAL / RB_ERR_RANGE: the parent's
 * refusals.  A refused call writes nothing.  Profiled under the parent's kernel id. */
int rb_c51_twohot_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                            const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                            const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z,
                            float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, float* y_out,
                            rb_stream_t stream);
int rb_c51_dueling_twohot_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                    const int64_t* actions, const float* returns, const float* nonterminals,
                                    const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                    float gamma_n, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                    float* y_out, rb_stream_t stream);

/* The two-hot entries under value rescaling (DESIGN.md §16, §21): support_q = fl32(h^-1(support)) in place of the support
 * for the arg-max and ybar (return units), and y = clamp(h(fl32(r + fl32(sc ybar))), vmin, vmax), h first as
 * rb_c51_vt_loss_grad forms its target atoms; y_out is then in h units.  support_q and eps after y_out.  Refusals:
 * rb_c51_vt_loss_grad's first (a null support_q, eps outside [0, 1] or NaN), then the parent's. */
int rb_c51_twohot_vt_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                               const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                               const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int A,
                               int Z, float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, float* y_out,
                               const float* support_q, float eps, rb_stream_t stream);
int rb_c51_dueling_twohot_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                       const int64_t* actions, const float* returns, const float* nonterminals,
                                       const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                       float gamma_n, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                       float* y_out, const float* support_q, float eps, rb_stream_t stream);

/* CQL(H)'s regulariser for training from a fixed replay (Kumar et al. 2020; DESIGN.md §22), added onto the gradient a
 * loss entry has just written.  For copy j < M of sample i (row jB + i of the online net's rows of s) with values Q_a --
 * the expected value sum_k softmax(q_a)_k support_k (the loss entries' arithmetic), or with a NULL support the mean
 * quantile (sum_k q_ak) / Z of the quantile head:
 *   R_ij = logsumexp_a Q_a - Q_{a_i}, stable (maximum first, sums in action order), pi = softmax_a Q;
 *   c    = fl32(fl32(alpha w_i) / (M B)), c_a = fl32(c (pi_a - [a == a_i]));
 *   grad += c_a fl32(p_ak fl32(support_k - Q_a)) (categorical) or fl32(c_a / Z) (quantile) on the logits of every action:
 * the gradient of sum_i w_i alpha (1/M) sum_j R_ij / B.  rb_cql_grad takes logit rows [M B][A][Z] (rb_c51_loss_grad's
 * layout) and adds onto grad [M B][A][Z]; rb_cql_dueling_grad takes the fused heads' z rows [Z + A Z] (their first M B
 * rows are read) and adds onto dz [M B][Z + A Z] through the dueling combination: dzv_k += gv_k = sum_a g_ak (action
 * order), dza_ak += g_ak - gv_k / A.  gap_out [B] (optional) = fl32(sum_j R_ij (j order) / M).  No atomics: results do
 * not depend on scheduling.  RB_ERR_INVAL: a NULL rows, actions, weights or grad, B or A <= 0, Z < 2, or alpha not a
 * positive finite normal fp32; RB_ERR_RANGE: Z > RB_MAX_ATOMS, M outside [1, RB_MAX_AUG_COPIES], or rows too large for
 * shared memory.  A refused call writes nothing.  Profiled under RB_K_C51 / RB_K_C51_DUELING. */
int rb_cql_grad(const float* q_online_s, const int64_t* actions, const float* weights, const float* support, float alpha,
                int M, int B, int A, int Z, float* grad, float* gap_out, rb_stream_t stream);
int rb_cql_dueling_grad(const float* z_online, const int64_t* actions, const float* weights, const float* support,
                        float alpha, int M, int B, int A, int Z, float* dz, float* gap_out, rb_stream_t stream);

/* model.py:43-44 NoisyLinear.forward weight composition W = mu + sigma*eps (elementwise),
 * used for both weights ([out*in]) and biases ([out]). */
int rb_noisy_compose(const float* mu, const float* sigma, const float* eps, int64_t count, float* out,
                     rb_stream_t stream);

/* agent.py:97-98 clip_grad_norm_(params, max_norm) + Adam.step() on FLAT float32 buffers of P
 * elements (all online-net parameters laid out back to back).  `step_count` is a device int64 holding
 * the number of steps already taken; the kernel increments it.  grad_scale multiplies the gradient
 * before everything else (1/world_size after a SUM all-reduce; 1.0 on one GPU).
 * partial_sums: scratch float64[rb_clip_adam_scratch_elems()], ZERO-INITIALISED once by the caller (its last element is a
 * self-resetting completion ticket).  norm_out (optional) receives the
 * pre-clip global L2 norm.  gate (optional device int32, may be NULL): when *gate == 0 neither the parameters, the
 * moments nor step_count change (rejected sample batch, see rb_tree_sample). */
int rb_clip_adam_scratch_elems(void);
int rb_clip_adam(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t P, float grad_scale,
                 float max_norm, float lr, float beta1, float beta2, float eps, int64_t* step_count,
                 double* partial_sums, float* norm_out, const int32_t* gate, rb_stream_t stream);

/* rb_clip_adam with decoupled weight decay (AdamW, torch.optim.AdamW) and Adam state per parameter GROUP.  The groups
 * tile [0, P) in order; group g has weight decay lambda_g and its own bias-correction count group_steps[g] (device
 * int64[n_groups], steps already taken by that group).  The norm, clip coefficient and grad_scale are rb_clip_adam's (one
 * global norm, decay not part of it).  For an element of group g, with t_g = group_steps[g] + 1:
 *   p = p * fl32(1 - lr lambda_g)           (rounded on its own; torch's param.mul_(1 - lr wd) before the moments)
 *   then rb_clip_adam's Adam step with the bias corrections of t_g.
 * The call advances *step_count (applied steps, as rb_clip_adam) and every group_steps[g].  A gate reading 0 writes only
 * norm_out.  With every lambda_g = 0 and every group_steps[g] == *step_count the result is rb_clip_adam's, bitwise.
 * A restart of group g's Adam state is the caller zeroing its moment range and group_steps[g].
 * groups: HOST array of n_groups entries, copied into the launch.  partial_sums as for rb_clip_adam.  Profiled under
 * RB_K_SQNORM and RB_K_CLIP_ADAM.
 * RB_ERR_INVAL: a NULL pointer (norm_out and gate may be NULL) or P <= 0; RB_ERR_RANGE: n_groups outside
 * [1, RB_MAX_ADAM_GROUPS], groups that do not tile [0, P) (a gap, an overlap, unsorted, empty, or a last end other than
 * P), a begin that is not a multiple of 4, lambda negative or not finite, fl32(lr) fl32(lambda) >= 1.  A refused call
 * launches nothing. */
#define RB_MAX_ADAM_GROUPS 4
typedef struct rb_adam_group {
  int64_t begin, end;      /* flat elements [begin, end) */
  float weight_decay;      /* lambda >= 0 */
} rb_adam_group;
int rb_clip_adamw(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t P, float grad_scale,
                  float max_norm, float lr, float beta1, float beta2, float eps, const rb_adam_group* groups, int n_groups,
                  int64_t* step_count, int64_t* group_steps, double* partial_sums, float* norm_out, const int32_t* gate,
                  rb_stream_t stream);

/* Polyak (soft) target update over FLAT float32 buffers of n elements (no reference counterpart; the reference only copies
 * the online net into the target, agent.py:102-103).  For every i < n:
 *   target[i] = fmaf(tau, param[i], fl32(1 - tau) * target[i])
 * with 1 - tau formed in fp32 and the product rounded on its own (no contraction).  tau = 1 copies param for finite target.
 * gate (optional device int32, may be NULL): when *gate == 0 nothing is written (rejected sample batch, as rb_clip_adam).
 * RB_ERR_INVAL: a NULL target or param, n < 0, or overlapping buffers; RB_ERR_RANGE: tau outside (0, 1] or NaN.  A refused
 * call launches nothing; n == 0 launches nothing and returns RB_OK. */
int rb_target_ema(float* target, const float* param, int64_t n, float tau, const int32_t* gate, rb_stream_t stream);

/* Shrink-and-perturb reset (Ash & Adams 2020; the later-layer resets of Nikishin et al. 2022) of a FLAT float32 parameter
 * buffer of n elements, over a table of segments (one per parameter tensor).  For every element j of segment s:
 *   theta0 = fmaf(bound_s, r, constant_s),  r = 2u - 1,  u = (w >> 8) * 2^-24
 *   param[j] = fmaf(alpha_s, param[j], fl32(1 - alpha_s) * theta0)
 * where w is word (j & 3) of Philox4x32-10 with key `seed` and counter (k_lo, k_hi, j >> 2, 0x52534554), k = reset_index.
 * A uniform initialisation U[-b, b) is {bound b, constant 0}, a constant c is {bound 0, constant c}.  alpha = 1 leaves a
 * segment bitwise unchanged, alpha = 0 re-draws it.  Elements outside every segment are never written.
 * segs: HOST array of n_segs entries, sorted by offset and non-overlapping, copied into the launch.
 * RB_ERR_INVAL: a NULL param or segs; RB_ERR_RANGE: n_segs outside [1, RB_MAX_RESET_SEGMENTS], a segment outside [0, n),
 * unsorted or overlapping, count <= 0, a negative or non-finite bound or constant, alpha outside [0, 1] or NaN.  A refused
 * call launches nothing. */
typedef struct rb_reset_segment {
  int64_t offset, count;
  float bound, constant, alpha;
} rb_reset_segment;
int rb_param_reset(float* param, int64_t n, const rb_reset_segment* segs, int n_segs, uint64_t seed, uint64_t reset_index,
                   rb_stream_t stream);

/* Dormant-neuron statistics and ReDo recycling (Sokar et al. 2023, "The Dormant Neuron Phenomenon in Deep RL"; no reference
 * counterpart).  Nothing here synchronises or reads back: the sums, the mask and the rewrite stay on the device.
 *
 * rb_neuron_scores: sums[c] = sum_{r < R, p < HW} act[r][c][p] for post-ReLU activations act [R][C][HW] (a linear layer:
 * HW = 1), one CTA per neuron: fp32 partial sums over chunks of 64 addends, added into float64, a fixed order (an eager
 * launch and a replay agree bitwise).  |sums[c] - exact| <= 63 * 2^-24 * exact for non-negative activations.
 * RB_ERR_INVAL: a NULL pointer, or R, C or HW <= 0. */
int rb_neuron_scores(const float* act, int R, int C, int HW, double* sums, rb_stream_t stream);

/* rb_redo_mask: one launch over every scored layer.  Layer l owns neurons [offset_l, offset_l + neurons_l) of sums and
 * mask; its scores are s_i = sums[i] / count_l (count_l = rows * HW behind each sum, over all ranks after an all-reduce of
 * the sums), its mean the float64 sum of the s_i in neuron order over neurons_l, and
 *   mask[i] = s_i <= (double)tau * mean        (tau = 0: exactly-dead neurons; a layer of mean 0 is all dormant).
 * record (device int64[RB_REDO_RECORD_WORDS]): {pass_index, n_layers, then (neurons_l, dormant_l) per layer}.
 * layers: HOST array, sorted by offset and non-overlapping, copied into the launch.
 * RB_ERR_INVAL: a NULL pointer; RB_ERR_RANGE: n_layers outside [1, RB_MAX_REDO_LAYERS], tau outside [0, 1] or NaN, a
 * negative pass_index, a layer empty, unsorted or overlapping, count outside [1, 2^53].  A refused call launches nothing. */
typedef struct rb_redo_scored {
  int32_t offset, neurons;
  double count;
} rb_redo_scored;
int rb_redo_mask(const double* sums, const rb_redo_scored* layers, int n_layers, float tau, uint8_t* mask, int64_t* record,
                 int64_t pass_index, rb_stream_t stream);

/* rb_redo_recycle: ReDo (Algorithm 1) on the FLAT float32 parameter buffer of n elements and the two Adam moment buffers
 * laid out like it, one launch.  For every neuron i of layer l with mask[mask_offset_l + i] != 0:
 *   incoming block {offset, per_neuron, bound, constant}: elements j in [offset + i per_neuron, offset + (i + 1) per_neuron)
 *     become theta0(j) = fmaf(bound, 2u - 1, constant), u = (w >> 8) * 2^-24, w = word (j & 3) of Philox4x32-10 with key
 *     `seed` and counter (k_lo, k_hi, j >> 2, 0x5245444F), k = pass_index: rb_param_reset's draw on a stream word of its own.
 *     src_span > 0: element e of the neuron's block reads from neuron e / src_span of the layer whose mask begins at
 *     src_mask_offset; where that neuron is dormant the element is left to the outgoing rule (it becomes +0);
 *   outgoing block {offset, rows, row_stride, span}: elements [offset + r row_stride + i span, ... + span) of every row
 *     r < rows become +0;
 *   exp_avg and exp_avg_sq of every element written become +0.
 * Nothing else is written; a table whose mask is all zero writes nothing.  layers: HOST array copied into the launch.
 * RB_ERR_INVAL: a NULL pointer; RB_ERR_RANGE: n_layers outside [1, RB_MAX_REDO_LAYERS], a layer without neurons (or more
 * than 65535), n_in outside [1, RB_MAX_REDO_BLOCKS], n_out outside [0, RB_MAX_REDO_BLOCKS], a block empty or outside
 * [0, n), rows of an outgoing block overlapping (row_stride < neurons * span), two incoming or two outgoing blocks
 * overlapping, two layers' mask ranges overlapping, a negative or non-finite bound or constant, a src_span that does not
 * divide per_neuron or names no other layer of the table.  A refused call launches nothing. */
typedef struct rb_redo_in {
  int64_t offset, per_neuron, src_span;
  int32_t src_mask_offset;
  float bound, constant;
} rb_redo_in;
typedef struct rb_redo_out {
  int64_t offset, rows, row_stride, span;
} rb_redo_out;
typedef struct rb_redo_layer {
  int32_t neurons, mask_offset, n_in, n_out;
  rb_redo_in in[RB_MAX_REDO_BLOCKS];
  rb_redo_out out[RB_MAX_REDO_BLOCKS];
} rb_redo_layer;
int rb_redo_recycle(float* param, float* exp_avg, float* exp_avg_sq, int64_t n, const rb_redo_layer* layers, int n_layers,
                    const uint8_t* mask, uint64_t seed, uint64_t pass_index, rb_stream_t stream);

/* Multi-GPU replacement of "all-reduce the flat gradient, then rb_clip_adam on every rank" (agent.py:97-98 under data
 * parallelism; no reference counterpart): reduce-scatter by peer loads + clip + Adam on the owned 1/world parts (moments
 * sharded) + all-gather by peer stores, ordered by epoch flags in peer-visible memory.  HOST arrays of length `world`:
 * peer_grad[q] / peer_param[q] = rank q's flat gradient / parameter buffer, peer_flags[q] = rank q's uint64[4*world] flag
 * block, peer_norms[q] = rank q's double[world] block (both zero-initialised once), all mapped on this device.
 * epoch: device uint64 (zero-initialised, advanced once per step by rb_peer_adam_gather); scratch: rb_peer_scratch_bytes()
 * zeroed bytes.  Every rank must make the same calls each step.
 *
 * The flat buffer is exchanged as one or two SEGMENTS [seg_begin, seg_begin + seg_len) (seg_len % (4*world) == 0); rank r
 * owns part r (seg_len / world elements) of each.  rb_peer_reduce reduces one segment (it may be enqueued on another
 * stream as soon as that segment's gradients are final -- the learner sends the noisy-head segment while the conv backward
 * still runs); gred_part receives this rank's reduced part, multiplied by grad_scale (1/world for averaging).
 * rb_peer_adam_gather (after every segment's rb_peer_reduce, stream-ordered) publishes the partial norms, clips, runs Adam
 * on the owned parts -- gred / exp_avg / exp_avg_sq hold the parts of segment 0, then segment 1, back to back --, stores the
 * new parameters into every rank's buffer and returns when all ranks' parts have landed here.  multicast_param (optional,
 * may be NULL): the NVLS multicast mapping of the parameter buffers (one address that the NVSwitch replicates to every
 * rank); when given, the all-gather is a single multimem.st per 16 bytes instead of `world` peer stores.
 * rb_peer_clip_adam = rb_peer_reduce over [0, P) + rb_peer_adam_gather with that single segment.
 * tools/peer_adam_check.py compares it against NCCL all-reduce + rb_clip_adam. */
int rb_peer_scratch_bytes(void);
int rb_peer_reduce(const float* const* peer_grad, uint64_t* const* peer_flags, int world, int rank, int seg, int64_t seg_begin,
                   int64_t seg_len, float grad_scale, float* gred_part, const uint64_t* epoch, void* scratch,
                   rb_stream_t stream);
int rb_peer_adam_gather(float* const* peer_param, uint64_t* const* peer_flags, double* const* peer_norms, int world, int rank,
                        int n_seg, const int64_t* seg_begin, const int64_t* seg_len, const float* gred, float* exp_avg,
                        float* exp_avg_sq, float max_norm, float lr, float beta1, float beta2, float eps, int64_t* step_count,
                        uint64_t* epoch, void* scratch, float* norm_out, float* multicast_param, rb_stream_t stream);
/* rb_peer_adam_gather with rb_clip_adamw's decoupled weight decay and Adam state per SEGMENT: seg_weight_decay (HOST
 * float[n_seg]) and seg_steps (device int64[n_seg], each segment's bias-correction count, advanced with step_count).  The
 * segments are the groups; the moment shards of a segment restart when the caller zeroes them and its count.  Refused
 * as rb_peer_adam_gather, and also for a NULL seg_weight_decay / seg_steps (RB_ERR_INVAL) or a lambda negative, not
 * finite or with fl32(lr) fl32(lambda) >= 1 (RB_ERR_RANGE).  With every lambda = 0 and every seg_steps[s] == *step_count
 * the result is rb_peer_adam_gather's, bitwise. */
int rb_peer_adamw_gather(float* const* peer_param, uint64_t* const* peer_flags, double* const* peer_norms, int world, int rank,
                         int n_seg, const int64_t* seg_begin, const int64_t* seg_len, const float* seg_weight_decay,
                         const float* gred, float* exp_avg, float* exp_avg_sq, float max_norm, float lr, float beta1,
                         float beta2, float eps, int64_t* step_count, int64_t* seg_steps, uint64_t* epoch, void* scratch,
                         float* norm_out, float* multicast_param, rb_stream_t stream);
int rb_peer_clip_adam(const float* const* peer_grad, float* const* peer_param, uint64_t* const* peer_flags,
                      double* const* peer_norms, int world, int rank, int64_t P, float* gred, float* exp_avg,
                      float* exp_avg_sq, float grad_scale, float max_norm, float lr, float beta1, float beta2, float eps,
                      int64_t* step_count, uint64_t* epoch, void* scratch, float* norm_out, rb_stream_t stream);

/* Learner statistics of one update (agent.py:66-98 computes most of them and discards them), recorded on the device.
 * One record, 48 bytes; i runs over the B samples of the batch:
 *   update       running index of the record (the value of *counter when it was written)
 *   loss_mean    mean_i loss_i, loss_i = -sum_z m_iz log p_iz (agent.py:94; the TD priority before ^omega)
 *   loss_max     max_i loss_i
 *   objective    mean_i w_i loss_i (agent.py:96)
 *   q_mean       mean_i sum_z softmax(q(s_i, a_i))_z support_z, the online logits of the taken action
 *   target_mean  mean_i sum_z m_iz support_z
 *   edge_mass    mean_i (m_i,0 + m_i,Z-1), the projected mass the clamp to [Vmin, Vmax] piles onto the end atoms
 *   weight_min   min_i w_i
 * Under the quantile loss (rb_learn_stats_batch_qr) loss_i is the quantile loss, q_mean = mean_i mean_k theta_ik of the
 * online quantiles of the taken action, target_mean = mean_i mean_k T_ik, and edge_mass is NaN: there is no support to
 * clamp to.
 *   grad_norm    *grad_norm (the pre-clip norm written by rb_clip_adam / rb_peer_adam_gather as norm_out)
 *   clip_coef    min(1, max_norm / (grad_norm + 1e-6)), the factor rb_clip_adam scaled the gradient by
 *   applied      1 if the optimiser stepped, 0 if *gate == 0 made it skip the step */
typedef struct rb_learn_stats_record {
  int64_t update;
  float loss_mean, loss_max, objective, q_mean, target_mean, edge_mass, weight_min, grad_norm, clip_coef, applied;
} rb_learn_stats_record;

/* The record of one update, in two parts so that only a one-thread launch has to follow the optimiser step:
 *   rb_learn_stats_batch   (as soon as the loss kernel has run; the learner puts it on a side stream beside the backward)
 *     computes the batch fields from loss[B], weights[B], actions[B] (int64), m[B][Z] (the m_out of rb_c51_loss_grad /
 *     rb_c51_dueling_loss_grad), support[Z] and the online logits of the s rows in exactly one of two layouts: z = the
 *     fused head's (z_value | z_advantage) [>= B rows][Z + A Z] (dueling combination model.py:75 applied here), or
 *     q = [B][A][Z]; the other pointer is NULL.  The results stay in `scratch`.
 *   rb_learn_stats_write   (after the optimiser step) writes them with *grad_norm (device float), the clip coefficient and
 *     the gate (optional device int32; NULL = the step was applied) into ring[*counter % capacity] and advances *counter
 *     (device int64), so each replay of a captured graph writes a fresh slot.
 * rb_learn_stats = both, in that order on one stream.  scratch: double[rb_learn_stats_scratch_elems()], ZERO-INITIALISED
 * once by the caller (its last element is a self-resetting completion ticket); one scratch per stream of records.  Sums
 * over the batch run in float64 in a fixed order (an eager launch and a graph replay agree bitwise).  RB_ERR_INVAL: a NULL
 * pointer, or both / neither of z and q; RB_ERR_RANGE: Z > RB_MAX_ATOMS or capacity <= 0.  A refused call writes nothing. */
int rb_learn_stats_scratch_elems(void);
int rb_learn_stats_batch(const float* loss, const float* weights, const int64_t* actions, const float* m, const float* support,
                         const float* z, const float* q, int B, int A, int Z, double* scratch, rb_stream_t stream);
int rb_learn_stats_write(const double* scratch, const float* grad_norm, const int32_t* gate, float max_norm,
                         rb_learn_stats_record* ring, int capacity, int64_t* counter, rb_stream_t stream);
/* rb_learn_stats_batch for rb_qr_*_loss_grad: theta[B][N] is their theta_out (the T rows), z / q the online quantile rows
 * in one of the two layouts above (N = atoms); no support.  Same scratch, refusals and rb_learn_stats_write. */
int rb_learn_stats_batch_qr(const float* loss, const float* weights, const int64_t* actions, const float* theta, const float* z,
                            const float* q, int B, int A, int N, double* scratch, rb_stream_t stream);
/* rb_learn_stats_batch_qr under value rescaling: theta from rb_qr_*_vt_loss_grad; q_mean = mean_i mean_k h^-1(theta_ik) and
 * target_mean = mean_i mean_k h^-1(T_ik), in return units.  RB_ERR_INVAL also for eps outside [0, 1] or NaN. */
int rb_learn_stats_batch_qr_vt(const float* loss, const float* weights, const int64_t* actions, const float* theta,
                               const float* z, const float* q, int B, int A, int N, double* scratch, float eps,
                               rb_stream_t stream);
int rb_learn_stats(const float* loss, const float* weights, const int64_t* actions, const float* m, const float* support,
                   const float* z, const float* q, int B, int A, int Z, const float* grad_norm, const int32_t* gate,
                   float max_norm, double* scratch, rb_learn_stats_record* ring, int capacity, int64_t* counter,
                   rb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* RAINBOW_B200_H */
