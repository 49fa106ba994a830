// rb_kernels.cu -- hand-written sm_90a kernels + C ABI for the Rainbow learner hot path.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC
//        (see rainbow_b200/_build.py).  Header: include/rainbow_b200.h.
//
// Every kernel here is HBM/L2-latency bound byte and index work (SURVEY.md 8(d)); none of it is
// GEMM shaped, so there is deliberately no tensor-core code in this file.  What matters instead:
// few dependent memory round trips per tree walk, 16-byte coalesced accesses for the frame traffic,
// no host synchronisation anywhere (everything is stream ordered and graph capturable).
//
// Numerics contract (SURVEY.md Appendix A): tree nodes are float32 sums recomputed from their
// children (never delta-accumulated), descents carry a float64 residual, the C51 projection uses
// separately rounded float32 operations in the reference's order (no FMA contraction: explicit
// __fmul_rn/__fadd_rn/__fsub_rn/__fdiv_rn intrinsics).

#include <cuda_runtime.h>
#include <float.h>
#include <math_constants.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "rainbow_b200.h"
#include "rb_internal.cuh"

namespace rbi {
thread_local char g_err[256] = "";
char* err_buffer() { return g_err; }
bool g_prof_on = false;
ProfKernel g_prof[RB_KERNEL_COUNT];
SmemGrant g_smem_grants[256] = {};
SmemGrant* smem_grants() { return g_smem_grants; }
bool& prof_on() { return g_prof_on; }
ProfKernel* prof_table() { return g_prof; }
}  // namespace rbi

namespace {

using rbi::box_muller;
using rbi::check_launch;
using rbi::fail;
using rbi::normal4;
using rbi::philox4x32_10;
using rbi::ProfKernel;
using rbi::ProfScope;
using rbi::scale_noise;
using rbi::u53;

__device__ __forceinline__ int64_t pymod(int64_t a, int64_t m) {
  int64_t r = a % m;
  return r < 0 ? r + m : r;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__host__ __device__ inline int tree_depth(int64_t tree_start) {  // edges root -> leaf
  int L = 0;
  while (((int64_t)1 << L) - 1 < tree_start) ++L;
  return L;
}

// ================================================================================================
// K4  tree_update : leaf scatter (last write wins) + propagate-to-root, one CTA.
// ================================================================================================
// One thread per updated leaf.  After the leaf writes every thread walks towards the root in
// lock step: a level is  tree[p] = tree[2p+1] + tree[2p+2]  for the thread's parent p, then a CTA
// barrier so the next level reads finished children (threads sharing a parent write the same value).
// Loads bypass L1 (__ldcg): other threads of the CTA have just written those addresses.
constexpr int UPD_THREADS = 1024;

__global__ void __launch_bounds__(UPD_THREADS, 1)
k_tree_update(float* tree, int64_t tree_start, int64_t size, const int64_t* __restrict__ tree_idx,
              const float* __restrict__ raw, float omega, int omega_is_applied, int B, float* running_max,
              int32_t* status, const int32_t* __restrict__ gate) {
  if (gate && *gate == 0) return;   // the batch these priorities belong to was rejected by rb_tree_sample: leave the tree alone
  __shared__ int64_t s_idx[UPD_THREADS];
  __shared__ float s_red[32];
  const int tid = threadIdx.x;
  const int64_t len = tree_start + size;
  float block_max = -CUDART_INF_F;

  for (int base = 0; base < B; base += UPD_THREADS) {
    const int nb = min(UPD_THREADS, B - base);
    int64_t node = -1;
    float val = 0.0f;
    if (tid < nb) {
      node = tree_idx[base + tid];
      float r = raw[base + tid];
      if (omega_is_applied) val = r;
      else if (omega == 0.5f) val = __fsqrt_rn(r);
      else if (omega == 1.0f) val = r;
      else val = (float)pow((double)r, (double)omega);
      if (node < tree_start || node >= len) {
        if (status) atomicExch(status, 1);
        node = -1;
      }
    }
    s_idx[tid] = node;
    __syncthreads();
    if (node >= 0) {
      bool wins = true;
      for (int j = tid + 1; j < nb; ++j) wins &= (s_idx[j] != node);
      if (wins) __stcg(&tree[node], val);
      block_max = fmaxf(block_max, val);
    }
    __syncthreads();
    // every valid thread sits on the leaf level: same number of levels for all
    const int L = tree_depth(tree_start);
    for (int lev = 0; lev < L; ++lev) {
      if (node >= 0) {
        node = (node - 1) >> 1;
        float l = __ldcg(&tree[2 * node + 1]);
        float r = __ldcg(&tree[2 * node + 2]);
        __stcg(&tree[node], __fadd_rn(l, r));
      }
      __syncthreads();
    }
  }
  // running max (memory.py:47-48)
  float m = warp_max(block_max);
  if ((tid & 31) == 0) s_red[tid >> 5] = m;
  __syncthreads();
  if (tid < 32) {
    m = warp_max(s_red[tid]);
    if (tid == 0 && m > *running_max) *running_max = m;
  }
}

// Fast path for B <= 32 (the learner's batch): ONE warp, no barriers.  Every lane first fetches all L siblings
// of its leaf-to-root path in one batch of independent loads (they are untouched by this kernel unless another
// lane's path owns them), then the warp walks the levels in registers: lanes that share a parent find each other
// with __match_any_sync, take the sibling value from the partner lane when the sibling is itself on an updated
// path (else from the prefetched value), and the lowest lane of each group writes the node.  L dependent global
// round trips (one per level, with a CTA barrier each) become one.
constexpr int UPD_MAX_LEVELS = 30;

__global__ void __launch_bounds__(32, 1)
k_tree_update_warp(float* tree, int64_t tree_start, int64_t size, const int64_t* __restrict__ tree_idx,
                   const float* __restrict__ raw, float omega, int omega_is_applied, int B, float* running_max,
                   int32_t* status, const int32_t* __restrict__ gate) {
  if (gate && *gate == 0) return;   // rejected batch (see k_tree_update)
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x;
  const int64_t len = tree_start + size;
  const int L = tree_depth(tree_start);
  int64_t node = -1;
  float val = 0.0f;
  if (lane < B) {
    node = tree_idx[lane];
    float r = raw[lane];
    if (omega_is_applied) val = r;
    else if (omega == 0.5f) val = __fsqrt_rn(r);
    else if (omega == 1.0f) val = r;
    else val = (float)pow((double)r, (double)omega);
    if (node < tree_start || node >= len) {
      if (status) atomicExch(status, 1);
      node = -1;
    }
  }
  const bool active = node >= 0;
  float vmax = active ? val : -CUDART_INF_F;
  vmax = warp_max(vmax);
  // duplicates: the highest lane (= last in index order) wins, memory.py:45 fancy assignment
  {
    const int key = active ? (int)node : -(lane + 1);   // node indices fit 31 bits (checked by the launcher)
    const unsigned grp = __match_any_sync(full, key);
    const int winner = 31 - __clz(grp);
    val = __shfl_sync(full, val, winner);
  }
  // prefetch the siblings along the path (independent loads)
  float sib[UPD_MAX_LEVELS];
#pragma unroll
  for (int l = 0; l < UPD_MAX_LEVELS; ++l) {
    sib[l] = 0.0f;
    if (l < L && active) {
      const int64_t nl = ((node + 1) >> l) - 1;           // ancestor l levels up
      const int64_t sn = (nl & 1) ? nl + 1 : nl - 1;      // odd index = left child
      sib[l] = __ldcg(tree + sn);
    }
  }
  {
    const int key = active ? (int)node : -(lane + 1);
    const unsigned grp = __match_any_sync(full, key);
    if (active && lane == __ffs(grp) - 1) __stcg(tree + node, val);
  }
#pragma unroll
  for (int l = 0; l < UPD_MAX_LEVELS; ++l) {
    if (l < L) {
      const int64_t parent = active ? ((node - 1) >> 1) : -(int64_t)(lane + 1);
      const bool is_left = active && (node & 1);
      const unsigned grp = __match_any_sync(full, (int)parent);
      const unsigned lefts = __ballot_sync(full, is_left);
      const unsigned other = grp & (is_left ? ~lefts : lefts);
      const float partner = __shfl_sync(full, val, other ? __ffs(other) - 1 : lane);
      const float sv = other ? partner : sib[l];
      val = __fadd_rn(val, sv);                            // fl32(left + right); float addition commutes
      node = parent;
      if (active && lane == __ffs(grp) - 1) __stcg(tree + node, val);
    }
  }
  if (lane == 0 && vmax > *running_max) *running_max = vmax;   // memory.py:47-48
}

// ================================================================================================
// Tree descent shared by K1 (sample) and rb_tree_find.
// ================================================================================================
// A warp walks one sample.  The top TOP_DEPTH levels are staged in shared memory by the CTA; below
// that the warp fetches up to five levels of the current subtree at once: relative to node i the
// nodes of depth j form the contiguous run [(i+1)*2^j - 1, (i+1)*2^j - 1 + 2^j), so lanes 2..31
// fetch depths 1..4 (30 nodes) and all 32 lanes fetch depth 5 as one 128-byte line.  The five
// compare/subtract steps then run on register values exchanged with shuffles: one memory round
// trip per five levels instead of five.
constexpr int TOP_DEPTH = 10;                        // depths 0..10 staged: 2047 nodes, 8 KB
constexpr int TOP_NODES = (2 << TOP_DEPTH) - 1;

struct Descent {
  int64_t node;
  float prob;
};

__device__ __forceinline__ Descent warp_descend(const float* __restrict__ tree, const float* s_top, int64_t tree_start,
                                                int64_t len, int L, double v) {
  const int lane = threadIdx.x & 31;
  int64_t i = 0;
  int d = 0;
  const int S = min(L, TOP_DEPTH);
  // ---- shared-memory phase (all lanes redundantly, uniform) ----
  for (; d < S; ++d) {
    int64_t cl = 2 * i + 1, cr = cl + 1;
    if (cl >= tree_start) {  // children are leaves: clip like memory.py:70-71
      cl = min(cl, len - 1);
      cr = min(cr, len - 1);
    }
    float left = s_top[cl];
    bool right = v > (double)left;
    if (right) v = __dsub_rn(v, (double)left);
    i = right ? cr : cl;
  }
  float prob = (L <= TOP_DEPTH) ? s_top[i] : 0.0f;
  // ---- chunked phase ----
  while (d < L) {
    const int nl = min(5, L - d);
    float lo = 0.0f, hi = 0.0f;
    {
      int h = lane;  // subtree positions 2..31 -> depths 1..4
      if (h >= 2) {
        int j = 31 - __clz(h);
        if (j <= nl) {
          int64_t nd = (i << j) + h - 1;
          if (d + j == L) nd = min(nd, len - 1);
          lo = __ldg(tree + nd);
        }
      }
      h = lane + 32;  // positions 32..63 -> depth 5
      if (nl == 5) {
        int64_t nd = (i << 5) + h - 1;
        if (d + 5 == L) nd = min(nd, len - 1);
        hi = __ldg(tree + nd);
      }
    }
    int h = 1;
    for (int j = 0; j < nl; ++j) {
      int hl = 2 * h;
      float a = __shfl_sync(0xffffffffu, lo, hl & 31);
      float b = __shfl_sync(0xffffffffu, hi, hl & 31);
      float left = (hl < 32) ? a : b;
      bool right = v > (double)left;
      if (right) v = __dsub_rn(v, (double)left);
      h = hl + (right ? 1 : 0);
    }
    {
      float a = __shfl_sync(0xffffffffu, lo, h & 31);
      float b = __shfl_sync(0xffffffffu, hi, h & 31);
      prob = (h < 32) ? a : b;
    }
    i = (i << nl) + h - 1;
    d += nl;
    if (d == L) i = min(i, len - 1);
  }
  Descent r;
  r.node = i;
  r.prob = prob;
  return r;
}

__device__ __forceinline__ void stage_top(const float* __restrict__ tree, float* s_top, int64_t len) {
  const int ntop = (int)min((int64_t)TOP_NODES, len);
  for (int i = threadIdx.x; i < ntop; i += blockDim.x) s_top[i] = __ldg(tree + i);
  __syncthreads();
}

constexpr int SAMPLE_THREADS = 1024;

__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
k_tree_find(const float* __restrict__ tree, int64_t tree_start, int64_t size, const double* __restrict__ values,
            int B, float* probs, int64_t* data_idx, int64_t* tree_idx) {
  __shared__ float s_top[TOP_NODES];
  const int64_t len = tree_start + size;
  const int L = tree_depth(tree_start);
  stage_top(tree, s_top, len);
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (int k = blockIdx.x * nwarps + warp; k < B; k += gridDim.x * nwarps) {
    Descent r = warp_descend(tree, s_top, tree_start, len, L, values[k]);
    if (lane == 0) {
      probs[k] = r.prob;
      data_idx[k] = r.node - tree_start;
      tree_idx[k] = r.node;
    }
  }
}

// ================================================================================================
// K1  tree_sample : stratified proportional sampling with whole-batch rejection + IS weights.
// ================================================================================================
__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
k_tree_sample(const float* __restrict__ tree, int64_t tree_start, int64_t size, const int64_t* __restrict__ ring_state,
              int n, int history, const double* __restrict__ u01, int u01_attempts, uint64_t seed,
              unsigned long long* rng_counter, int B, float beta, const float* __restrict__ beta_dev, int max_attempts,
              float* probs, int64_t* data_idx, int64_t* tree_idx, float* weights, int32_t* status) {
  __shared__ float s_top[TOP_NODES];
  __shared__ int s_valid;
  __shared__ float s_red[32];
  __shared__ float s_prob[SAMPLE_THREADS];   // leaf values of the first SAMPLE_THREADS samples (kept on chip for the weights)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
  const int64_t len = tree_start + size;
  const int L = tree_depth(tree_start);
  if (tid == 0) s_valid = 1;
  // every scalar the kernel needs is requested before the staging barrier, so these round trips overlap the staging loads
  const int64_t head = ring_state[0];
  const bool full = ring_state[1] != 0;
  const unsigned long long ctr0 = (u01 == nullptr) ? *rng_counter : 0ull;
  const float b = beta_dev ? *beta_dev : beta;
  stage_top(tree, s_top, len);

  const float p_total = s_top[0];                          // memory.py:149
  const float seg = __fdiv_rn(p_total, (float)B);          // memory.py:125 (float32)
  const double segd = (double)seg;
  const int tries = (u01 != nullptr) ? u01_attempts : max_attempts;

  int attempt = 0;
  bool ok_batch = false;
  for (; attempt < tries; ++attempt) {
    for (int k = warp; k < B; k += nwarps) {
      double u;
      if (u01 != nullptr) {
        u = u01[(size_t)attempt * B + k];
      } else {
        unsigned long long c = ctr0 + (unsigned long long)attempt;
        uint4 r = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), (uint32_t)k, 0x5A4D504Cu),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
        u = u53(r.x, r.y);
      }
      // memory.py:126,129: uniform(0, seg) + k*seg, float64, separately rounded
      double v = __dadd_rn(__dadd_rn(0.0, __dmul_rn(segd, u)), __dmul_rn((double)k, segd));
      Descent r = warp_descend(tree, s_top, tree_start, len, L, v);
      if (lane == 0) {
        int64_t di = r.node - tree_start;
        probs[k] = r.prob;
        if (k < SAMPLE_THREADS) s_prob[k] = r.prob;
        data_idx[k] = di;
        tree_idx[k] = r.node;
        bool ok = (pymod(head - di, size) > (int64_t)n) && (pymod(di - head, size) >= (int64_t)history) &&
                  (r.prob != 0.0f);                         // memory.py:131
        if (!ok) s_valid = 0;
      }
    }
    __syncthreads();
    ok_batch = (s_valid != 0);
    __syncthreads();
    if (ok_batch) { ++attempt; break; }
    if (tid == 0) s_valid = 1;
    __syncthreads();
  }

  // importance-sampling weights (memory.py:151-154), float32 like numpy
  const float nb = -b;
  const float count = (float)(full ? size : head);
  float wmax = -CUDART_INF_F;
  float w_first = 0.0f;   // weight of sample k = tid (kept in a register), later samples go through global memory
  for (int k = tid; k < B; k += blockDim.x) {
    float p = __fdiv_rn(k < SAMPLE_THREADS ? s_prob[k] : probs[k], p_total);
    float w = (float)pow((double)__fmul_rn(count, p), (double)nb);
    if (k == tid) w_first = w; else weights[k] = w;
    wmax = fmaxf(wmax, w);
  }
  wmax = warp_max(wmax);
  if (lane == 0) s_red[warp] = wmax;
  __syncthreads();
  wmax = warp_max(s_red[lane]);
  // A batch that is still invalid after the last allowed redraw (the reference would keep redrawing, memory.py:128-132)
  // must not train anything: its weights are zeroed -- so the loss gradient is exactly zero -- and status[0] = 0 gates
  // the optimiser step and the priority write-back (rb_clip_adam / rb_tree_update `gate`).
  for (int k = tid; k < B; k += blockDim.x)
    weights[k] = ok_batch ? __fdiv_rn(k == tid ? w_first : weights[k], wmax) : 0.0f;
  if (tid == 0) {
    status[0] = ok_batch ? 1 : 0;
    status[1] = attempt;
    if (!ok_batch && u01 == nullptr) status[2] = status[2] + 1;   // batches rejected for good so far (host diagnostics)
    if (u01 == nullptr) *rng_counter = ctr0 + (unsigned long long)attempt;
  }
}

// ================================================================================================
// K2  gather : frame-stack + n-step window gather with episode-boundary blanking.
// ================================================================================================
// grid = (used_slots * split, B).  A CTA converts (a slice of) ONE stored uint8 frame and writes it
// to every place it appears in the outputs (state slot and/or next-state slot), so each stored frame
// is read once.  16-byte loads, 4 x 16-byte stores per thread-iteration.
constexpr int GATHER_THREADS = 256;
constexpr int FRAME_VEC = RB_FRAME_BYTES / 16;  // 441 uint4 per frame

// bit k: record idx - (history - 1) + k starts an episode, for k < W
__device__ __forceinline__ uint64_t window_first_bits(const int32_t* __restrict__ timestep, int64_t size, int64_t idx,
                                                      int history, int W) {
  // lane s (and s+32) looks at window record s; ballot -> 64-bit "timestep == 0" mask (memory.py:114)
  const int lane = threadIdx.x & 31;
  bool f0 = false, f1 = false;
  if (lane < W) f0 = __ldg(timestep + pymod(idx - (history - 1) + lane, size)) == 0;
  if (lane + 32 < W) f1 = __ldg(timestep + pymod(idx - (history - 1) + lane + 32, size)) == 0;
  uint32_t b0 = __ballot_sync(0xffffffffu, f0), b1 = __ballot_sync(0xffffffffu, f1);
  return (uint64_t)b0 | ((uint64_t)b1 << 32);
}

__host__ __device__ __forceinline__ uint64_t low_bits(int k) {  // k in [0,64]
  return k >= 64 ? ~0ull : ((1ull << k) - 1ull);
}

// memory.py:116-119: slot s < H-1 is blank if any of s+1..H-1 starts an episode; slot s >= H is blank
// if any of H..s starts one; slot H-1 never is.
__device__ __forceinline__ bool slot_blank(uint64_t first, int s, int history) {
  if (s < history - 1) return (first & low_bits(history) & ~low_bits(s + 1)) != 0;
  if (s >= history) return (first & low_bits(s + 1) & ~low_bits(history)) != 0;
  return false;
}

__device__ __forceinline__ float4 u8x4_to_unit(uint32_t w) {
  return make_float4(__fdiv_rn((float)(w & 0xffu), 255.0f), __fdiv_rn((float)((w >> 8) & 0xffu), 255.0f),
                     __fdiv_rn((float)((w >> 16) & 0xffu), 255.0f), __fdiv_rn((float)(w >> 24), 255.0f));
}

// rb_gather_horizon: every gather body takes n (the n_max the grid and the blanking window are sized for) and gamma_pow
// from its arguments when HZ is false, and n_t = clamp(hz->n, 1, n_max), gamma_pow and gamma_n from the schedule's
// current row when it is true.  Window slots the grid holds for n_max but n_t does not use -- used slots
// >= H + min(n_t, H) -- exit at once; the rest map as for a launch with n = n_t.  A slot's blanking depends only on the
// slots between it and slot H - 1, so the wider ballot changes nothing.
//
// What a gather CTA knows of its sample and window slot.  gather_slot fills it, or returns false for a slot the current n
// does not use.
struct GatherSlot {
  int n, W, s, b, part;          // horizon in use; ballot width history + n_max; window slot; sample; part of the split
  const float* gamma_pow;
  float gamma_n;                 // 1 unless HZ
  int64_t idx, rec0, pos;        // the sample's data index; that of window slot 0; that of slot s, wrapped
  const uint4* src;              // the stored frame of slot s

  // where slot s appears in output row `row` (copy * B + b) of `states` / `next_states`, nullptr where it does not
  __device__ __forceinline__ float4* state_dst(float* __restrict__ states, size_t row, int history) const {
    return s < history ? reinterpret_cast<float4*>(states + (row * history + s) * RB_FRAME_BYTES) : nullptr;
  }
  __device__ __forceinline__ float4* next_state_dst(float* __restrict__ next_states, size_t row, int history) const {
    const int s = this->s, n = this->n;   // as values: through `this` the compares compile in another order
    return (s >= n && s < n + history)
               ? reinterpret_cast<float4*>(next_states + (row * history + (s - n)) * RB_FRAME_BYTES)
               : nullptr;
  }
};

// TRUNC (rb_gather_trunc): k = the offset of the first final-observation record (nonterminal byte RB_NONTERMINAL_FINAL) in
// records idx + 1 .. idx + n - 1, or n if there is none, from a 64-bit ballot like window_first_bits'.  Every warp forms it
// itself, so the CTA needs no barrier before it maps its slot.
__device__ __forceinline__ int first_final(const uint8_t* __restrict__ nonterminal, int64_t size, int64_t idx, int n) {
  const int lane = threadIdx.x & 31;
  bool f0 = false, f1 = false;
  if (lane < n - 1) f0 = __ldg(nonterminal + pymod(idx + 1 + lane, size)) == RB_NONTERMINAL_FINAL;
  if (lane + 32 < n - 1) f1 = __ldg(nonterminal + pymod(idx + 33 + lane, size)) == RB_NONTERMINAL_FINAL;
  const uint64_t m = (uint64_t)__ballot_sync(0xffffffffu, f0) | ((uint64_t)__ballot_sync(0xffffffffu, f1) << 32);
  return m ? __ffsll((long long)m) : n;   // bit j is record idx + 1 + j, so the first set bit's 1-based position is k
}

// TRUNC: the window is then gathered exactly as at n = k, with the nonterminal in discount form at gamma_k, which is the
// row's gamma_pow[k] for k < n (fl32(gamma ** k), the gamma_n of a horizon of k steps) and its gamma_n for k = n.
template <bool HZ, bool TRUNC = false>
__device__ __forceinline__ bool gather_slot(GatherSlot& g, int64_t size, const int64_t* __restrict__ data_idx, int history,
                                            int n, const float* __restrict__ gamma_pow, int split,
                                            const rb_horizon* __restrict__ hz,
                                            const uint8_t* __restrict__ nonterminal = nullptr) {
  g.b = blockIdx.y;
  g.W = history + n;
  g.n = n; g.gamma_pow = gamma_pow; g.gamma_n = 1.0f;
  if constexpr (HZ) { g.n = min(max(__ldg(&hz->n), 1), n); g.gamma_pow = hz->gamma_pow; g.gamma_n = __ldg(&hz->gamma_n); }
  if constexpr (TRUNC) {
    const int k = first_final(nonterminal, size, data_idx[g.b], g.n);
    if (k < g.n) { g.gamma_n = __ldg(g.gamma_pow + k); g.n = k; }
  }
  const int used = blockIdx.x / split;
  g.part = blockIdx.x % split;
  if (HZ && used >= history + min(g.n, history)) return false;
  // used-slot -> window slot: slots [0,H) feed `states`, [n,n+H) feed `next_states`
  g.s = (g.n >= history && used >= history) ? g.n + (used - history) : used;
  g.idx = data_idx[g.b];
  g.rec0 = g.idx - (history - 1);
  g.pos = pymod(g.rec0 + g.s, size);
  return true;
}

// Loads this thread's first vector of the caller's range [v0, v1) of the frame, and has warp 0 ballot the window's
// episode starts into s_first; the caller syncs before reading it.  Issue the (rarely discarded) frame load first so it
// overlaps the timestep loads that decide the blanking.
__device__ __forceinline__ uint4 gather_prefetch(GatherSlot& g, const uint8_t* __restrict__ frames,
                                                 const int32_t* __restrict__ timestep, int64_t size, int history, int v0,
                                                 int v1, uint64_t& s_first) {
  g.src = reinterpret_cast<const uint4*>(frames + (size_t)g.pos * RB_FRAME_BYTES);
  uint4 pre = make_uint4(0, 0, 0, 0);
  if (v0 + (int)threadIdx.x < v1) pre = __ldg(g.src + v0 + threadIdx.x);
  if (threadIdx.x < 32) {
    uint64_t f = window_first_bits(timestep, size, g.rec0, 1, g.W);   // the W records from slot 0's
    if (threadIdx.x == 0) s_first = f;
  }
  return pre;
}

// per-sample scalars, once per sample (memory.py:140-145).  HZ (rb_gather_horizon): the nonterminal is written in discount
// form, fl32(nonterminal * gamma_n), i.e. gamma_n or +0.
template <bool HZ>
__device__ __forceinline__ void gather_scalars(const GatherSlot& g, uint64_t first, const int32_t* __restrict__ action,
                                               const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal,
                                               int64_t size, int history, int64_t* __restrict__ actions,
                                               float* __restrict__ returns, float* __restrict__ nonterminals) {
  const int sa = history - 1;
  actions[g.b] = (int64_t)__ldg(action + pymod(g.idx, size));  // slot H-1 is never blanked
  float acc = 0.0f;
  for (int k = 0; k < g.n; ++k) {
    int sk = sa + k;
    float r = slot_blank(first, sk, history) ? 0.0f : __ldg(reward + pymod(g.idx + k, size));
    acc = __fadd_rn(acc, __fmul_rn(r, __ldg(g.gamma_pow + k)));
  }
  returns[g.b] = acc;
  const int sl = history + g.n - 1;
  const float nt = slot_blank(first, sl, history) ? 0.0f : (__ldg(nonterminal + pymod(g.idx + g.n, size)) ? 1.0f : 0.0f);
  if constexpr (HZ) nonterminals[g.b] = __fmul_rn(nt, g.gamma_n);
  else nonterminals[g.b] = nt;
}

template <bool HZ, bool TRUNC = false>
__device__ __forceinline__ void
gather_body(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
            const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal, int64_t size,
            const int64_t* __restrict__ data_idx, int history, int n, const float* __restrict__ gamma_pow,
            float* __restrict__ states, float* __restrict__ next_states, int64_t* __restrict__ actions,
            float* __restrict__ returns, float* __restrict__ nonterminals, int split, const rb_horizon* __restrict__ hz) {
  __shared__ uint64_t s_first;
  GatherSlot g;
  if (!gather_slot<HZ, TRUNC>(g, size, data_idx, history, n, gamma_pow, split, hz, nonterminal)) return;
  const int per = (FRAME_VEC + split - 1) / split;
  const int v0 = g.part * per, v1 = min(FRAME_VEC, v0 + per);
  const uint4 pre = gather_prefetch(g, frames, timestep, size, history, v0, v1, s_first);
  __syncthreads();
  const uint64_t first = s_first;
  const bool blank = slot_blank(first, g.s, history);

  float4* dst_s = g.state_dst(states, (size_t)g.b, history);
  float4* dst_n = g.next_state_dst(next_states, (size_t)g.b, history);
  for (int v = v0 + threadIdx.x; v < v1; v += GATHER_THREADS) {
    uint4 q = blank ? make_uint4(0, 0, 0, 0) : (v == v0 + (int)threadIdx.x ? pre : __ldg(g.src + v));
    float4 a = u8x4_to_unit(q.x), bq = u8x4_to_unit(q.y), c = u8x4_to_unit(q.z), d = u8x4_to_unit(q.w);
    if (dst_s) {
      __stcs(dst_s + 4 * v + 0, a); __stcs(dst_s + 4 * v + 1, bq); __stcs(dst_s + 4 * v + 2, c); __stcs(dst_s + 4 * v + 3, d);
    }
    if (dst_n) {
      __stcs(dst_n + 4 * v + 0, a); __stcs(dst_n + 4 * v + 1, bq); __stcs(dst_n + 4 * v + 2, c); __stcs(dst_n + 4 * v + 3, d);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    gather_scalars<HZ>(g, first, action, reward, nonterminal, size, history, actions, returns, nonterminals);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
         const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal, int64_t size,
         const int64_t* __restrict__ data_idx, int B, int history, int n, const float* __restrict__ gamma_pow,
         float* __restrict__ states, float* __restrict__ next_states, int64_t* __restrict__ actions,
         float* __restrict__ returns, float* __restrict__ nonterminals, int split) {
  gather_body<false>(frames, timestep, action, reward, nonterminal, size, data_idx, history, n, gamma_pow, states,
                     next_states, actions, returns, nonterminals, split, nullptr);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_hz(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
            const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal, int64_t size,
            const int64_t* __restrict__ data_idx, int B, int history, int n_max, const rb_horizon* __restrict__ hz,
            float* __restrict__ states, float* __restrict__ next_states, int64_t* __restrict__ actions,
            float* __restrict__ returns, float* __restrict__ nonterminals, int split) {
  gather_body<true>(frames, timestep, action, reward, nonterminal, size, data_idx, history, n_max, nullptr, states,
                    next_states, actions, returns, nonterminals, split, hz);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_hz_trunc(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep,
                  const int32_t* __restrict__ action, const float* __restrict__ reward,
                  const uint8_t* __restrict__ nonterminal, int64_t size, const int64_t* __restrict__ data_idx, int B,
                  int history, int n_max, const rb_horizon* __restrict__ hz, float* __restrict__ states,
                  float* __restrict__ next_states, int64_t* __restrict__ actions, float* __restrict__ returns,
                  float* __restrict__ nonterminals, int split) {
  gather_body<true, true>(frames, timestep, action, reward, nonterminal, size, data_idx, history, n_max, nullptr, states,
                          next_states, actions, returns, nonterminals, split, hz);
}

// ================================================================================================
// K2s gather_shift : k_gather + random-shift augmentation (DrQ): every observation is edge-padded by `pad` pixels and
// cropped back to 84 x 84 at its own offset (oy, ox) in [0, 2 pad]:  out[y][x] = in[clamp(y+oy-pad)][clamp(x+ox-pad)].
// ================================================================================================
// Same grid and CTA-per-stored-frame mapping as k_gather, but the split is by output rows (at split 2 part 0 writes rows
// [0, 42), part 1 rows [42, 84)).  The input rows those outputs can reach under any offset -- the CTA's rows and `pad` more
// on either side -- are staged once in shared memory with 16-byte loads; then each appearance of the frame (state and/or
// next state) is written from there with its own observation's offset.  An output row is 21 float4, so each streaming
// float4 store lies inside one row.
// Offsets: one Philox4x32-10 call per sample b, counter (c_lo, c_hi, b, SHIFT_STREAM) with c = *rng_counter (advanced by
// rb_tree_sample just before), key = seed; words x, y -> the state's (oy, ox), z, w -> the next state's;
// offset = (word * (2 pad + 1)) >> 32.  The kernels are k_gather_aug's body with one copy of each side and no intensity.
constexpr int FRAME_SIDE = 84;
constexpr int ROW_VEC = FRAME_SIDE / 4;              // float4 per output row
constexpr uint32_t SHIFT_STREAM = 0x53484654u;       // "SHFT": apart from sampling (0x5A4D504C) and noise (0x4E4F4953 + i)

__device__ __forceinline__ int clamp_px(int v) { return min(max(v, 0), FRAME_SIDE - 1); }

__device__ __forceinline__ int shift_offset(uint32_t word, int pad) {
  return (int)(((uint64_t)word * (uint64_t)(2 * pad + 1)) >> 32);
}

// four output pixels (y, x .. x+3) of a frame staged in shared memory, shifted by (dy, dx)
__device__ __forceinline__ float4 shifted4(const uint8_t* s_frame, int y, int x, int dy, int dx) {
  const uint8_t* row = s_frame + clamp_px(y + dy) * FRAME_SIDE;
  return make_float4(__fdiv_rn((float)row[clamp_px(x + dx)], 255.0f), __fdiv_rn((float)row[clamp_px(x + 1 + dx)], 255.0f),
                     __fdiv_rn((float)row[clamp_px(x + 2 + dx)], 255.0f), __fdiv_rn((float)row[clamp_px(x + 3 + dx)], 255.0f));
}

// ================================================================================================
// K2a gather_aug : k_gather_shift generalised to M copies of every state and K copies of every next state (DrQ's K / M),
// each copy with its own shift offset and its own intensity multiplier (SPR's intensity augmentation):
//   out = fl32(fl32(in / 255) * mult),  mult = fma(s, clamp(N(0, 1), -2, 2), 1)   (no multiply at all when s == 0)
// ================================================================================================
// Same grid, CTA-per-stored-frame mapping and row split as k_gather_shift: the reachable input rows are staged once, then
// every copy of each appearance of the frame is written from shared memory (copy j of the state to rows [jB, (j+1)B) of
// `states`, copy k of the next state to rows [kB, (k+1)B) of `next_states`).
// Draws, counter word 3 = the stream; c = *rng_counter as rb_tree_sample left it, key = seed:
//   copy j offsets     (c_lo, c_hi, b, SHIFT_STREAM + j): x, y -> the state's (oy, ox), z, w -> the next state's (copy 0's
//                      are k_gather_shift's);
//   copy j multiplier  (c_lo, c_hi, b, INTS_STREAM + j): box_muller(x, y).x -> the state's, box_muller(z, w).x -> the next
//                      state's.
// The streams in use: sampling 0x5A4D504C, noise 0x4E4F4953 + i (i < RB_MAX_NOISY_LAYERS), shift 0x53484654 + j and
// intensity 0x494E5453 + j (j < RB_MAX_AUG_COPIES), parameter reset 0x52534554 ("RSET", k_param_reset), recycling 0x5245444F
// ("REDO", k_redo_recycle): the six ranges [0x494E5453, 0x494E545A], [0x4E4F4953, 0x4E4F495A], {0x5245444F}, {0x52534554},
// [0x53484654, 0x5348465B] and {0x5A4D504C} are disjoint.
constexpr uint32_t INTS_STREAM = 0x494E5453u;        // "INTS"

__device__ __forceinline__ float4 aug4(const uint8_t* s_frame, int y, int x, int dy, int dx, bool scaled, float mult) {
  float4 v = shifted4(s_frame, y, x, dy, dx);
  if (scaled) v = make_float4(__fmul_rn(v.x, mult), __fmul_rn(v.y, mult), __fmul_rn(v.z, mult), __fmul_rn(v.w, mult));
  return v;
}

__device__ __forceinline__ float intensity_mult(float s, float normal) {
  return __fmaf_rn(s, fminf(fmaxf(normal, -2.0f), 2.0f), 1.0f);
}

// SHIFT (k_gather_shift*): one copy of each side and no intensity, fixed at compile time; `scales` is neither read nor
// written.  Copy 0 draws from SHIFT_STREAM + 0 and [2][1][B][2] is the [2][B][2] offsets layout, so the draws and
// `shifts` are those documented for k_gather_shift above.
template <bool HZ, bool SHIFT, bool TRUNC = false>
__device__ __forceinline__ void
gather_aug_body(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
                const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal, int64_t size,
                const int64_t* __restrict__ data_idx, int B, int history, int n, const float* __restrict__ gamma_pow,
                float* __restrict__ states, float* __restrict__ next_states, int64_t* __restrict__ actions,
                float* __restrict__ returns, float* __restrict__ nonterminals, int split, int pad, float intensity,
                int m_copies, int k_copies, uint64_t seed, const unsigned long long* __restrict__ rng_counter,
                int32_t* __restrict__ shifts, float* __restrict__ scales, const rb_horizon* __restrict__ hz) {
  constexpr int MAX_COPIES = SHIFT ? 1 : RB_MAX_AUG_COPIES;
  __shared__ uint64_t s_first;
  __shared__ int s_off[2][MAX_COPIES][2];   // (side, copy, (dy, dx)) = offset - pad
  __shared__ float s_mult[2][MAX_COPIES];
  __shared__ __align__(16) uint8_t s_frame[RB_FRAME_BYTES];
  GatherSlot g;
  if (!gather_slot<HZ, TRUNC>(g, size, data_idx, history, n, gamma_pow, split, hz, nonterminal)) return;
  const int b = g.b, s = g.s;
  const int copies = SHIFT ? 1 : max(m_copies, k_copies);
  const bool scaled = !SHIFT && intensity > 0.0f;
  const int rows = (FRAME_SIDE + split - 1) / split;
  const int r0 = g.part * rows, r1 = min(FRAME_SIDE, r0 + rows);
  // the 16-byte vectors covering input rows [r0 - pad, r1 + pad) (a frame starts on a 16-byte boundary: 7056 = 441 x 16)
  const int v0 = max(r0 - pad, 0) * FRAME_SIDE / 16;
  const int v1 = min(FRAME_VEC, (min(r1 + pad, FRAME_SIDE) * FRAME_SIDE + 15) / 16);
  const uint4 pre = gather_prefetch(g, frames, timestep, size, history, v0, v1, s_first);
  if (threadIdx.x >= 32 && threadIdx.x < 32 + copies) {   // one thread per copy draws its offsets and multipliers
    const int j = threadIdx.x - 32;
    const unsigned long long c = *rng_counter;
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    int oy_s = 0, ox_s = 0, oy_n = 0, ox_n = 0;
    if (pad > 0) {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), (uint32_t)b, SHIFT_STREAM + (uint32_t)j), key);
      oy_s = shift_offset(r.x, pad); ox_s = shift_offset(r.y, pad);
      oy_n = shift_offset(r.z, pad); ox_n = shift_offset(r.w, pad);
    }
    float m_s = 1.0f, m_n = 1.0f;
    if (scaled) {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), (uint32_t)b, INTS_STREAM + (uint32_t)j), key);
      m_s = intensity_mult(intensity, box_muller(r.x, r.y).x);
      m_n = intensity_mult(intensity, box_muller(r.z, r.w).x);
    }
    s_off[0][j][0] = oy_s - pad; s_off[0][j][1] = ox_s - pad;
    s_off[1][j][0] = oy_n - pad; s_off[1][j][1] = ox_n - pad;
    s_mult[0][j] = m_s; s_mult[1][j] = m_n;
    if (blockIdx.x == 0) {   // int32 [2][copies][B][2] and float32 [2][copies][B]: (side, copy, sample)
      int32_t* sh_s = shifts + 2 * ((size_t)j * B + b);
      int32_t* sh_n = shifts + 2 * ((size_t)(copies + j) * B + b);
      sh_s[0] = oy_s; sh_s[1] = ox_s;
      sh_n[0] = oy_n; sh_n[1] = ox_n;
      if constexpr (!SHIFT) {
        scales[(size_t)j * B + b] = m_s;
        scales[(size_t)(copies + j) * B + b] = m_n;
      }
    }
  }
  __syncthreads();
  const uint64_t first = s_first;
  const bool blank = slot_blank(first, s, history);
  if (!blank) {
    uint4* dst = reinterpret_cast<uint4*>(s_frame);
    for (int v = v0 + threadIdx.x; v < v1; v += GATHER_THREADS) dst[v] = (v == v0 + (int)threadIdx.x) ? pre : __ldg(g.src + v);
  }
  __syncthreads();

  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = 0; j < copies; ++j) {
    float4* dst_s = j < m_copies ? g.state_dst(states, (size_t)j * B + b, history) : nullptr;
    float4* dst_n = j < k_copies ? g.next_state_dst(next_states, (size_t)j * B + b, history) : nullptr;
    const int dy_s = s_off[0][j][0], dx_s = s_off[0][j][1], dy_n = s_off[1][j][0], dx_n = s_off[1][j][1];
    const float m_s = s_mult[0][j], m_n = s_mult[1][j];
    for (int i = r0 * ROW_VEC + threadIdx.x; i < r1 * ROW_VEC; i += GATHER_THREADS) {
      const int y = i / ROW_VEC, x = (i - y * ROW_VEC) * 4;
      if (dst_s) __stcs(dst_s + i, blank ? zero : aug4(s_frame, y, x, dy_s, dx_s, scaled, m_s));
      if (dst_n) __stcs(dst_n + i, blank ? zero : aug4(s_frame, y, x, dy_n, dx_n, scaled, m_n));
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    gather_scalars<HZ>(g, first, action, reward, nonterminal, size, history, actions, returns, nonterminals);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_shift(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
               const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal, int64_t size,
               const int64_t* __restrict__ data_idx, int B, int history, int n, const float* __restrict__ gamma_pow,
               float* __restrict__ states, float* __restrict__ next_states, int64_t* __restrict__ actions,
               float* __restrict__ returns, float* __restrict__ nonterminals, int split, int pad, uint64_t seed,
               const unsigned long long* __restrict__ rng_counter, int32_t* __restrict__ shifts) {
  gather_aug_body<false, true>(frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n, gamma_pow,
                               states, next_states, actions, returns, nonterminals, split, pad, 0.0f, 1, 1, seed,
                               rng_counter, shifts, nullptr, nullptr);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_shift_hz(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep,
                  const int32_t* __restrict__ action, const float* __restrict__ reward,
                  const uint8_t* __restrict__ nonterminal, int64_t size, const int64_t* __restrict__ data_idx, int B,
                  int history, int n_max, const rb_horizon* __restrict__ hz, float* __restrict__ states,
                  float* __restrict__ next_states, int64_t* __restrict__ actions, float* __restrict__ returns,
                  float* __restrict__ nonterminals, int split, int pad, uint64_t seed,
                  const unsigned long long* __restrict__ rng_counter, int32_t* __restrict__ shifts) {
  gather_aug_body<true, true>(frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max, nullptr,
                              states, next_states, actions, returns, nonterminals, split, pad, 0.0f, 1, 1, seed,
                              rng_counter, shifts, nullptr, hz);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_aug(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
             const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal, int64_t size,
             const int64_t* __restrict__ data_idx, int B, int history, int n, const float* __restrict__ gamma_pow,
             float* __restrict__ states, float* __restrict__ next_states, int64_t* __restrict__ actions,
             float* __restrict__ returns, float* __restrict__ nonterminals, int split, int pad, float intensity, int m_copies,
             int k_copies, uint64_t seed, const unsigned long long* __restrict__ rng_counter, int32_t* __restrict__ shifts,
             float* __restrict__ scales) {
  gather_aug_body<false, false>(frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n, gamma_pow,
                                states, next_states, actions, returns, nonterminals, split, pad, intensity, m_copies,
                                k_copies, seed, rng_counter, shifts, scales, nullptr);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_aug_hz(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
                const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal, int64_t size,
                const int64_t* __restrict__ data_idx, int B, int history, int n_max, const rb_horizon* __restrict__ hz,
                float* __restrict__ states, float* __restrict__ next_states, int64_t* __restrict__ actions,
                float* __restrict__ returns, float* __restrict__ nonterminals, int split, int pad, float intensity,
                int m_copies, int k_copies, uint64_t seed, const unsigned long long* __restrict__ rng_counter,
                int32_t* __restrict__ shifts, float* __restrict__ scales) {
  gather_aug_body<true, false>(frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max, nullptr,
                               states, next_states, actions, returns, nonterminals, split, pad, intensity, m_copies,
                               k_copies, seed, rng_counter, shifts, scales, hz);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_shift_hz_trunc(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep,
                        const int32_t* __restrict__ action, const float* __restrict__ reward,
                        const uint8_t* __restrict__ nonterminal, int64_t size, const int64_t* __restrict__ data_idx, int B,
                        int history, int n_max, const rb_horizon* __restrict__ hz, float* __restrict__ states,
                        float* __restrict__ next_states, int64_t* __restrict__ actions, float* __restrict__ returns,
                        float* __restrict__ nonterminals, int split, int pad, uint64_t seed,
                        const unsigned long long* __restrict__ rng_counter, int32_t* __restrict__ shifts) {
  gather_aug_body<true, true, true>(frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max,
                                    nullptr, states, next_states, actions, returns, nonterminals, split, pad, 0.0f, 1, 1,
                                    seed, rng_counter, shifts, nullptr, hz);
}

__global__ void __launch_bounds__(GATHER_THREADS)
k_gather_aug_hz_trunc(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep,
                      const int32_t* __restrict__ action, const float* __restrict__ reward,
                      const uint8_t* __restrict__ nonterminal, int64_t size, const int64_t* __restrict__ data_idx, int B,
                      int history, int n_max, const rb_horizon* __restrict__ hz, float* __restrict__ states,
                      float* __restrict__ next_states, int64_t* __restrict__ actions, float* __restrict__ returns,
                      float* __restrict__ nonterminals, int split, int pad, float intensity, int m_copies, int k_copies,
                      uint64_t seed, const unsigned long long* __restrict__ rng_counter, int32_t* __restrict__ shifts,
                      float* __restrict__ scales) {
  gather_aug_body<true, false, true>(frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max,
                                     nullptr, states, next_states, actions, returns, nonterminals, split, pad, intensity,
                                     m_copies, k_copies, seed, rng_counter, shifts, scales, hz);
}

// One thread: current <- table[min(*counter, T)] (a negative counter reads row 0), then ++*counter.  The first node of an
// update that anneals its horizon; it runs beside rb_tree_sample, and the gather waits for it.
__global__ void __launch_bounds__(1)
k_horizon_advance(const rb_horizon* __restrict__ table, int T, long long* __restrict__ counter,
                  rb_horizon* __restrict__ current) {
  const long long u = *counter;
  const int row = u <= 0 ? 0 : (u >= T ? T : (int)u);
  const rb_horizon* __restrict__ src = table + row;
  current->n = src->n;
  current->gamma_n = src->gamma_n;
#pragma unroll
  for (int k = 0; k < RB_MAX_WINDOW; ++k) current->gamma_pow[k] = src->gamma_pow[k];
  *counter = u + 1;
}

// memory.py:166-178 validation iterator, batched: grid = (history, count)
__global__ void __launch_bounds__(GATHER_THREADS)
k_iter_states(const uint8_t* __restrict__ frames, const int32_t* __restrict__ timestep, int64_t size, int64_t first_idx,
              int history, float* __restrict__ out) {
  __shared__ uint64_t s_first;
  const int s = blockIdx.x;
  const int64_t cur = first_idx + blockIdx.y;
  if (threadIdx.x < 32) {
    uint64_t f = window_first_bits(timestep, size, cur, history, history);
    if (threadIdx.x == 0) s_first = f;
  }
  __syncthreads();
  const bool blank = slot_blank(s_first, s, history);
  const int64_t pos = pymod(cur - (history - 1) + s, size);
  const uint4* src = reinterpret_cast<const uint4*>(frames + (size_t)pos * RB_FRAME_BYTES);
  float4* dst = reinterpret_cast<float4*>(out + ((size_t)blockIdx.y * history + s) * RB_FRAME_BYTES);
  for (int v = threadIdx.x; v < FRAME_VEC; v += GATHER_THREADS) {
    uint4 q = blank ? make_uint4(0, 0, 0, 0) : __ldg(src + v);
    dst[4 * v + 0] = u8x4_to_unit(q.x);
    dst[4 * v + 1] = u8x4_to_unit(q.y);
    dst[4 * v + 2] = u8x4_to_unit(q.z);
    dst[4 * v + 3] = u8x4_to_unit(q.w);
  }
}

// ================================================================================================
// K5  append : up to RB_APPEND_BATCH transitions in ONE launch (rb_append: one; rb_append_batch: the actor's queue,
// SURVEY 8(f).2).  Each is quantised and stored, its leaf set to the running max, and the tree walked to the root.
// ================================================================================================
constexpr int APPEND_THREADS = 256;

// Equivalent to k single appends in order: the records go to slots head, head+1, ... (mod size), the
// in-episode counter follows the terminals, every new leaf gets the running max (which appends never change) and,
// because every internal node is recomputed from its children, the tree after k sequential walks equals the tree
// after ONE level-synchronous batched walk over the k leaves (same argument as for rb_tree_update).  The frame
// pointers may be device memory or pinned host memory (read in place over PCIe: no staging copy, no extra launch).
struct AppendBatch {
  const float* frame[RB_APPEND_BATCH];
  int32_t action[RB_APPEND_BATCH];
  float reward[RB_APPEND_BATCH];
  int32_t terminal[RB_APPEND_BATCH];
  int k;
};

// FINAL (rb_append_batch_trunc): terminal[j] == RB_NONTERMINAL_FINAL stores a final-observation record -- nonterminal byte
// RB_NONTERMINAL_FINAL, leaf 0 -- and, like a terminal, makes the next record start an episode.
template <bool FINAL>
__device__ __forceinline__ void
append_batch_body(float* tree, int64_t tree_start, int64_t size, uint8_t* __restrict__ frames, int32_t* timestep,
                  int32_t* action, float* reward, uint8_t* nonterminal, int64_t* ring_state, const float* running_max,
                  const AppendBatch& ab) {
  // grid = k CTAs: CTA j quantises frame j (all of a thread's 16-byte loads in flight at once -- the frames may sit in
  // pinned host memory, where every dependent load is a PCIe round trip); warp 0 of CTA 0 also writes the k records and
  // walks the tree.  ring_state is read by every CTA when it starts and advanced by the LAST CTA to finish (ticket in
  // ring_state[4]), so no CTA can see the new head.
  const int tid = threadIdx.x;
  const int j = blockIdx.x;
  const int64_t head = ring_state[0];
  const int64_t t_ep0 = ring_state[2];
  const int k = ab.k;
  {  // frame j: f32 * 255 then truncating cast (memory.py:106)
    int64_t slot = head + j;
    if (slot >= size) slot -= size;
    uint32_t* dst = reinterpret_cast<uint32_t*>(frames + (size_t)slot * RB_FRAME_BYTES);
    const float4* src = reinterpret_cast<const float4*>(ab.frame[j]);
    constexpr int PER = (RB_FRAME_BYTES / 4 + APPEND_THREADS - 1) / APPEND_THREADS;   // 7
    float4 x[PER];
#pragma unroll
    for (int u = 0; u < PER; ++u) {
      const int v = tid + u * APPEND_THREADS;
      x[u] = (v < RB_FRAME_BYTES / 4) ? src[v] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < PER; ++u) {
      const int v = tid + u * APPEND_THREADS;
      if (v < RB_FRAME_BYTES / 4) {
        const uint32_t a = (uint32_t)(uint8_t)(int)__fmul_rn(x[u].x, 255.0f);
        const uint32_t b = (uint32_t)(uint8_t)(int)__fmul_rn(x[u].y, 255.0f);
        const uint32_t c = (uint32_t)(uint8_t)(int)__fmul_rn(x[u].z, 255.0f);
        const uint32_t d = (uint32_t)(uint8_t)(int)__fmul_rn(x[u].w, 255.0f);
        dst[v] = a | (b << 8) | (c << 16) | (d << 24);
      }
    }
  }
  if (j == 0 && tid < 32) {
    const unsigned full = 0xffffffffu;
    const int lane = tid;
    const int L = tree_depth(tree_start);
    const bool active = lane < k;
    int64_t slot = head + lane;
    if (slot >= size) slot -= size;
    int64_t node = active ? slot + tree_start : -1;
    float val = *running_max;  // memory.py:107
    if (active) {              // record fields; timestep follows the terminals of the earlier queued transitions
      int64_t t = t_ep0;
      for (int i = 0; i < lane; ++i) t = ab.terminal[i] ? 0 : t + 1;
      timestep[slot] = (int32_t)t;
      action[slot] = ab.action[lane];
      reward[slot] = ab.reward[lane];
      if (FINAL && ab.terminal[lane] == RB_NONTERMINAL_FINAL) {
        nonterminal[slot] = RB_NONTERMINAL_FINAL;
        val = 0.0f;
      } else {
        nonterminal[slot] = ab.terminal[lane] ? 0 : 1;
      }
    }
    float sib[32];
#pragma unroll
    for (int l = 0; l < 32; ++l) {
      sib[l] = 0.0f;
      if (l < L && active) {
        const int64_t nl = ((node + 1) >> l) - 1;
        const int64_t sn = (nl & 1) ? nl + 1 : nl - 1;
        sib[l] = __ldcg(tree + sn);
      }
    }
    if (active) __stcg(tree + node, val);  // k distinct leaves (k <= size is checked by the launcher)
#pragma unroll
    for (int l = 0; l < 32; ++l) {
      if (l < L) {
        const int64_t parent = active ? ((node - 1) >> 1) : -(int64_t)(lane + 1);
        const bool is_left = active && (node & 1);
        const unsigned grp = __match_any_sync(full, (int)parent);
        const unsigned lefts = __ballot_sync(full, is_left);
        const unsigned other = grp & (is_left ? ~lefts : lefts);
        const float partner = __shfl_sync(full, val, other ? __ffs(other) - 1 : lane);
        val = __fadd_rn(val, other ? partner : sib[l]);
        node = parent;
        if (active && lane == __ffs(grp) - 1) __stcg(tree + node, val);
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    unsigned long long* ticket = reinterpret_cast<unsigned long long*>(ring_state + 4);
    if (atomicAdd(ticket, 1ull) == (unsigned long long)(k - 1)) {   // last CTA: everybody has read the old head
      *ticket = 0ull;
      int64_t nh = head + k;
      bool wrapped = false;
      if (nh >= size) {
        nh -= size;
        wrapped = true;
      }
      int64_t t = t_ep0;
      for (int i = 0; i < k; ++i) t = ab.terminal[i] ? 0 : t + 1;
      ring_state[0] = nh;
      if (wrapped) ring_state[1] = 1;
      ring_state[2] = t;
      ring_state[3] = ring_state[3] + k;
    }
  }
}

__global__ void __launch_bounds__(APPEND_THREADS)
k_append_batch(float* tree, int64_t tree_start, int64_t size, uint8_t* __restrict__ frames, int32_t* timestep,
               int32_t* action, float* reward, uint8_t* nonterminal, int64_t* ring_state, const float* running_max,
               const __grid_constant__ AppendBatch ab) {
  append_batch_body<false>(tree, tree_start, size, frames, timestep, action, reward, nonterminal, ring_state, running_max,
                           ab);
}

__global__ void __launch_bounds__(APPEND_THREADS)
k_append_batch_final(float* tree, int64_t tree_start, int64_t size, uint8_t* __restrict__ frames, int32_t* timestep,
                     int32_t* action, float* reward, uint8_t* nonterminal, int64_t* ring_state, const float* running_max,
                     const __grid_constant__ AppendBatch ab) {
  append_batch_body<true>(tree, tree_start, size, frames, timestep, action, reward, nonterminal, ring_state, running_max,
                          ab);
}

// ================================================================================================
// Bulk append (rb_append_bulk): k records of a dataset in one call, equal to k appends in order (DESIGN §23).  The frames
// are copies issued by the entry; these kernels write the records, the leaves, the touched ancestors and the ring state.
//   1. k_bulk_block_reset  : per tile of BULK_TILE records, the last index whose flag is nonzero (-1 if none);
//   2. k_bulk_scan_tiles   : one CTA, exclusive max-scan of those over the tiles, in place, and the block's total;
//   3. k_bulk_records      : r_j = the last index < j with a nonzero flag, t_j = r_j < 0 ? t_ep0 + j : j - r_j - 1; the
//                            record at slot (head + j) mod size and its leaf (*running_max, 0 for a FINAL record);
//   4. k_bulk_tree_level   : one grid-wide launch per wide level: each touched ancestor = fl32(left + right);
//   5. k_bulk_tree_top     : one CTA finishes the narrow top levels, then advances the ring state once.
// Every launch reads the head from ring_state[0]; only the last one writes it.  k <= size, so every record survives.
// ================================================================================================
constexpr int BULK_THREADS = 256;
constexpr int BULK_ITEMS = 4;
constexpr int BULK_TILE = BULK_THREADS * BULK_ITEMS;
constexpr int BULK_TOP_THREADS = 1024;

__device__ __forceinline__ int warp_max_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide max of v over BULK_THREADS threads (the result in every thread).
__device__ __forceinline__ int bulk_block_max(int v, int* s_warp) {
  v = warp_max_int(v);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  int m = -1;
#pragma unroll
  for (int w = 0; w < BULK_THREADS / 32; ++w) m = max(m, s_warp[w]);
  return m;
}

__global__ void __launch_bounds__(BULK_THREADS)
k_bulk_block_reset(const uint8_t* __restrict__ flags, int k, int* __restrict__ tile_reset) {
  __shared__ int s_warp[BULK_THREADS / 32];
  const int base = blockIdx.x * BULK_TILE;
  int r = -1;
#pragma unroll
  for (int u = 0; u < BULK_ITEMS; ++u) {
    const int j = base + u * BULK_THREADS + threadIdx.x;
    if (j < k && flags[j]) r = max(r, j);
  }
  r = bulk_block_max(r, s_warp);
  if (threadIdx.x == 0) tile_reset[blockIdx.x] = r;
}

// tile_reset[0 .. tiles) -> the exclusive prefix max (-1 before tile 0); tile_reset[tiles] = the max over all tiles.
__global__ void __launch_bounds__(BULK_TOP_THREADS)
k_bulk_scan_tiles(int* tile_reset, int tiles) {
  __shared__ int s_warp[BULK_TOP_THREADS / 32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = -1;
  __syncthreads();
  for (int base = 0; base < tiles; base += BULK_TOP_THREADS) {
    const int i = base + threadIdx.x;
    const int v = i < tiles ? tile_reset[i] : -1;
    int inc = v;   // inclusive max within the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc = max(inc, y);
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    int before = s_carry, total = s_carry;
    for (int w = 0; w < BULK_TOP_THREADS / 32; ++w) {
      if (w < warp) before = max(before, s_warp[w]);
      total = max(total, s_warp[w]);
    }
    const int prev = __shfl_up_sync(0xffffffffu, inc, 1);
    const int excl = lane > 0 ? max(before, prev) : before;
    __syncthreads();   // s_carry and s_warp read by every thread
    if (i < tiles) tile_reset[i] = excl;
    if (threadIdx.x == 0) s_carry = total;
    __syncthreads();
  }
  if (threadIdx.x == 0) tile_reset[tiles] = s_carry;
}

__global__ void __launch_bounds__(BULK_THREADS)
k_bulk_records(float* tree, int64_t tree_start, int64_t size, int32_t* timestep, int32_t* action, float* reward,
               uint8_t* nonterminal, const int64_t* ring_state, const float* running_max,
               const int32_t* __restrict__ actions, const float* __restrict__ rewards, const uint8_t* __restrict__ flags,
               int k, const int* __restrict__ tile_reset) {
  __shared__ int s_warp[BULK_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t head = ring_state[0];
  const int64_t t_ep0 = ring_state[2];
  const float leaf = *running_max;
  // thread-contiguous items: thread x of tile b holds records base + BULK_ITEMS x + u
  const int base = blockIdx.x * BULK_TILE + BULK_ITEMS * threadIdx.x;
  uint8_t f[BULK_ITEMS];
  int own = -1;
#pragma unroll
  for (int u = 0; u < BULK_ITEMS; ++u) {
    const int j = base + u;
    f[u] = j < k ? flags[j] : (uint8_t)0;
    if (f[u]) own = j;
  }
  int inc = own;   // inclusive max over the threads of the warp, then exclusive over the block
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc = max(inc, y);
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int r = tile_reset[blockIdx.x];   // the last reset before this tile
  for (int w = 0; w < warp; ++w) r = max(r, s_warp[w]);
  const int prev = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane > 0) r = max(r, prev);
#pragma unroll
  for (int u = 0; u < BULK_ITEMS; ++u) {
    const int j = base + u;
    if (j < k) {
      const int64_t t = r < 0 ? t_ep0 + j : (int64_t)(j - r - 1);
      int64_t slot = head + j;
      if (slot >= size) slot -= size;
      const bool fin = f[u] == RB_NONTERMINAL_FINAL;
      timestep[slot] = (int32_t)t;
      action[slot] = fin ? 0 : actions[j];
      reward[slot] = fin ? 0.0f : rewards[j];
      nonterminal[slot] = fin ? (uint8_t)RB_NONTERMINAL_FINAL : f[u] ? (uint8_t)0 : (uint8_t)1;
      __stcg(tree + tree_start + slot, fin ? 0.0f : leaf);
      if (f[u]) r = j;
    }
  }
}

// The touched nodes s levels above the leaves, as two disjoint intervals [a1, b1] and [a2, b2] of heap indices (the second
// may be empty: b2 < a2).  The leaves are slots head .. head + k - 1 (mod size): [head, min(head + k, size)) and, after a
// wrap, [0, head + k - size).  Both children of every such node lie inside the array (size is even).
__device__ __forceinline__ void bulk_level_nodes(int64_t head, int64_t k, int64_t size, int64_t tree_start, int s,
                                                 int64_t& a1, int64_t& b1, int64_t& a2, int64_t& b2) {
  const int64_t end = head + k;
  const int64_t hi1 = (end < size ? end : size) - 1;
  a1 = ((tree_start + head + 1) >> s) - 1;
  b1 = ((tree_start + hi1 + 1) >> s) - 1;
  a2 = 0;
  b2 = -1;
  if (end > size) {
    a2 = ((tree_start + 1) >> s) - 1;
    b2 = ((tree_start + (end - size - 1) + 1) >> s) - 1;
    if (b2 + 1 >= a1) {   // the wrapped range lies left of the first; merge where they meet or overlap
      a1 = a2;
      a2 = 0;
      b2 = -1;
    }
  }
}

__device__ __forceinline__ void bulk_rebuild_node(float* tree, int64_t p) {
  __stcg(tree + p, __fadd_rn(__ldcg(tree + 2 * p + 1), __ldcg(tree + 2 * p + 2)));
}

__global__ void __launch_bounds__(BULK_THREADS)
k_bulk_tree_level(float* tree, int64_t tree_start, int64_t size, const int64_t* ring_state, int k, int s) {
  int64_t a1, b1, a2, b2;
  bulk_level_nodes(ring_state[0], k, size, tree_start, s, a1, b1, a2, b2);
  const int64_t n2 = b2 - a2 + 1, n = n2 + (b1 - a1 + 1);
  const int64_t i = (int64_t)blockIdx.x * BULK_THREADS + threadIdx.x;
  if (i < n) bulk_rebuild_node(tree, i < n2 ? a2 + i : a1 + (i - n2));
}

__global__ void __launch_bounds__(BULK_TOP_THREADS)
k_bulk_tree_top(float* tree, int64_t tree_start, int64_t size, int64_t* ring_state, int k, int s_first,
                const int* tile_reset, int tiles) {
  const int64_t head = ring_state[0];
  const int L = tree_depth(tree_start);
  for (int s = s_first; s <= L; ++s) {
    int64_t a1, b1, a2, b2;
    bulk_level_nodes(head, k, size, tree_start, s, a1, b1, a2, b2);
    const int64_t n2 = b2 - a2 + 1, n = n2 + (b1 - a1 + 1);
    for (int64_t i = threadIdx.x; i < n; i += BULK_TOP_THREADS) bulk_rebuild_node(tree, i < n2 ? a2 + i : a1 + (i - n2));
    __syncthreads();
  }
  if (threadIdx.x == 0) {   // every earlier launch has read the old head
    const int r_last = tile_reset[tiles];
    int64_t nh = head + k;
    if (nh >= size) {
      nh -= size;
      ring_state[1] = 1;
    }
    ring_state[2] = r_last < 0 ? ring_state[2] + k : (int64_t)(k - 1 - r_last);
    ring_state[0] = nh;
    ring_state[3] = ring_state[3] + k;
  }
}

// ================================================================================================
// Value rescaling (Pohlen et al. 2018): h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x and its inverse, in cancellation-free
// forms (DESIGN.md §16): every step adds or multiplies nonnegative terms, each rounded explicitly (no contraction), with
// IEEE sqrtf and __fdiv_rn.  0 <= eps <= 1 (the host entries refuse anything else).
//   h(x)      = sign(x) |x| / (sqrt(|x| + 1) + 1) + eps x
//   h^-1(y)   = sign(y) d (d + 2),  d = 2|y| / ((1 + 2 eps) + sqrt((1 + 2 eps)^2 + 4 eps |y|))
// ================================================================================================
__device__ __forceinline__ float vt_h(float x, float eps) {
  const float ax = fabsf(x);
  const float r = __fdiv_rn(ax, __fadd_rn(sqrtf(__fadd_rn(ax, 1.0f)), 1.0f));
  return __fadd_rn(copysignf(r, x), __fmul_rn(eps, x));
}

__device__ __forceinline__ float vt_hinv(float y, float eps) {
  const float ay = fabsf(y);
  const float c = __fadd_rn(1.0f, __fmul_rn(2.0f, eps));
  const float disc = __fadd_rn(__fmul_rn(c, c), __fmul_rn(__fmul_rn(4.0f, eps), ay));
  const float d = __fdiv_rn(__fmul_rn(2.0f, ay), __fadd_rn(c, sqrtf(disc)));
  return copysignf(__fmul_rn(d, __fadd_rn(d, 2.0f)), y);
}

// ================================================================================================
// K3  c51_loss_grad : double-DQN argmax + categorical projection + IS-weighted CE loss + gradient.
// ================================================================================================
// One warp per sample; lane owns atoms z = lane + 32*r.  The projected distribution is built as a
// GATHER (thread per target atom scans the source atoms in order, l-side terms first, then u-side
// terms): deterministic and in the reference CPU index_add_ order (agent.py:91-92), no atomics.
// c51_core works on logit ROWS given by generic pointers (global memory for the plain entry point,
// warp-private shared memory for the dueling entry point) and returns, per lane, the gradient row
// g[z] = (w/B)(p*sum(m) - m) of the taken action.
constexpr int C51_WARPS = 4;
// atoms per lane: templates are instantiated for R = 2 (Z <= 64, the usual 51 atoms) and R = 4 (Z <= 128)

struct C51Scratch {  // per warp
  float pt[RB_MAX_ATOMS];  // target probabilities p(s', a*)
  float b[RB_MAX_ATOMS];
  int l[RB_MAX_ATOMS];
  int u[RB_MAX_ATOMS];
};

template <int C51_R>
__device__ __forceinline__ void softmax_row(const float* row, int Z, int lane, float (&e)[C51_R], float (&x)[C51_R],
                                            float& mx, float& sum) {
  mx = -CUDART_INF_F;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    int z = lane + 32 * r;
    x[r] = (z < Z) ? row[z] : -CUDART_INF_F;
    mx = fmaxf(mx, x[r]);
  }
  mx = warp_max(mx);
  sum = 0.0f;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    e[r] = (lane + 32 * r < Z) ? expf(x[r] - mx) : 0.0f;
    sum = __fadd_rn(sum, e[r]);
  }
  sum = warp_sum(sum);
}

// Expected value sum_z support_z * p_z of one logit row held in registers (x[r] = logit of atom lane + 32 r, -inf past Z),
// p = e / sum(e): the numerator and sum(e) ride the same shuffle butterfly (two independent shuffles per step) and one
// division finishes the row (agent.py:71-72).  All lanes return the value.
template <int C51_R>
__device__ __forceinline__ float c51_expected_value(const float (&x)[C51_R], const float (&sup)[C51_R], int Z, int lane) {
  float mx = -CUDART_INF_F;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) mx = fmaxf(mx, x[r]);
  mx = warp_max(mx);
  float se = 0.0f, sn = 0.0f;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    const float ee = (lane + 32 * r < Z) ? expf(x[r] - mx) : 0.0f;
    se = __fadd_rn(se, ee);
    sn = __fadd_rn(sn, __fmul_rn(sup[r], ee));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se = __fadd_rn(se, __shfl_xor_sync(0xffffffffu, se, o));
    sn = __fadd_rn(sn, __shfl_xor_sync(0xffffffffu, sn, o));
  }
  return __fdiv_rn(sn, se);
}

// ---- Risk-sensitive values: distortion risk measures of the return distribution (DESIGN.md §18) ----
// The loss kernels' risk instantiations carry this bit in their atoms-per-lane parameter R (k_qr_dueling<2 | RISK_INST,
// false> is k_qr_dueling<2, false> with the distorted arg-max): their template argument lists, and so the names graph
// dumps and profiles show for the parent instantiations, stay as they were.
constexpr int RISK_INST = 16;
// beta(t) of the distortion `kind`, the weight of the levels [0, t]: RB_RISK_CVAR min(t / eta, 1), RB_RISK_WANG
// Phi(Phi^-1(t) - eta) -- the inverses of IQN's level maps eta tau and Phi(Phi^-1(tau) + eta), so eta keeps IQN's sign
// (normcdfinvf gives -inf / +inf at t = 0 / 1, so beta(0) = 0 and beta(1) = 1 exactly for both).
__device__ __forceinline__ float risk_beta(float t, int kind, float eta) {
  if (kind == RB_RISK_CVAR) return fminf(__fdiv_rn(t, eta), 1.0f);
  return normcdff(__fsub_rn(normcdfinvf(t), eta));
}

// Distorted value Q_beta = sum_k w_k support_k of one logit row held as c51_expected_value takes it (support
// non-decreasing), w_k = beta(F_k) - beta(F_{k-1}).  With e = expf(x - max x) and se = sum e (c51_expected_value's lane
// sums and butterfly): S_k is the inclusive scan of e in atom order (per 32-atom segment a Hillis-Steele scan over the
// lanes, offsets 1, 2, 4, 8, 16, then the previous segment's total added in front), F_k = min(S_k / se, 1) and
// F_{Z-1} = 1.  Each lane sums w_k support_k over its atoms in r order, then the butterfly.  All lanes return the value.
template <int C51_R>
__device__ __forceinline__ float c51_risk_value(const float (&x)[C51_R], const float (&sup)[C51_R], int Z, int lane,
                                                int kind, float eta) {
  float mx = -CUDART_INF_F;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) mx = fmaxf(mx, x[r]);
  mx = warp_max(mx);
  float e[C51_R], se = 0.0f;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    e[r] = (lane + 32 * r < Z) ? expf(x[r] - mx) : 0.0f;
    se = __fadd_rn(se, e[r]);
  }
  se = warp_sum(se);
  float carry = 0.0f, b_carry = 0.0f, s = 0.0f;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    const int k = lane + 32 * r;
    float v = e[r];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float y = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v = __fadd_rn(v, y);
    }
    v = __fadd_rn(carry, v);
    carry = __shfl_sync(0xffffffffu, v, 31);
    const float F = k >= Z - 1 ? 1.0f : fminf(__fdiv_rn(v, se), 1.0f);
    const float b = risk_beta(F, kind, eta);
    float bp = __shfl_up_sync(0xffffffffu, b, 1);
    if (lane == 0) bp = b_carry;
    b_carry = __shfl_sync(0xffffffffu, b, 31);
    if (k < Z) s = __fadd_rn(s, __fmul_rn(__fsub_rn(b, bp), sup[r]));
  }
  return warp_sum(s);
}

// Level weights of the quantiles a lane owns (j = lane + 32 r): quantile j stands for the levels [j/N, (j+1)/N] in index
// order (not value order: quantiles can cross), w_j = beta(fl32((j+1)/N)) - beta(fl32(j/N)), 0 past N.  They depend on
// no row, so a warp forms them once for all the actions it takes.
template <int R>
__device__ __forceinline__ void qr_risk_weights(int N, int lane, int kind, float eta, float (&w)[R]) {
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int j = lane + 32 * r;
    w[r] = 0.0f;
    if (j < N) {
      const float lo = risk_beta(__fdiv_rn((float)j, (float)N), kind, eta);
      const float hi = risk_beta(__fdiv_rn((float)(j + 1), (float)N), kind, eta);
      w[r] = __fsub_rn(hi, lo);
    }
  }
}

// Distorted value of one quantile row held as qr_row_mean takes it, with qr_risk_weights' w: each lane sums w_j theta_j
// over its quantiles in r order, then the butterfly.  All lanes return the value.
template <int R>
__device__ __forceinline__ float qr_risk_value(const float (&x)[R], const float (&w)[R], int N, int lane) {
  float s = 0.0f;
#pragma unroll
  for (int r = 0; r < R; ++r)
    if (lane + 32 * r < N) s = __fadd_rn(s, __fmul_rn(w[r], x[r]));
  return warp_sum(s);
}

// q_on_ns / q_tg_ns: A rows of Z (row stride Z); q_on_s_act: the row of the taken action.
// best_known >= 0: a* was already determined by the caller (q_on_ns is then not read, q_tg_ns points at the row of a*).
// VT (value rescaling): support_q = fl32(h^-1(support)) replaces the support in the arg-max and in Tz, and the target atoms
// are h(r + fl32(scale * support_q)) (support itself is then not read); the projection onto the h-space grid is unchanged.
template <int C51_R, bool VT = false>
__device__ __forceinline__ void c51_core(C51Scratch& sc, int lane, int i, int B, int A, int Z, const float* q_on_ns,
                                         const float* q_tg_ns, const float* q_on_s_act, float ret, float nonterminal,
                                         float weight, const float* __restrict__ support, float vmin, float vmax,
                                         float delta_z, float gamma_n, float* __restrict__ loss, float* __restrict__ m_out,
                                         int64_t* __restrict__ astar_out, float (&g)[C51_R], int best_known = -1,
                                         const float* __restrict__ support_q = nullptr, float eps = 0.0f) {
  float sup[C51_R];
  if constexpr (VT) support = support_q;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    int z = lane + 32 * r;
    sup[r] = (z < Z) ? __ldg(support + z) : 0.0f;
  }
  float e[C51_R], x[C51_R], mx, sum;

  // ---- agent.py:71-73: a* = argmax_a sum_z support_z * softmax(q_online(s'))[a,z] ----
  int best = 0;
  if (best_known >= 0) {
    best = best_known;
  } else {
    float best_ev = -CUDART_INF_F;
    for (int a = 0; a < A; ++a) {
      const float* row = q_on_ns + (size_t)a * Z;
#pragma unroll
      for (int r = 0; r < C51_R; ++r) {
        int z = lane + 32 * r;
        x[r] = (z < Z) ? row[z] : -CUDART_INF_F;
      }
      const float ev = c51_expected_value<C51_R>(x, sup, Z, lane);
      if (ev > best_ev) {  // first maximum wins, like torch.argmax
        best_ev = ev;
        best = a;
      }
    }
  }
  if (astar_out && lane == 0) astar_out[i] = best;

  // ---- agent.py:75-76: target distribution of the selected action ----
  softmax_row(q_tg_ns + (best_known >= 0 ? (size_t)0 : (size_t)best * Z), Z, lane, e, x, mx, sum);
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    int z = lane + 32 * r;
    if (z < Z) sc.pt[z] = __fdiv_rn(e[r], sum);
  }

  // ---- agent.py:66-67: log p(s, a) and p(s, a) of the online net ----
  float p_on[C51_R], logp[C51_R];
  softmax_row(q_on_s_act, Z, lane, e, x, mx, sum);
  {
    const float lsum = logf(sum);
#pragma unroll
    for (int r = 0; r < C51_R; ++r) {
      p_on[r] = __fdiv_rn(e[r], sum);
      logp[r] = (lane + 32 * r < Z) ? __fsub_rn(__fsub_rn(x[r], mx), lsum) : 0.0f;
    }
  }

  // ---- agent.py:79-86: Tz, b, l, u ----
  const float scale = __fmul_rn(nonterminal, gamma_n);
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    int z = lane + 32 * r;
    if (z < Z) {
      float tz = __fadd_rn(ret, __fmul_rn(scale, sup[r]));
      if constexpr (VT) tz = vt_h(tz, eps);
      tz = fminf(fmaxf(tz, vmin), vmax);
      float bb = __fdiv_rn(__fsub_rn(tz, vmin), delta_z);
      int lo = (int)floorf(bb), up = (int)ceilf(bb);
      if (up > 0 && lo == up) lo -= 1;
      if (lo < Z - 1 && lo == up) up += 1;
      sc.b[z] = bb;
      sc.l[z] = lo;
      sc.u[z] = up;
    }
  }
  __syncwarp();

  // ---- agent.py:89-92: m, deterministic gather in index_add_ order ----
  // Tz is non-decreasing in the atom index (support increasing, scale >= 0, h monotone) and u == l + 1 after the fix-ups, so
  // the source atoms feeding target k on the l side form the contiguous run {j : l[j] == k} and on the u side the
  // run {j : l[j] == k - 1}: two binary searches replace the 2*Z-long scans.  The additions still happen in atom
  // order, l side first (bit-identical to the scan).  Odd inputs (NaN, decreasing support) take the full scan.
  bool mono = true;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    const int z = lane + 32 * r;
    if (z < Z) mono = mono && (sc.u[z] == sc.l[z] + 1) && (z + 1 >= Z || sc.l[z] <= sc.l[z + 1]);
  }
  mono = __all_sync(0xffffffffu, mono);
  float m[C51_R];
  float ce = 0.0f, msum = 0.0f;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    const int k = lane + 32 * r;
    float acc = 0.0f;
    if (k < Z) {
      if (mono) {
        int lo = 0, hi = Z;              // first j with l[j] >= k - 1
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (sc.l[mid] < k - 1) lo = mid + 1; else hi = mid;
        }
        int j = lo;
        const int ju = j;                // start of the u-side run (l == k - 1)
        while (j < Z && sc.l[j] == k - 1) ++j;
        for (int jj = j; jj < Z && sc.l[jj] == k; ++jj)
          acc = __fadd_rn(acc, __fmul_rn(sc.pt[jj], __fsub_rn((float)sc.u[jj], sc.b[jj])));
        for (int jj = ju; jj < j; ++jj)
          acc = __fadd_rn(acc, __fmul_rn(sc.pt[jj], __fsub_rn(sc.b[jj], (float)sc.l[jj])));
      } else {
        for (int j = 0; j < Z; ++j)
          if (sc.l[j] == k) acc = __fadd_rn(acc, __fmul_rn(sc.pt[j], __fsub_rn((float)sc.u[j], sc.b[j])));
        for (int j = 0; j < Z; ++j)
          if (sc.u[j] == k) acc = __fadd_rn(acc, __fmul_rn(sc.pt[j], __fsub_rn(sc.b[j], (float)sc.l[j])));
      }
      if (m_out) m_out[(size_t)i * Z + k] = acc;
    }
    m[r] = acc;
    ce = __fadd_rn(ce, __fmul_rn(acc, logp[r]));
    msum = __fadd_rn(msum, acc);
  }
  ce = warp_sum(ce);
  msum = warp_sum(msum);
  if (lane == 0) loss[i] = -ce;  // agent.py:94

  // ---- agent.py:96: d mean(w*loss) / d q_online(s)[i, act, :] ----
  const float wi = __fdiv_rn(weight, (float)B);
#pragma unroll
  for (int r = 0; r < C51_R; ++r) g[r] = __fmul_rn(wi, __fsub_rn(__fmul_rn(p_on[r], msum), m[r]));
  __syncwarp();
}

// VT: the value-rescaled instantiation (c51_core's VT); support_q / eps are read only there.
// RISK (R with RISK_INST set): a* = argmax_a c51_risk_value of online(s') (first maximum wins), found here and handed to
// c51_core as best_known; risk_kind / risk_eta are read only there.
template <int C51_R_RISK, bool VT>
__global__ void __launch_bounds__(C51_WARPS * 32)
k_c51(const float* __restrict__ q_on_s, const float* __restrict__ q_on_ns, const float* __restrict__ q_tg_ns,
      const int64_t* __restrict__ actions, const float* __restrict__ returns, const float* __restrict__ nonterminals,
      const float* __restrict__ weights, const float* __restrict__ support, float vmin, float vmax, float delta_z,
      float gamma_n, int B, int A, int Z, float* __restrict__ loss, float* __restrict__ grad,
      float* __restrict__ m_out, int64_t* __restrict__ astar_out, const float* __restrict__ support_q, float eps,
      int risk_kind, float risk_eta) {
  constexpr int C51_R = C51_R_RISK & ~RISK_INST;
  constexpr bool RISK = (C51_R_RISK & RISK_INST) != 0;
  __shared__ C51Scratch s_sc[C51_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * C51_WARPS + warp;
  if (i >= B) return;
  const int act = (int)actions[i];
  float g[C51_R];
  const float* q_tg = q_tg_ns + (size_t)i * A * Z;
  int best_known = -1;
  if constexpr (RISK) {
    float best_v = -CUDART_INF_F;
    best_known = 0;
    for (int a = 0; a < A; ++a) {
      const float* row = q_on_ns + ((size_t)i * A + a) * Z;
      float sup[C51_R], x[C51_R];
#pragma unroll
      for (int r = 0; r < C51_R; ++r) {
        const int z = lane + 32 * r;
        sup[r] = (z < Z) ? __ldg(support + z) : 0.0f;
        x[r] = (z < Z) ? row[z] : -CUDART_INF_F;
      }
      const float v = c51_risk_value<C51_R>(x, sup, Z, lane, risk_kind, risk_eta);
      if (v > best_v) {  // first maximum wins, like torch.argmax
        best_v = v;
        best_known = a;
      }
    }
    q_tg += (size_t)best_known * Z;
  }
  c51_core<C51_R, VT>(s_sc[warp], lane, i, B, A, Z, q_on_ns + (size_t)i * A * Z, q_tg,
           q_on_s + ((size_t)i * A + act) * Z, __ldg(returns + i), __ldg(nonterminals + i), __ldg(weights + i), support, vmin,
           vmax, delta_z, gamma_n, loss, m_out, astar_out, g, best_known, support_q, eps);
  float* gq = grad + (size_t)i * A * Z;
  for (int j = lane; j < A * Z; j += 32) gq[j] = 0.0f;
  __syncwarp();
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    int z = lane + 32 * r;
    if (z < Z) gq[(size_t)act * Z + z] = g[r];
  }
}

// ---- stages the dueling kernels share: a z row is (z_value [Z] | z_advantage [A][Z]), N2 = Z + A Z floats ----

// Mean advantage at atom c of z row zr (model.py:75): summed over the actions in order from 0, divided once by A.  This
// and dueling_q define the dueling combination for the quantile, select and statistics kernels, which agree bitwise with
// the loss kernels because of it.  k_c51_dueling and k_c51_dueling_avg spell the same arithmetic out inline: through these
// helpers ptxas gives them more registers, and a spill at R = 4.  LDG: the row is in global memory, read through the
// read-only cache (else shared).
template <bool LDG = false>
__device__ __forceinline__ float dueling_mean(const float* zr, int A, int Z, int c) {
  float acc = 0.0f;
  for (int a = 0; a < A; ++a) acc += LDG ? __ldg(zr + Z + a * Z + c) : zr[Z + a * Z + c];
  return acc / (float)A;
}

// q_a[c] = v[c] + adv_a[c] - mean[c], from values the caller loaded (sites that reuse v and the mean across actions)
__device__ __forceinline__ float dueling_q(float v, float adv, float mean) { return v + adv - mean; }

// q_a[c] of z row zr, the mean formed for this one atom and action
template <bool LDG = false>
__device__ __forceinline__ float dueling_q(const float* zr, int A, int Z, int c, int a) {
  const float mean = dueling_mean<LDG>(zr, A, Z, c);
  return dueling_q(LDG ? __ldg(zr + c) : zr[c], LDG ? __ldg(zr + Z + a * Z + c) : zr[Z + a * Z + c], mean);
}

// Stage sample i's M + 2K z rows into zs [M + 2K][N2] with all T threads: online(s_j) from z_on row jB + i, online(s'_k)
// from z_on row (M + k)B + i, target(s'_k) from z_tg row kB + i.  Eight independent loads in flight per thread, then the
// stores: the fused loss kernels are pure dependent latency, so every load is issued before any is waited on.
template <int T>
__device__ __forceinline__ void stage_z_rows(float* zs, const float* __restrict__ z_on, const float* __restrict__ z_tg,
                                             int i, int B, int N2, int M, int K) {
  const int total = (M + 2 * K) * N2;
  const size_t BN2 = (size_t)B * N2;
  z_on += (size_t)i * N2;
  z_tg += (size_t)i * N2;
  for (int base = threadIdx.x; base < total; base += T * 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int idx = base + u * T;
      v[u] = 0.0f;
      if (idx < total) {
        const int t = idx / N2;
        const float* src = t < M + K ? z_on + (size_t)t * BN2 : z_tg + (size_t)(t - M - K) * BN2;
        v[u] = __ldg(src + (idx - t * N2));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int idx = base + u * T;
      if (idx < total) zs[idx] = v[u];
    }
  }
}

// dz row of one sample from the gradient row g [Z] of its taken action, with all T threads: the dueling combination's
// backward, dzv[c] = g[c] and dza[a][c] = g[c] ([a == act] - 1/A).
template <int T>
__device__ __forceinline__ void dueling_dz(float* __restrict__ dzi, const float* g, int A, int Z, int act) {
  const float inv_a = 1.0f / (float)A;
  for (int idx = threadIdx.x; idx < Z + A * Z; idx += T) {
    if (idx < Z) {
      dzi[idx] = g[idx];
    } else {
      const int a = (idx - Z) / Z, c = (idx - Z) - a * Z;
      dzi[idx] = g[c] * ((a == act ? 1.0f : 0.0f) - inv_a);
    }
  }
}

// dueling_dz for a gradient row on every action, g [A][Z], ADDED onto the dz row with all T threads:
// dzv[c] += gv[c] = sum_a g[a][c] (action order from 0), dza[a][c] += g[a][c] - gv[c] / A.  gv is [Z] of shared scratch.
// The caller synchronises before the call (g complete) and after it (before g or gv are written again).
template <int T>
__device__ __forceinline__ void dueling_dz_rows_add(float* __restrict__ dzi, const float* g, float* gv, int A, int Z) {
  for (int c = threadIdx.x; c < Z; c += T) {
    float acc = 0.0f;
    for (int a = 0; a < A; ++a) acc = __fadd_rn(acc, g[a * Z + c]);
    gv[c] = acc;
  }
  __syncthreads();
  const float inv_a = 1.0f / (float)A;
  for (int idx = threadIdx.x; idx < Z + A * Z; idx += T) {
    if (idx < Z) {
      dzi[idx] = __fadd_rn(dzi[idx], gv[idx]);
    } else {
      const int c = (idx - Z) % Z;
      dzi[idx] = __fadd_rn(dzi[idx], __fsub_rn(g[idx - Z], __fmul_rn(gv[c], inv_a)));
    }
  }
}

// arg-max of s[0, n): the first maximum wins, like torch.argmax
__device__ __forceinline__ int first_argmax(const float* s, int n) {
  int best = 0;
  float best_v = -CUDART_INF_F;
  for (int a = 0; a < n; ++a) {
    const float v = s[a];
    if (v > best_v) {
      best_v = v;
      best = a;
    }
  }
  return best;
}

// Dueling entry point: fed by the fused heads' outputs z = (z_value | z_advantage) [rows][Z + A*Z]
// (online net: 2B rows, s then s'; target net: B rows).  ONE CTA PER SAMPLE, 8 warps: the kernel is pure dependent latency
// (184 KB in, 46 KB out), so the serial chain per sample is cut instead of packing samples into few CTAs:
//   phase 0  all threads stage the sample's three z rows in shared memory (every load in flight at once);
//   phase 1  warp a computes the expected value of action a of the online net on s' (model.py:75 dueling combination on the
//            fly, softmax, expectation) -- the A softmax rows of the double-DQN arg-max run side by side, not in sequence;
//   phase 2  warp 0 takes the arg-max (first maximum wins), assembles the two logit rows still needed (target net at a*,
//            online net at the taken action) and runs the projection / loss / gradient (c51_core, same arithmetic as the
//            plain entry point);
//   phase 3  all threads write dz:  dzv[z] = g[z],  dza[a][z] = g[z] * ([a == act] - 1/A).
constexpr int C51D_T = 256;

// RISK (R with RISK_INST set): phase 1 computes c51_risk_value in place of the expected value; risk_kind / risk_eta
// are read only there.
template <int C51_R_RISK, bool VT>
__global__ void __launch_bounds__(C51D_T)
k_c51_dueling(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
              const float* __restrict__ returns, const float* __restrict__ nonterminals,
              const float* __restrict__ weights, const float* __restrict__ support, float vmin, float vmax,
              float delta_z, float gamma_n, int B, int A, int Z, float* __restrict__ loss, float* __restrict__ dz,
              float* __restrict__ m_out, int64_t* __restrict__ astar_out, const float* __restrict__ support_q,
              float eps, int risk_kind, float risk_eta) {
  constexpr int C51_R = C51_R_RISK & ~RISK_INST;
  constexpr bool RISK = (C51_R_RISK & RISK_INST) != 0;
  extern __shared__ __align__(16) float s_dyn[];
  __shared__ C51Scratch s_sc;
  const int N2 = Z + A * Z;
  float* zs = s_dyn;              // [3][N2]: online(s), online(s'), target(s')
  float* q_t = zs + 3 * N2;       // [Z] target logits of a*
  float* q_s = q_t + Z;           // [Z] online logits of the taken action
  float* s_g = q_s + Z;           // [Z] gradient row
  float* s_ev = s_g + Z;          // [A] expected values
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if constexpr (RISK) {
    // the same three rows in the same order through the shared stager, which keeps no stack array of row pointers
    stage_z_rows<C51D_T>(zs, z_on, z_tg, i, B, N2, 1, 1);
  } else {
    const int total = 3 * N2;
    const float* src[3] = {z_on + (size_t)i * N2, z_on + (size_t)(B + i) * N2, z_tg + (size_t)i * N2};
    for (int base = tid; base < total; base += C51D_T * 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {  // eight independent loads in flight per thread, then the stores
        const int idx = base + u * C51D_T;
        v[u] = 0.0f;
        if (idx < total) {
          const int t = idx / N2;
          v[u] = __ldg(src[t] + (idx - t * N2));
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int idx = base + u * C51D_T;
        if (idx < total) zs[idx] = v[u];
      }
    }
  }
  __syncthreads();
  const int act = (int)actions[i];
  float sup[C51_R];
  const float* sup_ev = support;   // the arg-max's support: support_q under VT (return units)
  if constexpr (VT) sup_ev = support_q;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) sup[r] = (lane + 32 * r < Z) ? __ldg(sup_ev + lane + 32 * r) : 0.0f;
  {  // phase 1: expected value of every action of online(s'), one warp per action
    const float* r1 = zs + N2;
    float mean[C51_R];
#pragma unroll
    for (int r = 0; r < C51_R; ++r) {
      const int c = lane + 32 * r;
      float acc = 0.0f;
      if (c < Z)
        for (int a = 0; a < A; ++a) acc += r1[Z + a * Z + c];
      mean[r] = acc / (float)A;
    }
    for (int a = warp; a < A; a += C51D_T / 32) {
      float x[C51_R];
#pragma unroll
      for (int r = 0; r < C51_R; ++r) {
        const int c = lane + 32 * r;
        x[r] = (c < Z) ? r1[c] + r1[Z + a * Z + c] - mean[r] : -CUDART_INF_F;
      }
      float ev;
      if constexpr (RISK) ev = c51_risk_value<C51_R>(x, sup, Z, lane, risk_kind, risk_eta);
      else ev = c51_expected_value<C51_R>(x, sup, Z, lane);
      if (lane == 0) s_ev[a] = ev;
    }
  }
  __syncthreads();
  if (warp == 0) {  // phase 2
    int best = 0;
    float best_ev = -CUDART_INF_F;
    for (int a = 0; a < A; ++a) {
      const float ev = s_ev[a];
      if (ev > best_ev) {  // first maximum wins, like torch.argmax
        best_ev = ev;
        best = a;
      }
    }
    for (int c = lane; c < Z; c += 32) {
      {  // online(s): the taken action only
        const float* r = zs;
        float mean = 0.0f;
        for (int a = 0; a < A; ++a) mean += r[Z + a * Z + c];
        q_s[c] = r[c] + r[Z + act * Z + c] - mean / (float)A;
      }
      {  // target(s') at a*
        const float* r = zs + 2 * N2;
        float mean = 0.0f;
        for (int a = 0; a < A; ++a) mean += r[Z + a * Z + c];
        mean = mean / (float)A;
        q_t[c] = r[c] + r[Z + best * Z + c] - mean;
      }
    }
    __syncwarp();
    float g[C51_R];
    c51_core<C51_R, VT>(s_sc, lane, i, B, A, Z, nullptr, q_t, q_s, __ldg(returns + i), __ldg(nonterminals + i),
                        __ldg(weights + i), support, vmin, vmax, delta_z, gamma_n, loss, m_out, astar_out, g, best, support_q,
                        eps);
#pragma unroll
    for (int r = 0; r < C51_R; ++r)
      if (lane + 32 * r < Z) s_g[lane + 32 * r] = g[r];
  }
  __syncthreads();
  {  // phase 3
    float* dzi = dz + (size_t)i * N2;
    const float inv_a = 1.0f / (float)A;
    for (int idx = tid; idx < N2; idx += C51D_T) {
      if (idx < Z) {
        dzi[idx] = s_g[idx];
      } else {
        const int a = (idx - Z) / Z, c = (idx - Z) - a * Z;
        dzi[idx] = s_g[c] * ((a == act ? 1.0f : 0.0f) - inv_a);
      }
    }
  }
}

// The loss half of c51_core against a given target distribution m (m[r] = atom lane + 32 r, 0 past Z): log p and p of the
// online logit row q_on_s_act, loss = -sum m log p and the gradient row g = wi (p sum(m) - m), with c51_core's arithmetic.
template <int C51_R>
__device__ __forceinline__ float c51_loss_row(int lane, int Z, const float* q_on_s_act, const float (&m)[C51_R], float wi,
                                              float (&g)[C51_R]) {
  float e[C51_R], x[C51_R], mx, sum, p_on[C51_R], logp[C51_R];
  softmax_row(q_on_s_act, Z, lane, e, x, mx, sum);
  {
    const float lsum = logf(sum);
#pragma unroll
    for (int r = 0; r < C51_R; ++r) {
      p_on[r] = __fdiv_rn(e[r], sum);
      logp[r] = (lane + 32 * r < Z) ? __fsub_rn(__fsub_rn(x[r], mx), lsum) : 0.0f;
    }
  }
  float ce = 0.0f, msum = 0.0f;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    ce = __fadd_rn(ce, __fmul_rn(m[r], logp[r]));
    msum = __fadd_rn(msum, m[r]);
  }
  ce = warp_sum(ce);
  msum = warp_sum(msum);
#pragma unroll
  for (int r = 0; r < C51_R; ++r) g[r] = __fmul_rn(wi, __fsub_rn(__fmul_rn(p_on[r], msum), m[r]));
  return -ce;
}

// DrQ's K / M averaging (Kostrikov et al. 2020, Algorithm 1) on the fused heads' outputs: z_on has (M + K) B rows (copy j of
// s at row jB + i, copy k of s' at row (M + k) B + i), z_tg K B rows (copy k of s' at row kB + i).  ONE CTA PER SAMPLE, as
// k_c51_dueling, with the sample's M + 2K z rows staged in shared memory:
//   phase 1  the expected value of every (target copy k, action a) of online(s'_k), one warp per pair;
//   phase 2  warp k: a*_k (first maximum wins) and the projection m_k of target(s'_k) at a*_k -- c51_core itself, its
//            loss and gradient unused;
//   phase 3  m = (sum_k m_k in k order) / K, rounded once (m_0 exactly at K = 1);
//   phase 4  warp j: loss_j and the gradient row of online(s_j) at the taken action against m (c51_loss_row), with
//            wi = w / (M B);
//   phase 5  loss = (sum_j loss_j in j order) / M; dz rows jB + i get phase 3 of k_c51_dueling.
// At M = K = 1 every output is k_c51_dueling's, bitwise.
template <int C51_R, bool VT>
__global__ void __launch_bounds__(C51D_T)
k_c51_dueling_avg(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
                  const float* __restrict__ returns, const float* __restrict__ nonterminals,
                  const float* __restrict__ weights, const float* __restrict__ support, float vmin, float vmax, float delta_z,
                  float gamma_n, int B, int A, int Z, int M, int K, float* __restrict__ loss, float* __restrict__ dz,
                  float* __restrict__ m_out, int64_t* __restrict__ astar_out, const float* __restrict__ support_q,
                  float eps) {
  extern __shared__ __align__(16) float s_dyn[];
  __shared__ C51Scratch s_sc[C51D_T / 32];
  __shared__ float s_junk[C51D_T / 32];
  constexpr int WARPS = C51D_T / 32;
  const int N2 = Z + A * Z;
  const int rows = M + 2 * K;
  float* zs = s_dyn;               // [M + 2K][N2]: online(s_j), online(s'_k), target(s'_k)
  float* q_t = zs + rows * N2;     // [K][Z] target logits of a*_k
  float* q_s = q_t + K * Z;        // [M][Z] online logits of the taken action
  float* s_g = q_s + M * Z;        // [M][Z] gradient rows
  float* s_m = s_g + M * Z;        // [K][Z] projections m_k
  float* s_mavg = s_m + K * Z;     // [Z] averaged target
  float* s_ev = s_mavg + Z;        // [K][A] expected values
  float* s_loss = s_ev + K * A;    // [M] loss_j
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* on_s = zs;
  const float* on_ns = zs + (size_t)M * N2;
  const float* tg_ns = zs + (size_t)(M + K) * N2;
  {
    const int total = rows * N2;
    for (int base = tid; base < total; base += C51D_T * 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {  // eight independent loads in flight per thread, then the stores
        const int idx = base + u * C51D_T;
        v[u] = 0.0f;
        if (idx < total) {
          const int t = idx / N2;    // staged row t: online rows 0 .. M + K - 1, then the target rows
          const float* src = (t < M + K) ? z_on + ((size_t)t * B + i) * N2 : z_tg + ((size_t)(t - M - K) * B + i) * N2;
          v[u] = __ldg(src + (idx - t * N2));
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int idx = base + u * C51D_T;
        if (idx < total) zs[idx] = v[u];
      }
    }
  }
  __syncthreads();
  const int act = (int)actions[i];
  float sup[C51_R];
  const float* sup_ev = support;   // the arg-max's support: support_q under VT (return units)
  if constexpr (VT) sup_ev = support_q;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) sup[r] = (lane + 32 * r < Z) ? __ldg(sup_ev + lane + 32 * r) : 0.0f;
  for (int t = warp; t < K * A; t += WARPS) {  // phase 1
    const int k = t / A, a = t - k * A;
    const float* r1 = on_ns + (size_t)k * N2;
    float x[C51_R];
#pragma unroll
    for (int r = 0; r < C51_R; ++r) {
      const int c = lane + 32 * r;
      float acc = 0.0f;
      if (c < Z)
        for (int aa = 0; aa < A; ++aa) acc += r1[Z + aa * Z + c];
      const float mean = acc / (float)A;
      x[r] = (c < Z) ? r1[c] + r1[Z + a * Z + c] - mean : -CUDART_INF_F;
    }
    const float ev = c51_expected_value<C51_R>(x, sup, Z, lane);
    if (lane == 0) s_ev[t] = ev;
  }
  __syncthreads();
  const float ret = __ldg(returns + i), nt = __ldg(nonterminals + i), w = __ldg(weights + i);
  for (int k = warp; k < K; k += WARPS) {  // phase 2
    int best = 0;
    float best_ev = -CUDART_INF_F;
    for (int a = 0; a < A; ++a) {
      const float ev = s_ev[k * A + a];
      if (ev > best_ev) {  // first maximum wins, like torch.argmax
        best_ev = ev;
        best = a;
      }
    }
    const float* r = tg_ns + (size_t)k * N2;
    float* qt = q_t + k * Z;
    for (int c = lane; c < Z; c += 32) {
      float mean = 0.0f;
      for (int a = 0; a < A; ++a) mean += r[Z + a * Z + c];
      mean = mean / (float)A;
      qt[c] = r[c] + r[Z + best * Z + c] - mean;
    }
    __syncwarp();
    // c51_core with sample index 0 on per-copy outputs: m_k into s_m[k], a*_k into astar_out[k][i]; its loss row
    // (fed qt again) and gradient are not used
    float g[C51_R];
    c51_core<C51_R, VT>(s_sc[warp], lane, 0, B, A, Z, nullptr, qt, qt, ret, nt, w, support, vmin, vmax, delta_z, gamma_n,
                        s_junk + warp, s_m + k * Z, astar_out ? astar_out + (size_t)k * B + i : nullptr, g, best, support_q,
                        eps);
  }
  __syncthreads();
  for (int c = tid; c < Z; c += C51D_T) {  // phase 3
    float acc = s_m[c];
    for (int k = 1; k < K; ++k) acc = __fadd_rn(acc, s_m[k * Z + c]);
    acc = __fdiv_rn(acc, (float)K);
    s_mavg[c] = acc;
    if (m_out) m_out[(size_t)i * Z + c] = acc;
  }
  __syncthreads();
  const float wi = __fdiv_rn(w, (float)(M * B));
  for (int j = warp; j < M; j += WARPS) {  // phase 4
    const float* r = on_s + (size_t)j * N2;
    float* qs = q_s + j * Z;
    for (int c = lane; c < Z; c += 32) {
      float mean = 0.0f;
      for (int a = 0; a < A; ++a) mean += r[Z + a * Z + c];
      qs[c] = r[c] + r[Z + act * Z + c] - mean / (float)A;
    }
    __syncwarp();
    float m[C51_R], g[C51_R];
#pragma unroll
    for (int rr = 0; rr < C51_R; ++rr) m[rr] = (lane + 32 * rr < Z) ? s_mavg[lane + 32 * rr] : 0.0f;
    const float lj = c51_loss_row<C51_R>(lane, Z, qs, m, wi, g);
    if (lane == 0) s_loss[j] = lj;
#pragma unroll
    for (int rr = 0; rr < C51_R; ++rr)
      if (lane + 32 * rr < Z) s_g[j * Z + lane + 32 * rr] = g[rr];
  }
  __syncthreads();
  if (tid == 0) {  // phase 5
    float acc = s_loss[0];
    for (int j = 1; j < M; ++j) acc = __fadd_rn(acc, s_loss[j]);
    loss[i] = __fdiv_rn(acc, (float)M);
  }
  const float inv_a = 1.0f / (float)A;
  for (int j = 0; j < M; ++j) {
    float* dzi = dz + ((size_t)j * B + i) * N2;
    const float* gj = s_g + j * Z;
    for (int idx = tid; idx < N2; idx += C51D_T) {
      if (idx < Z) {
        dzi[idx] = gj[idx];
      } else {
        const int a = (idx - Z) / Z, c = (idx - Z) - a * Z;
        dzi[idx] = gj[c] * ((a == act ? 1.0f : 0.0f) - inv_a);
      }
    }
  }
}

// ---- HL-Gauss targets (Farebrother et al. 2024; DESIGN.md §20): the scalar double-DQN target as a Gaussian histogram ----
// y = clamp(fl32(ret + fl32(sc ybar)), vmin, vmax).  Bin k is [e_k, e_{k+1}]: e_k = fl32(z_k - h) for k < Z,
// e_Z = fl32(z_{Z-1} + h), h = fl32(delta_z / 2), so the atoms are the bin centres.  t_k = fl32(fl32(e_k - y) c),
// c = fl32(1 / fl32(sqrt(2) sigma)); the mass of N(y, sigma^2) in bin k is u_k = 1/2 (erfc(t_k) - erfc(t_{k+1})) above y,
// 1/2 (erfc(-t_{k+1}) - erfc(-t_k)) below y and 1/2 (erf(t_{k+1}) - erf(t_k)) in the bin holding y: each tail keeps its
// relative accuracy.  U = sum u_k (each lane over its atoms in r order, then the xor butterfly), m_k = fl32(u_k / U), 0
// past Z.  erff / erfcf at full precision.  Returns y; all lanes hold it.
template <int C51_R>
__device__ __forceinline__ float hlg_target(int lane, int Z, const float* __restrict__ support, float delta_z, float vmin,
                                            float vmax, float sigma, float ret, float sc, float ybar, float (&m)[C51_R]) {
  const float y = fminf(fmaxf(__fadd_rn(ret, __fmul_rn(sc, ybar)), vmin), vmax);
  const float h = __fmul_rn(delta_z, 0.5f);
  const float c = __fdiv_rn(1.0f, __fmul_rn(1.41421356f, sigma));
  float u[C51_R], usum = 0.0f;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    const int k = lane + 32 * r;
    u[r] = 0.0f;
    if (k < Z) {
      const float zk = __ldg(support + k);
      const float hi = k + 1 < Z ? __fsub_rn(__ldg(support + k + 1), h) : __fadd_rn(zk, h);
      const float t0 = __fmul_rn(__fsub_rn(__fsub_rn(zk, h), y), c), t1 = __fmul_rn(__fsub_rn(hi, y), c);
      float d;
      if (t0 >= 0.0f) d = __fsub_rn(erfcf(t0), erfcf(t1));
      else if (t1 <= 0.0f) d = __fsub_rn(erfcf(-t1), erfcf(-t0));
      else d = __fsub_rn(erff(t1), erff(t0));
      u[r] = __fmul_rn(0.5f, d);
      usum = __fadd_rn(usum, u[r]);
    }
  }
  usum = warp_sum(usum);
#pragma unroll
  for (int r = 0; r < C51_R; ++r) m[r] = lane + 32 * r < Z ? __fdiv_rn(u[r], usum) : 0.0f;
  return y;
}

// ---- Two-hot targets (Farebrother et al. 2024; MuZero, Schrittwieser et al. 2020, App. F; DESIGN.md §21) ----
// y = clamp(fl32(ret + fl32(sc ybar)), vmin, vmax), or under VT clamp(h(fl32(ret + fl32(sc ybar))), vmin, vmax) (c51_core's
// order for its target atoms: h first, then the clamp).  b = fl32(fl32(y - vmin) / delta_z), l = floor(b), u = ceil(b)
// with c51_core's two fix-ups (so a y on an atom keeps its mass), m_l = fl32(u - b), m_u = fl32(b - l), m_k = 0 elsewhere
// (an index u = Z, where fp32 rounding puts b past Z - 1, is dropped, as c51_core drops it).  Returns y; all lanes hold it.
template <int C51_R, bool VT>
__device__ __forceinline__ float twohot_target(int lane, int Z, float delta_z, float vmin, float vmax, float eps, float ret,
                                               float sc, float ybar, float (&m)[C51_R]) {
  float y = __fadd_rn(ret, __fmul_rn(sc, ybar));
  if constexpr (VT) y = vt_h(y, eps);
  y = fminf(fmaxf(y, vmin), vmax);
  const float b = __fdiv_rn(__fsub_rn(y, vmin), delta_z);
  int lo = (int)floorf(b), up = (int)ceilf(b);
  if (up > 0 && lo == up) lo -= 1;
  if (lo < Z - 1 && lo == up) up += 1;
  const float ml = __fsub_rn((float)up, b), mu = __fsub_rn(b, (float)lo);
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    const int k = lane + 32 * r;
    m[r] = k >= Z ? 0.0f : (k == lo ? ml : (k == up ? mu : 0.0f));
  }
  return y;
}

// The one stage the scalar-target kernels differ in, as a functor the shared bodies below call: stage(lane, Z, ret, sc,
// ybar, m) forms m from ybar and returns y.
template <int C51_R>
struct HlgStage {
  const float* __restrict__ support;
  float delta_z, vmin, vmax, sigma;
  __device__ __forceinline__ float operator()(int lane, int Z, float ret, float sc, float ybar, float (&m)[C51_R]) const {
    return hlg_target<C51_R>(lane, Z, support, delta_z, vmin, vmax, sigma, ret, sc, ybar, m);
  }
};

template <int C51_R, bool VT>
struct TwoHotStage {
  float delta_z, vmin, vmax, eps;
  __device__ __forceinline__ float operator()(int lane, int Z, float ret, float sc, float ybar, float (&m)[C51_R]) const {
    return twohot_target<C51_R, VT>(lane, Z, delta_z, vmin, vmax, eps, ret, sc, ybar, m);
  }
};

// Scalar-target loss on the fused heads' rows, laid out as k_c51_dueling (one CTA of C51D_T threads per sample):
//   phase 0  all threads stage online(s), online(s') and target(s') (stage_z_rows);
//   phase 1  warp a: the expected value of action a of online(s') over sup_ev;
//   phase 2  warp 0: a* (first maximum wins), ybar = the expected value of target(s') at a* over sup_ev, y and m (the
//            stage), then the loss and gradient row of online(s) at the taken action against m (c51_loss_row);
//   phase 3  dz (dueling_dz).
// sup_ev: the support the expected values take (support_q, in return units, under value rescaling).
template <int C51_R, typename Stage>
__device__ __forceinline__ void
c51_dueling_scalar(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
                   const float* __restrict__ returns, const float* __restrict__ nonterminals,
                   const float* __restrict__ weights, const float* __restrict__ sup_ev, float gamma_n, int B, int A, int Z,
                   float* __restrict__ loss, float* __restrict__ dz, float* __restrict__ m_out,
                   int64_t* __restrict__ astar_out, float* __restrict__ y_out, const Stage& stage) {
  extern __shared__ __align__(16) float s_dyn[];
  const int N2 = Z + A * Z;
  float* zs = s_dyn;              // [3][N2]: online(s), online(s'), target(s')
  float* q_s = zs + 3 * N2;       // [Z] online logits of the taken action
  float* s_g = q_s + Z;           // [Z] gradient row
  float* s_ev = s_g + Z;          // [A] expected values
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  stage_z_rows<C51D_T>(zs, z_on, z_tg, i, B, N2, 1, 1);
  __syncthreads();
  const int act = (int)actions[i];
  float sup[C51_R];
#pragma unroll
  for (int r = 0; r < C51_R; ++r) sup[r] = (lane + 32 * r < Z) ? __ldg(sup_ev + lane + 32 * r) : 0.0f;
  {  // phase 1
    const float* r1 = zs + N2;
    float mean[C51_R];
#pragma unroll
    for (int r = 0; r < C51_R; ++r) mean[r] = lane + 32 * r < Z ? dueling_mean(r1, A, Z, lane + 32 * r) : 0.0f;
    for (int a = warp; a < A; a += C51D_T / 32) {
      float x[C51_R];
#pragma unroll
      for (int r = 0; r < C51_R; ++r) {
        const int c = lane + 32 * r;
        x[r] = (c < Z) ? dueling_q(r1[c], r1[Z + a * Z + c], mean[r]) : -CUDART_INF_F;
      }
      const float ev = c51_expected_value<C51_R>(x, sup, Z, lane);
      if (lane == 0) s_ev[a] = ev;
    }
  }
  __syncthreads();
  if (warp == 0) {  // phase 2
    const int best = first_argmax(s_ev, A);
    float x[C51_R];
#pragma unroll
    for (int r = 0; r < C51_R; ++r) {
      const int c = lane + 32 * r;
      x[r] = (c < Z) ? dueling_q(zs + 2 * N2, A, Z, c, best) : -CUDART_INF_F;
      if (c < Z) q_s[c] = dueling_q(zs, A, Z, c, act);
    }
    __syncwarp();
    const float ybar = c51_expected_value<C51_R>(x, sup, Z, lane);
    float m[C51_R], g[C51_R];
    const float y = stage(lane, Z, __ldg(returns + i), __fmul_rn(__ldg(nonterminals + i), gamma_n), ybar, m);
    const float l = c51_loss_row<C51_R>(lane, Z, q_s, m, __fdiv_rn(__ldg(weights + i), (float)B), g);
    if (lane == 0) {
      loss[i] = l;
      if (astar_out) astar_out[i] = best;
      if (y_out) y_out[i] = y;
    }
#pragma unroll
    for (int r = 0; r < C51_R; ++r) {
      const int c = lane + 32 * r;
      if (c < Z) {
        s_g[c] = g[r];
        if (m_out) m_out[(size_t)i * Z + c] = m[r];
      }
    }
  }
  __syncthreads();
  dueling_dz<C51D_T>(dz + (size_t)i * N2, s_g, A, Z, act);  // phase 3
}

// Scalar-target loss on plain logit rows [B][A][Z] (the library head), k_c51's layout: one warp per sample, grad [B][A][Z]
// zero but for the taken action's row.  sup_ev as in c51_dueling_scalar.
template <int C51_R, typename Stage>
__device__ __forceinline__ void
c51_scalar(const float* __restrict__ q_on_s, const float* __restrict__ q_on_ns, const float* __restrict__ q_tg_ns,
           const int64_t* __restrict__ actions, const float* __restrict__ returns, const float* __restrict__ nonterminals,
           const float* __restrict__ weights, const float* __restrict__ sup_ev, float gamma_n, int B, int A, int Z,
           float* __restrict__ loss, float* __restrict__ grad, float* __restrict__ m_out, int64_t* __restrict__ astar_out,
           float* __restrict__ y_out, const Stage& stage) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * C51_WARPS + warp;
  if (i >= B) return;
  const int act = (int)actions[i];
  float sup[C51_R], x[C51_R];
#pragma unroll
  for (int r = 0; r < C51_R; ++r) sup[r] = (lane + 32 * r < Z) ? __ldg(sup_ev + lane + 32 * r) : 0.0f;
  int best = 0;
  float best_ev = -CUDART_INF_F;
  for (int a = 0; a < A; ++a) {
    const float* row = q_on_ns + ((size_t)i * A + a) * Z;
#pragma unroll
    for (int r = 0; r < C51_R; ++r) x[r] = (lane + 32 * r < Z) ? row[lane + 32 * r] : -CUDART_INF_F;
    const float ev = c51_expected_value<C51_R>(x, sup, Z, lane);
    if (ev > best_ev) {  // first maximum wins, like torch.argmax
      best_ev = ev;
      best = a;
    }
  }
  const float* row_t = q_tg_ns + ((size_t)i * A + best) * Z;
#pragma unroll
  for (int r = 0; r < C51_R; ++r) x[r] = (lane + 32 * r < Z) ? row_t[lane + 32 * r] : -CUDART_INF_F;
  const float ybar = c51_expected_value<C51_R>(x, sup, Z, lane);
  float m[C51_R], g[C51_R];
  const float y = stage(lane, Z, __ldg(returns + i), __fmul_rn(__ldg(nonterminals + i), gamma_n), ybar, m);
  const float l = c51_loss_row<C51_R>(lane, Z, q_on_s + ((size_t)i * A + act) * Z, m,
                                      __fdiv_rn(__ldg(weights + i), (float)B), g);
  if (lane == 0) {
    loss[i] = l;
    if (astar_out) astar_out[i] = best;
    if (y_out) y_out[i] = y;
  }
  float* gq = grad + (size_t)i * A * Z;
  for (int j = lane; j < A * Z; j += 32) gq[j] = 0.0f;
  __syncwarp();
#pragma unroll
  for (int r = 0; r < C51_R; ++r) {
    const int c = lane + 32 * r;
    if (c < Z) {
      gq[(size_t)act * Z + c] = g[r];
      if (m_out) m_out[(size_t)i * Z + c] = m[r];
    }
  }
}

// HL-Gauss loss on the fused heads' rows: c51_dueling_scalar with hlg_target, the expected values over the support.
template <int C51_R>
__global__ void __launch_bounds__(C51D_T)
k_c51_dueling_hlg(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
                  const float* __restrict__ returns, const float* __restrict__ nonterminals,
                  const float* __restrict__ weights, const float* __restrict__ support, float vmin, float vmax,
                  float delta_z, float gamma_n, float sigma, int B, int A, int Z, float* __restrict__ loss,
                  float* __restrict__ dz, float* __restrict__ m_out, int64_t* __restrict__ astar_out,
                  float* __restrict__ y_out) {
  c51_dueling_scalar<C51_R>(z_on, z_tg, actions, returns, nonterminals, weights, support, gamma_n, B, A, Z, loss, dz, m_out,
                            astar_out, y_out, HlgStage<C51_R>{support, delta_z, vmin, vmax, sigma});
}

// HL-Gauss loss on plain logit rows [B][A][Z] (the library head): c51_scalar with hlg_target.
template <int C51_R>
__global__ void __launch_bounds__(C51_WARPS * 32)
k_c51_hlg(const float* __restrict__ q_on_s, const float* __restrict__ q_on_ns, const float* __restrict__ q_tg_ns,
          const int64_t* __restrict__ actions, const float* __restrict__ returns, const float* __restrict__ nonterminals,
          const float* __restrict__ weights, const float* __restrict__ support, float vmin, float vmax, float delta_z,
          float gamma_n, float sigma, int B, int A, int Z, float* __restrict__ loss, float* __restrict__ grad,
          float* __restrict__ m_out, int64_t* __restrict__ astar_out, float* __restrict__ y_out) {
  c51_scalar<C51_R>(q_on_s, q_on_ns, q_tg_ns, actions, returns, nonterminals, weights, support, gamma_n, B, A, Z, loss, grad,
                    m_out, astar_out, y_out, HlgStage<C51_R>{support, delta_z, vmin, vmax, sigma});
}

// Two-hot loss on the fused heads' rows: c51_dueling_scalar with twohot_target.  VT (value rescaling): the expected values
// (arg-max and ybar) over support_q, y = h(.) before the clamp; support_q / eps are read only there.
template <int C51_R, bool VT>
__global__ void __launch_bounds__(C51D_T)
k_c51_dueling_twohot(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
                     const float* __restrict__ returns, const float* __restrict__ nonterminals,
                     const float* __restrict__ weights, const float* __restrict__ support, float vmin, float vmax,
                     float delta_z, float gamma_n, int B, int A, int Z, float* __restrict__ loss, float* __restrict__ dz,
                     float* __restrict__ m_out, int64_t* __restrict__ astar_out, float* __restrict__ y_out,
                     const float* __restrict__ support_q, float eps) {
  c51_dueling_scalar<C51_R>(z_on, z_tg, actions, returns, nonterminals, weights, VT ? support_q : support, gamma_n, B, A, Z,
                            loss, dz, m_out, astar_out, y_out, TwoHotStage<C51_R, VT>{delta_z, vmin, vmax, eps});
}

// Two-hot loss on plain logit rows [B][A][Z] (the library head): c51_scalar with twohot_target; VT as above.
template <int C51_R, bool VT>
__global__ void __launch_bounds__(C51_WARPS * 32)
k_c51_twohot(const float* __restrict__ q_on_s, const float* __restrict__ q_on_ns, const float* __restrict__ q_tg_ns,
             const int64_t* __restrict__ actions, const float* __restrict__ returns, const float* __restrict__ nonterminals,
             const float* __restrict__ weights, const float* __restrict__ support, float vmin, float vmax, float delta_z,
             float gamma_n, int B, int A, int Z, float* __restrict__ loss, float* __restrict__ grad,
             float* __restrict__ m_out, int64_t* __restrict__ astar_out, float* __restrict__ y_out,
             const float* __restrict__ support_q, float eps) {
  c51_scalar<C51_R>(q_on_s, q_on_ns, q_tg_ns, actions, returns, nonterminals, weights, VT ? support_q : support, gamma_n, B,
                    A, Z, loss, grad, m_out, astar_out, y_out, TwoHotStage<C51_R, VT>{delta_z, vmin, vmax, eps});
}

// ================================================================================================
// Q-values for acting / evaluation (agent.py:53-55 act, :110-112 evaluate_q): one warp per state.
// From the head output z = (z_value | z_advantage): q[a][z] = zv + za[a] - mean_a za (model.py:75), softmax over
// atoms (model.py:79), expected value sum_z support_z p_z (agent.py:55), then the arg-max / max over actions --
// everything after the network body in ONE launch, results stay on the device (no .item() per state).
// ================================================================================================
// RISK: c51_risk_value in place of the expected value (risk_kind / risk_eta are read only there).
template <bool RISK>
__global__ void __launch_bounds__(128)
k_q_select(const float* __restrict__ z, int M, int A, int Z, const float* __restrict__ support,
           float* __restrict__ q_out, int64_t* __restrict__ best_action, float* __restrict__ best_q, int risk_kind,
           float risk_eta) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * 4 + warp;
  if (m >= M) return;
  const float* zr = z + (size_t)m * (Z + A * Z);
  constexpr int R = RB_MAX_ATOMS / 32;
  float sup[R], zv[R], mean[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int c = lane + 32 * r;
    sup[r] = zv[r] = mean[r] = 0.0f;
    if (c < Z) {
      sup[r] = __ldg(support + c);
      zv[r] = __ldg(zr + c);
      mean[r] = dueling_mean<true>(zr, A, Z, c);
    }
  }
  int best = 0;
  float best_ev = -CUDART_INF_F;
  for (int a = 0; a < A; ++a) {
    float x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      x[r] = (c < Z) ? dueling_q(zv[r], __ldg(zr + Z + a * Z + c), mean[r]) : -CUDART_INF_F;
    }
    float ev;
    if constexpr (RISK) ev = c51_risk_value<R>(x, sup, Z, lane, risk_kind, risk_eta);
    else ev = c51_expected_value<R>(x, sup, Z, lane);
    if (q_out && lane == 0) q_out[(size_t)m * A + a] = ev;
    if (ev > best_ev) {   // first maximum wins, like torch.argmax / max
      best_ev = ev;
      best = a;
    }
  }
  if (lane == 0) {
    if (best_action) best_action[m] = best;
    if (best_q) best_q[m] = best_ev;
  }
}

// ================================================================================================
// Quantile regression (QR-DQN, Dabney et al. 2018): loss, gradient and the mean-quantile greedy values.
// ================================================================================================
// N quantiles per action at the midpoints tau_i = (2i + 1) / (2N).  For sample b with taken action a:
//   theta_i = q_online(s, a)_i,  a* = argmax_a mean_j q_online(s', a)_j (first maximum wins),
//   T_j = r + fl32(nt gamma_n) q_target(s', a*)_j,  u_ij = T_j - theta_i,
//   loss = sum_i (1/N) sum_j |tau_i - [u_ij < 0]| H_kappa(u_ij) / kappa       (also the priority),
//   g_i  = -(w / B) (1/N) sum_j |tau_i - [u_ij < 0]| clamp(u_ij, -kappa, kappa) / kappa.
// One CTA of QR_T threads per sample (k_qr_dueling on the fused heads' z rows, k_qr on plain [B][A][N] rows):
//   phase 1  warp a: the mean quantile of action a of online(s') (lane owns quantiles lane + 32 r) into s_mean[a];
//   phase 2  a* (every thread runs the same scan of s_mean), then the rows theta and T into shared memory;
//   phase 3  warp w takes the online quantiles i = w, w + 8, ...: each lane sums its R target quantiles, two interleaved
//            butterflies finish sum_j; the loss sum of row i and g_i land in shared memory (qr_core);
//   phase 4  warp 0 sums the rows' loss sums in i order; all threads write the gradient rows.
// Every sum runs in a fixed order: an eager launch and a graph replay agree bitwise.
constexpr int QR_T = 256;
constexpr int QR_WARPS = QR_T / 32;

// mean of one row held as x[r] = quantile lane + 32 r (0 past N); every lane returns it
template <int R>
__device__ __forceinline__ float qr_row_mean(const float (&x)[R], int N) {
  float s = 0.0f;
#pragma unroll
  for (int r = 0; r < R; ++r) s = __fadd_rn(s, x[r]);
  return __fdiv_rn(warp_sum(s), (float)N);
}

// Target quantile T = r + scale q with scale = fl32(nt gamma_n); VT: h(r + scale h^-1(q)), q in h units
template <bool VT>
__device__ __forceinline__ float qr_target(float ret, float scale, float q, float eps) {
  if constexpr (VT) return vt_h(__fadd_rn(ret, __fmul_rn(scale, vt_hinv(q, eps))), eps);
  return __fadd_rn(ret, __fmul_rn(scale, q));
}

// Phases 3 and 4 (without the gradient write) from the rows s_theta, s_T [N] in shared memory: s_g [N] receives the
// gradient row of the taken action, loss[i_sample] the loss (written by warp 0; loss may be global or shared: the
// averaging kernel passes its per-copy slots); s_l is N floats of scratch.  s_g is complete on return; a caller that
// runs it again on the same s_l synchronises first (warp 0 may still read it).
template <int R>
__device__ __forceinline__ void qr_core(const float* s_theta, const float* s_T, float* s_l, float* s_g, int N, float kappa,
                                        float wi, int i_sample, float* __restrict__ loss) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float t[R];
#pragma unroll
  for (int r = 0; r < R; ++r) t[r] = (lane + 32 * r < N) ? s_T[lane + 32 * r] : 0.0f;
  const float nk = __fmul_rn((float)N, kappa), half_k = 0.5f * kappa;
  for (int i = warp; i < N; i += QR_WARPS) {
    const float th = s_theta[i];
    const float tau_lo = __fdiv_rn((float)(2 * i + 1), (float)(2 * N));        // |tau_i - 0|
    const float tau_hi = __fdiv_rn((float)(2 * (N - i) - 1), (float)(2 * N));  // |tau_i - 1|
    float sl = 0.0f, sg = 0.0f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (lane + 32 * r < N) {
        const float u = __fsub_rn(t[r], th), au = fabsf(u);
        const float tw = u < 0.0f ? tau_hi : tau_lo;
        const float h = au <= kappa ? __fmul_rn(__fmul_rn(0.5f, u), u) : __fmul_rn(kappa, __fsub_rn(au, half_k));
        sl = __fadd_rn(sl, __fmul_rn(tw, h));
        sg = __fadd_rn(sg, __fmul_rn(tw, fminf(fmaxf(u, -kappa), kappa)));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sl = __fadd_rn(sl, __shfl_xor_sync(0xffffffffu, sl, o));
      sg = __fadd_rn(sg, __shfl_xor_sync(0xffffffffu, sg, o));
    }
    if (lane == 0) {
      s_l[i] = sl;
      s_g[i] = -__fmul_rn(wi, __fdiv_rn(sg, nk));
    }
  }
  __syncthreads();
  if (warp == 0) {
    float s = 0.0f;
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (lane + 32 * r < N) s = __fadd_rn(s, s_l[lane + 32 * r]);
    s = warp_sum(s);
    if (lane == 0) loss[i_sample] = __fdiv_rn(s, nk);
  }
}

// Dueling entry point: z rows as k_c51_dueling takes them (online 2B rows, s then s'; target B rows).
// VT (value rescaling, quantiles in h units): a* = argmax_a mean_j h^-1(q_online(s', a)_j) and
// T_j = h(r + fl32(scale * h^-1(q_target(s', a*)_j))); theta, the loss and the gradient stay in h units.
// RISK (R with RISK_INST set): phase 1 computes qr_risk_value in place of the mean (risk_kind / risk_eta are read
// only there).
template <int R_RISK, bool VT>
__global__ void __launch_bounds__(QR_T)
k_qr_dueling(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
             const float* __restrict__ returns, const float* __restrict__ nonterminals,
             const float* __restrict__ weights, float kappa, float gamma_n, int B, int A, int N,
             float* __restrict__ loss, float* __restrict__ dz, float* __restrict__ theta_out,
             int64_t* __restrict__ astar_out, float eps, int risk_kind, float risk_eta) {
  constexpr int R = R_RISK & ~RISK_INST;
  constexpr bool RISK = (R_RISK & RISK_INST) != 0;
  extern __shared__ __align__(16) float s_dyn[];
  const int N2 = N + A * N;
  float* zs = s_dyn;              // [3][N2]: online(s), online(s'), target(s')
  float* s_theta = zs + 3 * N2;   // [N] online quantiles of the taken action
  float* s_T = s_theta + N;       // [N] target quantiles T_j
  float* s_g = s_T + N;           // [N] gradient row
  float* s_l = s_g + N;           // [N] loss sum of every online quantile
  float* s_mean = s_l + N;        // [A] mean quantile of every action of online(s')
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  stage_z_rows<QR_T>(zs, z_on, z_tg, i, B, N2, 1, 1);  // phase 0
  __syncthreads();
  const int act = (int)actions[i];
  {  // phase 1
    const float* r1 = zs + N2;
    float mean[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      mean[r] = (c < N) ? dueling_mean(r1, A, N, c) : 0.0f;
    }
    float w[R];
    if constexpr (RISK) qr_risk_weights<R>(N, lane, risk_kind, risk_eta, w);
    for (int a = warp; a < A; a += QR_WARPS) {
      float x[R];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int c = lane + 32 * r;
        x[r] = (c < N) ? dueling_q(r1[c], r1[N + a * N + c], mean[r]) : 0.0f;
        if constexpr (VT) x[r] = (c < N) ? vt_hinv(x[r], eps) : 0.0f;
      }
      float q;
      if constexpr (RISK) q = qr_risk_value<R>(x, w, N, lane);
      else q = qr_row_mean<R>(x, N);
      if (lane == 0) s_mean[a] = q;
    }
  }
  __syncthreads();
  const int best = first_argmax(s_mean, A);  // phase 2
  if (astar_out && tid == 0) astar_out[i] = best;
  const float ret = __ldg(returns + i), scale = __fmul_rn(__ldg(nonterminals + i), gamma_n);
  for (int c = tid; c < N; c += QR_T) {
    s_theta[c] = dueling_q(zs, A, N, c, act);
    const float T = qr_target<VT>(ret, scale, dueling_q(zs + 2 * N2, A, N, c, best), eps);
    s_T[c] = T;
    if (theta_out) theta_out[(size_t)i * N + c] = T;
  }
  __syncthreads();
  qr_core<R>(s_theta, s_T, s_l, s_g, N, kappa, __fdiv_rn(__ldg(weights + i), (float)B), i, loss);
  dueling_dz<QR_T>(dz + (size_t)i * N2, s_g, A, N, act);  // phase 4
}

// DrQ's K / M averaging under the quantile loss: z rows as k_c51_dueling_avg takes them (z_on (M + K) B rows, copy j of s
// at row jB + i, copy k of s' at row (M + k) B + i; z_tg K B rows, copy k of s' at row kB + i).  ONE CTA PER SAMPLE with
// the sample's M + 2K z rows staged in shared memory:
//   phase 1  the mean quantile of every (target copy k, action a) of online(s'_k), one warp per pair (k_qr_dueling's
//            phase 1 per pair, bitwise);
//   phase 2  thread k: a*_k (first maximum wins); then per quantile n, T_k,n (qr_target) and
//            Tbar_n = (sum_k T_k,n in k order) / K, rounded once -- the quantile-wise average of the K target quantile
//            functions (in h units under VT), not the mixture of their K N samples; theta_j of every online copy;
//   phase 3  qr_core once per online copy j against Tbar, with wi = w / (M B): loss_j and g_j;
//   phase 4  loss = (sum_j loss_j in j order) / M; dz rows jB + i from g_j (dueling_dz).
// At M = K = 1 every output is k_qr_dueling's, bitwise.
template <int R, bool VT>
__global__ void __launch_bounds__(QR_T)
k_qr_dueling_avg(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
                 const float* __restrict__ returns, const float* __restrict__ nonterminals,
                 const float* __restrict__ weights, float kappa, float gamma_n, int B, int A, int N, int M, int K,
                 float* __restrict__ loss, float* __restrict__ dz, float* __restrict__ theta_out,
                 int64_t* __restrict__ astar_out, float eps) {
  extern __shared__ __align__(16) float s_dyn[];
  __shared__ int s_best[RB_MAX_AUG_COPIES];
  const int N2 = N + A * N;
  const int rows = M + 2 * K;
  float* zs = s_dyn;                 // [M + 2K][N2]: online(s_j), online(s'_k), target(s'_k)
  float* s_theta = zs + rows * N2;   // [M][N] online quantiles of the taken action, per copy
  float* s_T = s_theta + M * N;      // [N] averaged target quantiles Tbar
  float* s_g = s_T + N;              // [M][N] gradient rows
  float* s_l = s_g + M * N;          // [N] qr_core's loss sums
  float* s_mean = s_l + N;           // [K][A] mean quantile of every action of online(s'_k)
  float* s_loss = s_mean + K * A;    // [M] loss_j
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  stage_z_rows<QR_T>(zs, z_on, z_tg, i, B, N2, M, K);  // phase 0
  __syncthreads();
  const int act = (int)actions[i];
  for (int t = warp; t < K * A; t += QR_WARPS) {  // phase 1
    const int k = t / A, a = t - k * A;
    const float* r1 = zs + (size_t)(M + k) * N2;
    float x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      x[r] = (c < N) ? dueling_q(r1, A, N, c, a) : 0.0f;
      if constexpr (VT) x[r] = (c < N) ? vt_hinv(x[r], eps) : 0.0f;
    }
    const float q = qr_row_mean<R>(x, N);
    if (lane == 0) s_mean[t] = q;
  }
  __syncthreads();
  if (tid < K) {  // phase 2
    const int best = first_argmax(s_mean + tid * A, A);
    s_best[tid] = best;
    if (astar_out) astar_out[(size_t)tid * B + i] = best;
  }
  __syncthreads();
  const float ret = __ldg(returns + i), scale = __fmul_rn(__ldg(nonterminals + i), gamma_n);
  for (int c = tid; c < N; c += QR_T) {
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) {
      const float T = qr_target<VT>(ret, scale, dueling_q(zs + (size_t)(M + K + k) * N2, A, N, c, s_best[k]), eps);
      acc = (k == 0) ? T : __fadd_rn(acc, T);
    }
    const float Tbar = __fdiv_rn(acc, (float)K);
    s_T[c] = Tbar;
    if (theta_out) theta_out[(size_t)i * N + c] = Tbar;
    for (int j = 0; j < M; ++j) s_theta[j * N + c] = dueling_q(zs + (size_t)j * N2, A, N, c, act);
  }
  __syncthreads();
  const float wi = __fdiv_rn(__ldg(weights + i), (float)(M * B));
  for (int j = 0; j < M; ++j) {  // phase 3
    qr_core<R>(s_theta + j * N, s_T, s_l, s_g + j * N, N, kappa, wi, j, s_loss);
    __syncthreads();   // warp 0 has read s_l and written s_loss[j]
  }
  if (tid == 0) {  // phase 4
    float acc = s_loss[0];
    for (int j = 1; j < M; ++j) acc = __fadd_rn(acc, s_loss[j]);
    loss[i] = __fdiv_rn(acc, (float)M);
  }
  for (int j = 0; j < M; ++j) dueling_dz<QR_T>(dz + ((size_t)j * B + i) * N2, s_g + j * N, A, N, act);
}

// Plain entry point: quantile rows [B][A][N] of online(s), online(s') and target(s'); grad [B][A][N] is the gradient row
// at the taken action and 0 elsewhere.
// RISK: as k_qr_dueling's.
template <int R_RISK, bool VT>
__global__ void __launch_bounds__(QR_T)
k_qr(const float* __restrict__ q_on_s, const float* __restrict__ q_on_ns, const float* __restrict__ q_tg_ns,
     const int64_t* __restrict__ actions, const float* __restrict__ returns, const float* __restrict__ nonterminals,
     const float* __restrict__ weights, float kappa, float gamma_n, int B, int A, int N, float* __restrict__ loss,
     float* __restrict__ grad, float* __restrict__ theta_out, int64_t* __restrict__ astar_out, float eps,
     int risk_kind, float risk_eta) {
  constexpr int R = R_RISK & ~RISK_INST;
  constexpr bool RISK = (R_RISK & RISK_INST) != 0;
  extern __shared__ __align__(16) float s_dyn[];
  float* s_theta = s_dyn;
  float* s_T = s_theta + N;
  float* s_g = s_T + N;
  float* s_l = s_g + N;
  float* s_mean = s_l + N;        // [A]
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const size_t row0 = (size_t)i * A;
  float w[R];
  if constexpr (RISK) qr_risk_weights<R>(N, lane, risk_kind, risk_eta, w);
  for (int a = warp; a < A; a += QR_WARPS) {  // phase 1
    float x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      x[r] = (c < N) ? __ldg(q_on_ns + (row0 + a) * N + c) : 0.0f;
      if constexpr (VT) x[r] = (c < N) ? vt_hinv(x[r], eps) : 0.0f;
    }
    float q;
    if constexpr (RISK) q = qr_risk_value<R>(x, w, N, lane);
    else q = qr_row_mean<R>(x, N);
    if (lane == 0) s_mean[a] = q;
  }
  __syncthreads();
  const int act = (int)actions[i];
  const int best = first_argmax(s_mean, A);  // phase 2
  if (astar_out && tid == 0) astar_out[i] = best;
  const float ret = __ldg(returns + i), scale = __fmul_rn(__ldg(nonterminals + i), gamma_n);
  for (int c = tid; c < N; c += QR_T) {
    s_theta[c] = __ldg(q_on_s + (row0 + act) * N + c);
    const float T = qr_target<VT>(ret, scale, __ldg(q_tg_ns + (row0 + best) * N + c), eps);
    s_T[c] = T;
    if (theta_out) theta_out[(size_t)i * N + c] = T;
  }
  __syncthreads();
  qr_core<R>(s_theta, s_T, s_l, s_g, N, kappa, __fdiv_rn(__ldg(weights + i), (float)B), i, loss);
  float* gq = grad + row0 * N;
  for (int idx = tid; idx < A * N; idx += QR_T) {
    const int a = idx / N;
    gq[idx] = (a == act) ? s_g[idx - a * N] : 0.0f;
  }
}

// ---- Munchausen targets under the quantile loss (M-RL, Vieillard et al. 2020; DESIGN.md §17) ----
// q(x, a) = (1/N) sum_j theta_j(x, a) of the TARGET net (qr_row_mean of the dueling combination, k_qr_dueling's phase 1).
// Per row q[A]: m = max_a q_a, e_a = exp((q_a - m) / tau), S = sum_a e_a in action order, pi_a = e_a / S and
// l_a = (q_a - m) - tau log S = tau ln pi_a in the stable form (<= 0 exactly: S >= 1).  For sample i, taken action a:
//   b   = alpha max(l_a(s), l0)                                          (target row of s)
//   c_j = sum_a' pi_a'(s') (theta_j(s', a') - l_a'(s')) in action order   (target row of s')
//   T_j = fl32(r + b) + fl32(fl32(nt gamma_n) c_j)
// then qr_core against T.  expf / logf at full precision; every other step rounded explicitly.

// One row's policy from its A mean quantiles q: pi [A] and l [A] (either may be NULL); returns l_act (act in [0, A)) or 0.
__device__ __forceinline__ float munchausen_policy(const float* q, int A, float tau, float* pi, float* ell, int act) {
  float m = q[0];
  for (int a = 1; a < A; ++a) m = fmaxf(m, q[a]);
  float S = 0.0f;
  for (int a = 0; a < A; ++a) S = __fadd_rn(S, expf(__fdiv_rn(__fsub_rn(q[a], m), tau)));
  const float tlog = __fmul_rn(tau, logf(S));
  float l_act = 0.0f;
  for (int a = 0; a < A; ++a) {
    const float d = __fsub_rn(q[a], m);
    const float l = __fsub_rn(d, tlog);
    if (pi) pi[a] = __fdiv_rn(expf(__fdiv_rn(d, tau)), S);
    if (ell) ell[a] = l;
    if (a == act) l_act = l;
  }
  return l_act;
}

// The scalar stage both Munchausen kernels share, after phase 1 has left the target mean quantiles in s_q [2][A] (row 0:
// s, row 1: s'): warp 0 lane 0 forms b from row 0 into *s_b (and bonus_out), warp 1 lane 0 pi and l of row 1 into s_pi,
// s_ell.  The caller synchronises afterwards.
__device__ __forceinline__ void munchausen_stage(const float* s_q, float* s_pi, float* s_ell, float* s_b, int A, int act,
                                                 float alpha, float tau, float l0, int i, float* __restrict__ bonus_out) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    const float b = __fmul_rn(alpha, fmaxf(munchausen_policy(s_q, A, tau, nullptr, nullptr, act), l0));
    *s_b = b;
    if (bonus_out) bonus_out[i] = b;
  } else if (tid == 32) {
    munchausen_policy(s_q + A, A, tau, s_pi, s_ell, -1);
  }
}

// c_j of one quantile from the s' quantiles theta_j(s', a') = q(a'), summed over a' in action order
template <typename Q>
__device__ __forceinline__ float munchausen_soft_value(const Q& q, const float* s_pi, const float* s_ell, int A) {
  float acc = 0.0f;
  for (int a = 0; a < A; ++a) acc = __fadd_rn(acc, __fmul_rn(s_pi[a], __fsub_rn(q(a), s_ell[a])));
  return acc;
}

// Stage sample i's three z rows into zs [3][N2] with all T threads: online(s) from z_on row i, target(s) from z_tg row i,
// target(s') from z_tg row B + i (stage_z_rows' pattern: every load issued before any is waited on).
template <int T>
__device__ __forceinline__ void stage_munchausen_rows(float* zs, const float* __restrict__ z_on,
                                                      const float* __restrict__ z_tg, int i, int B, int N2) {
  const int total = 3 * N2;
  for (int base = threadIdx.x; base < total; base += T * 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int idx = base + u * T;
      v[u] = 0.0f;
      if (idx < total) {
        const int t = idx / N2;
        const float* src = t == 0 ? z_on + (size_t)i * N2 : z_tg + (size_t)(t == 1 ? i : B + i) * N2;
        v[u] = __ldg(src + (idx - t * N2));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int idx = base + u * T;
      if (idx < total) zs[idx] = v[u];
    }
  }
}

// Dueling entry point: z_on B rows (s), z_tg 2B rows (s, then s').  One CTA of QR_T threads per sample:
//   phase 0  stage online(s), target(s), target(s');
//   phase 1  the 2A target mean quantiles, one warp per (row, action), into s_q;
//   phase 2  m, S, pi, l of both rows (munchausen_stage), then b and T_j per quantile, theta of the taken action;
//   phase 3  qr_core; phase 4 dueling_dz.
template <int R>
__global__ void __launch_bounds__(QR_T)
k_qr_dueling_munchausen(const float* __restrict__ z_on, const float* __restrict__ z_tg, const int64_t* __restrict__ actions,
                        const float* __restrict__ returns, const float* __restrict__ nonterminals,
                        const float* __restrict__ weights, float kappa, float gamma_n, float alpha, float tau, float l0,
                        int B, int A, int N, float* __restrict__ loss, float* __restrict__ dz,
                        float* __restrict__ theta_out, float* __restrict__ bonus_out) {
  extern __shared__ __align__(16) float s_dyn[];
  __shared__ float s_b;
  const int N2 = N + A * N;
  float* zs = s_dyn;              // [3][N2]: online(s), target(s), target(s')
  float* s_theta = zs + 3 * N2;   // [N] online quantiles of the taken action
  float* s_T = s_theta + N;       // [N] target quantiles T_j
  float* s_g = s_T + N;           // [N] gradient row
  float* s_l = s_g + N;           // [N] loss sum of every online quantile
  float* s_q = s_l + N;           // [2][A] target mean quantiles of s and s'
  float* s_pi = s_q + 2 * A;      // [A] pi(s')
  float* s_ell = s_pi + A;        // [A] l(s')
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  stage_munchausen_rows<QR_T>(zs, z_on, z_tg, i, B, N2);  // phase 0
  __syncthreads();
  const int act = (int)actions[i];
  for (int t = warp; t < 2 * A; t += QR_WARPS) {  // phase 1
    const int row = t / A, a = t - row * A;
    const float* r1 = zs + (size_t)(1 + row) * N2;
    float x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      x[r] = (c < N) ? dueling_q(r1, A, N, c, a) : 0.0f;
    }
    const float q = qr_row_mean<R>(x, N);
    if (lane == 0) s_q[t] = q;
  }
  __syncthreads();
  munchausen_stage(s_q, s_pi, s_ell, &s_b, A, act, alpha, tau, l0, i, bonus_out);  // phase 2
  __syncthreads();
  const float ret = __ldg(returns + i), scale = __fmul_rn(__ldg(nonterminals + i), gamma_n);
  const float rb = __fadd_rn(ret, s_b);
  const float* r2 = zs + 2 * N2;
  for (int c = tid; c < N; c += QR_T) {
    s_theta[c] = dueling_q(zs, A, N, c, act);
    const float v = r2[c], mean = dueling_mean(r2, A, N, c);
    const float cj = munchausen_soft_value([&](int a) { return dueling_q(v, r2[N + a * N + c], mean); }, s_pi, s_ell, A);
    const float T = __fadd_rn(rb, __fmul_rn(scale, cj));
    s_T[c] = T;
    if (theta_out) theta_out[(size_t)i * N + c] = T;
  }
  __syncthreads();
  qr_core<R>(s_theta, s_T, s_l, s_g, N, kappa, __fdiv_rn(__ldg(weights + i), (float)B), i, loss);  // phase 3
  dueling_dz<QR_T>(dz + (size_t)i * N2, s_g, A, N, act);  // phase 4
}

// Plain entry point: quantile rows [B][A][N] of online(s), target(s) and target(s'); grad [B][A][N] as k_qr writes it.
template <int R>
__global__ void __launch_bounds__(QR_T)
k_qr_munchausen(const float* __restrict__ q_on_s, const float* __restrict__ q_tg_s, const float* __restrict__ q_tg_ns,
                const int64_t* __restrict__ actions, const float* __restrict__ returns,
                const float* __restrict__ nonterminals, const float* __restrict__ weights, float kappa, float gamma_n,
                float alpha, float tau, float l0, int B, int A, int N, float* __restrict__ loss, float* __restrict__ grad,
                float* __restrict__ theta_out, float* __restrict__ bonus_out) {
  extern __shared__ __align__(16) float s_dyn[];
  __shared__ float s_b;
  float* s_theta = s_dyn;
  float* s_T = s_theta + N;
  float* s_g = s_T + N;
  float* s_l = s_g + N;
  float* s_q = s_l + N;           // [2][A]
  float* s_pi = s_q + 2 * A;      // [A]
  float* s_ell = s_pi + A;        // [A]
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const size_t row0 = (size_t)i * A;
  for (int t = warp; t < 2 * A; t += QR_WARPS) {  // phase 1
    const int row = t / A, a = t - row * A;
    const float* src = (row == 0 ? q_tg_s : q_tg_ns) + (row0 + a) * N;
    float x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      x[r] = (c < N) ? __ldg(src + c) : 0.0f;
    }
    const float q = qr_row_mean<R>(x, N);
    if (lane == 0) s_q[t] = q;
  }
  __syncthreads();
  const int act = (int)actions[i];
  munchausen_stage(s_q, s_pi, s_ell, &s_b, A, act, alpha, tau, l0, i, bonus_out);  // phase 2
  __syncthreads();
  const float ret = __ldg(returns + i), scale = __fmul_rn(__ldg(nonterminals + i), gamma_n);
  const float rb = __fadd_rn(ret, s_b);
  const float* tn = q_tg_ns + row0 * N;
  for (int c = tid; c < N; c += QR_T) {
    s_theta[c] = __ldg(q_on_s + (row0 + act) * N + c);
    const float cj = munchausen_soft_value([&](int a) { return __ldg(tn + (size_t)a * N + c); }, s_pi, s_ell, A);
    const float T = __fadd_rn(rb, __fmul_rn(scale, cj));
    s_T[c] = T;
    if (theta_out) theta_out[(size_t)i * N + c] = T;
  }
  __syncthreads();
  qr_core<R>(s_theta, s_T, s_l, s_g, N, kappa, __fdiv_rn(__ldg(weights + i), (float)B), i, loss);
  float* gq = grad + row0 * N;
  for (int idx = tid; idx < A * N; idx += QR_T) {
    const int a = idx / N;
    gq[idx] = (a == act) ? s_g[idx - a * N] : 0.0f;
  }
}

// ---- CQL(H)'s regulariser (Kumar et al. 2020; DESIGN.md §22) ----
// For copy j of sample i (row jB + i of the online net's rows of s) and its values Q_a -- the expected value over the
// support with c51_expected_value's arithmetic (categorical head), or the mean quantile with qr_row_mean's (support NULL)
// -- R = logsumexp_a Q_a - Q_act = -l_act of munchausen_policy at temperature 1, whose pi is softmax_a Q.  With
// c = fl32(fl32(alpha w_i) / (M B)) and c_a = fl32(c (pi_a - [a == act])) the gradient on the logits of action a is
//   categorical  g_ak = fl32(c_a fl32(p_ak fl32(z_k - Q_a))),  p_ak = softmax(q_a)_k;    quantile  g_ak = fl32(c_a / N),
// ADDED onto the incoming gradient (through dueling_dz_rows_add on the fused head).  One CTA per sample walks its M rows
// in j order (one CTA per row at M = 1):
//   phase 0  (fused head) all threads stage the z row;
//   phase 1  warp a forms action a's logits, Q_a and, categorical, p_ak (z_k - Q_a) into s_g;
//   phase 2  thread 0 forms pi and R (munchausen_policy) and adds R to the gap in j order;
//   phase 3  all threads scale s_g into g; phase 4 the gradient row += g.
// gap_out[i] = fl32(sum_j R_ij / M).  No atomics: an eager launch and a graph replay agree bitwise.
constexpr int CQL_T = 256;
constexpr int CQL_WARPS = CQL_T / 32;

template <int R, bool QUANTILE, bool DUELING>
__device__ __forceinline__ void cql_sample(const float* __restrict__ rows, const int64_t* __restrict__ actions,
                                           const float* __restrict__ weights, const float* __restrict__ support,
                                           float alpha, int M, int B, int A, int Z, float* __restrict__ grad,
                                           float* __restrict__ gap_out) {
  extern __shared__ __align__(16) float s_dyn[];
  const int N2 = DUELING ? Z + A * Z : A * Z;   // floats per row
  float* zs = s_dyn;                            // [N2] the staged z row (fused head)
  float* s_g = zs + (DUELING ? N2 : 0);         // [A][Z] logits (fused head), then dQ_a / dq_ak, then g
  float* s_gv = s_g + A * Z;                    // [Z] dueling_dz_rows_add's scratch (fused head)
  float* s_q = s_gv + (DUELING ? Z : 0);        // [A] Q_a
  float* s_pi = s_q + A;                        // [A] softmax_a Q
  const int i = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int act = (int)actions[i];
  const float c = __fdiv_rn(__fmul_rn(alpha, __ldg(weights + i)), (float)(M * B));
  float sup[R];
#pragma unroll
  for (int r = 0; r < R; ++r) sup[r] = (!QUANTILE && lane + 32 * r < Z) ? __ldg(support + lane + 32 * r) : 0.0f;
  float gap = 0.0f;
  for (int j = 0; j < M; ++j) {
    const size_t row = (size_t)j * B + i;
    const float* src = rows + row * N2;
    if constexpr (DUELING) {  // phase 0: the one row (M = 1, K = 0) of copy j through the shared stager
      stage_z_rows<CQL_T>(zs, rows + (size_t)j * B * N2, rows, i, B, N2, 1, 0);
      __syncthreads();
    }
    {  // phase 1
      float mean[R];
#pragma unroll
      for (int r = 0; r < R; ++r) mean[r] = (DUELING && lane + 32 * r < Z) ? dueling_mean(zs, A, Z, lane + 32 * r) : 0.0f;
      for (int a = warp; a < A; a += CQL_WARPS) {
        float* ga = s_g + (size_t)a * Z;
        const float* qa = DUELING ? ga : src + (size_t)a * Z;
        if constexpr (DUELING) {
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const int k = lane + 32 * r;
            if (k < Z) ga[k] = dueling_q(zs[k], zs[Z + a * Z + k], mean[r]);
          }
          __syncwarp();
        }
        float q;
        if constexpr (QUANTILE) {
          float x[R];
#pragma unroll
          for (int r = 0; r < R; ++r) x[r] = (lane + 32 * r < Z) ? qa[lane + 32 * r] : 0.0f;
          q = qr_row_mean<R>(x, Z);
        } else {
          float e[R], x[R], mx, sum;
          softmax_row(qa, Z, lane, e, x, mx, sum);
          q = c51_expected_value<R>(x, sup, Z, lane);
#pragma unroll
          for (int r = 0; r < R; ++r)
            if (lane + 32 * r < Z) ga[lane + 32 * r] = __fmul_rn(__fdiv_rn(e[r], sum), __fsub_rn(sup[r], q));
        }
        if (lane == 0) s_q[a] = q;
      }
    }
    __syncthreads();
    if (tid == 0) {  // phase 2
      const float Rj = __fsub_rn(0.0f, munchausen_policy(s_q, A, 1.0f, s_pi, nullptr, act));
      gap = j == 0 ? Rj : __fadd_rn(gap, Rj);
    }
    __syncthreads();
#pragma unroll 1
    for (int a = tid; a < A; a += CQL_T) {  // phase 3: c_a (quantile: c_a / N) over s_q, then g
      const float ca = __fmul_rn(c, __fsub_rn(s_pi[a], a == act ? 1.0f : 0.0f));
      s_q[a] = QUANTILE ? __fdiv_rn(ca, (float)Z) : ca;
    }
    __syncthreads();
    for (int idx = tid; idx < A * Z; idx += CQL_T) {
      const float ca = s_q[idx / Z];
      s_g[idx] = QUANTILE ? ca : __fmul_rn(ca, s_g[idx]);
    }
    __syncthreads();
    float* gi = grad + row * N2;  // phase 4
    if constexpr (DUELING) {
      dueling_dz_rows_add<CQL_T>(gi, s_g, s_gv, A, Z);
    } else {
      for (int idx = tid; idx < A * Z; idx += CQL_T) gi[idx] = __fadd_rn(gi[idx], s_g[idx]);
    }
    __syncthreads();  // before the next row rewrites zs, s_g and s_gv
  }
  if (gap_out && tid == 0) gap_out[i] = __fdiv_rn(gap, (float)M);
}

// Fused-head entry: z_on rows [Z + A Z] as k_c51_dueling takes them (copy j of s at row jB + i); dz [M B][Z + A Z].
template <int R, bool QUANTILE>
__global__ void __launch_bounds__(CQL_T)
k_cql_dueling(const float* __restrict__ z_on, const int64_t* __restrict__ actions, const float* __restrict__ weights,
              const float* __restrict__ support, float alpha, int M, int B, int A, int Z, float* __restrict__ dz,
              float* __restrict__ gap_out) {
  cql_sample<R, QUANTILE, true>(z_on, actions, weights, support, alpha, M, B, A, Z, dz, gap_out);
}

// Library-head entry: logit rows [M B][A][Z] in k_c51's layout; grad [M B][A][Z].
template <int R, bool QUANTILE>
__global__ void __launch_bounds__(CQL_T)
k_cql(const float* __restrict__ q_on_s, const int64_t* __restrict__ actions, const float* __restrict__ weights,
      const float* __restrict__ support, float alpha, int M, int B, int A, int Z, float* __restrict__ grad,
      float* __restrict__ gap_out) {
  cql_sample<R, QUANTILE, false>(q_on_s, actions, weights, support, alpha, M, B, A, Z, grad, gap_out);
}

// Greedy values for acting / evaluation under quantiles: k_q_select with the mean over quantiles in place of
// softmax . support.  One warp per state; the dueling combination and the mean are k_qr_dueling's phase 1, bitwise.
// VT: the mean of h^-1 of the quantiles (return units).
// RISK: qr_risk_value in place of the mean (risk_kind / risk_eta are read only there).
template <bool VT, bool RISK>
__global__ void __launch_bounds__(128)
k_qr_select(const float* __restrict__ z, int M, int A, int N, float* __restrict__ q_out,
            int64_t* __restrict__ best_action, float* __restrict__ best_q, float eps, int risk_kind, float risk_eta) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * 4 + warp;
  if (m >= M) return;
  const float* zr = z + (size_t)m * (N + A * N);
  constexpr int R = RB_MAX_ATOMS / 32;
  float zv[R], mean[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int c = lane + 32 * r;
    zv[r] = mean[r] = 0.0f;
    if (c < N) {
      zv[r] = __ldg(zr + c);
      mean[r] = dueling_mean<true>(zr, A, N, c);
    }
  }
  int best = 0;
  float best_v = -CUDART_INF_F;
  float w[R];
  if constexpr (RISK) qr_risk_weights<R>(N, lane, risk_kind, risk_eta, w);
  for (int a = 0; a < A; ++a) {
    float x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      x[r] = (c < N) ? dueling_q(zv[r], __ldg(zr + N + a * N + c), mean[r]) : 0.0f;
      if constexpr (VT) x[r] = (c < N) ? vt_hinv(x[r], eps) : 0.0f;
    }
    float q;
    if constexpr (RISK) q = qr_risk_value<R>(x, w, N, lane);
    else q = qr_row_mean<R>(x, N);
    if (q_out && lane == 0) q_out[(size_t)m * A + a] = q;
    if (q > best_v) {   // first maximum wins, like torch.argmax / max
      best_v = q;
      best = a;
    }
  }
  if (lane == 0) {
    if (best_action) best_action[m] = best;
    if (best_q) best_q[m] = best_v;
  }
}

// ================================================================================================
// Learner statistics (agent.py:66-98 computes most of them and discards them): one record per update into a device ring.
// ================================================================================================
// Two launches, so that only a one-thread kernel has to wait for the optimiser step:
//   k_learn_stats_batch   everything that needs only the loss kernel's outputs.  Warp g of the grid takes the samples g,
//                         g + warps, ... (lane owns atoms lane + 32 r): q(s, a) of the taken action with the arithmetic of
//                         c51_expected_value, sum m * support as a warp sum, the end-atom mass, the loss / weight terms.
//                         Sums are float64: each warp in sample order, each CTA over its warps in order into its partial
//                         slot of the scratch; the last CTA to finish (self-resetting ticket) reduces the partials in CTA
//                         order (fixed xor butterflies, then the warps in order) and leaves the seven finished fields in
//                         the scratch.  Which CTA is last does not change the order: eager launches and graph replays agree
//                         bitwise.
//   k_learn_stats_record  after the optimiser step: those fields, the norm, clip coefficient and gate into slot
//                         *counter % capacity; advances *counter.
// Scratch (double, zero-initialised once): [0, 7) the finished fields, [8, 8 + 8 * STATS_MAX_CTAS) the per-CTA partials,
// then the ticket word.
constexpr int STATS_THREADS = 256;
constexpr int STATS_WARPS = STATS_THREADS / 32;
constexpr int STATS_MAX_CTAS = 256;                 // = STATS_THREADS: the last CTA reduces one partial per thread
constexpr int STATS_PART = 8;
constexpr int STATS_SCRATCH = STATS_PART + STATS_PART * STATS_MAX_CTAS + 1;

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double warp_max_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ double warp_min_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// per-warp values of the 7 accumulators -> s_part[k][warp] (lane 0); k: loss, w * loss, q(s, a), sum m * support, edge
// mass (sums), loss max, weight min
__device__ __forceinline__ void stats_store(double (&s_part)[7][STATS_WARPS], const double (&v)[7], int warp, int lane) {
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 7; ++k) s_part[k][warp] = v[k];
  }
}

__device__ __forceinline__ void stats_combine(const double (&s_part)[7][STATS_WARPS], double (&t)[7]) {
  t[0] = t[1] = t[2] = t[3] = t[4] = 0.0;
  t[5] = -CUDART_INF;
  t[6] = CUDART_INF;
  for (int w = 0; w < STATS_WARPS; ++w) {
#pragma unroll
    for (int k = 0; k < 5; ++k) t[k] += s_part[k][w];
    t[5] = fmax(t[5], s_part[5][w]);
    t[6] = fmin(t[6], s_part[6][w]);
  }
}

// The CTA's accumulators v -> its partial slot; the last CTA reduces the partials in CTA order into scratch[0, 7).
// no_edge: scratch[4] (edge_mass) is NaN.
__device__ __forceinline__ void stats_finish(double (&s_part)[7][STATS_WARPS], bool& s_last, const double (&v)[7], int B,
                                             double* __restrict__ scratch, bool no_edge) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  stats_store(s_part, v, warp, lane);
  __syncthreads();
  unsigned int* ticket = reinterpret_cast<unsigned int*>(scratch + STATS_SCRATCH - 1);
  if (tid == 0) {
    double t[7];
    stats_combine(s_part, t);
    double* part = scratch + STATS_PART + STATS_PART * blockIdx.x;
#pragma unroll
    for (int k = 0; k < 7; ++k) part[k] = t[k];
    __threadfence();
    s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double p[7] = {0.0, 0.0, 0.0, 0.0, 0.0, -CUDART_INF, CUDART_INF};
  if (tid < (int)gridDim.x) {
    const double* part = scratch + STATS_PART + STATS_PART * tid;
#pragma unroll
    for (int k = 0; k < 7; ++k) p[k] = __ldcg(part + k);
  }
#pragma unroll
  for (int k = 0; k < 5; ++k) p[k] = warp_sum_f64(p[k]);
  p[5] = warp_max_f64(p[5]);
  p[6] = warp_min_f64(p[6]);
  stats_store(s_part, p, warp, lane);
  __syncthreads();
  if (tid == 0) {
    double t[7];
    stats_combine(s_part, t);
#pragma unroll
    for (int k = 0; k < 5; ++k) scratch[k] = (double)(float)(t[k] / B);   // loss_mean, objective, q_mean, target_mean, edge_mass
    if (no_edge) scratch[4] = CUDART_NAN;
    scratch[5] = t[5];                                                    // loss_max
    scratch[6] = t[6];                                                    // weight_min
    *ticket = 0u;
  }
}

__global__ void __launch_bounds__(STATS_THREADS)
k_learn_stats_batch(const float* __restrict__ loss, const float* __restrict__ weights, const int64_t* __restrict__ actions,
                    const float* __restrict__ m, const float* __restrict__ support, const float* __restrict__ z,
                    const float* __restrict__ q, int B, int A, int Z, double* __restrict__ scratch) {
  __shared__ double s_part[7][STATS_WARPS];
  __shared__ bool s_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int R = RB_MAX_ATOMS / 32;
  float sup[R];
#pragma unroll
  for (int r = 0; r < R; ++r) sup[r] = (lane + 32 * r < Z) ? __ldg(support + lane + 32 * r) : 0.0f;
  double v[7] = {0.0, 0.0, 0.0, 0.0, 0.0, -CUDART_INF, CUDART_INF};
  const int warps = gridDim.x * STATS_WARPS;
  for (int i = blockIdx.x * STATS_WARPS + warp; i < B; i += warps) {
    const int act = (int)actions[i];
    const float* mr = m + (size_t)i * Z;
    const float l = __ldg(loss + i), w = __ldg(weights + i);
    float tv = 0.0f;
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (lane + 32 * r < Z) tv = __fadd_rn(tv, __fmul_rn(__ldg(mr + lane + 32 * r), sup[r]));
    const float edge = __fadd_rn(__ldg(mr), __ldg(mr + Z - 1));
    float x[R];
    if (z) {
      const float* zr = z + (size_t)i * (Z + A * Z);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int c = lane + 32 * r;
        x[r] = -CUDART_INF_F;
        if (c < Z) x[r] = dueling_q<true>(zr, A, Z, c, act);
      }
    } else {
      const float* qr = q + ((size_t)i * A + act) * Z;
#pragma unroll
      for (int r = 0; r < R; ++r) x[r] = (lane + 32 * r < Z) ? __ldg(qr + lane + 32 * r) : -CUDART_INF_F;
    }
    const float ev = c51_expected_value<R>(x, sup, Z, lane);
    tv = warp_sum(tv);   // the butterflies leave the same value in every lane
    v[0] += (double)l;
    v[1] += (double)w * (double)l;   // exact product
    v[2] += (double)ev;
    v[3] += (double)tv;
    v[4] += (double)edge;
    v[5] = fmax(v[5], (double)l);
    v[6] = fmin(v[6], (double)w);
  }
  stats_finish(s_part, s_last, v, B, scratch, false);
}

// k_learn_stats_batch for the quantile loss: theta = the T rows [B][N] of the loss kernel (theta_out); per sample
// q(s, a) = mean_i theta_i of the online quantiles of the taken action (dueling_q from z, or the row of q) and
// the target value mean_j T_j; edge_mass is NaN (there is no support to clamp to).  VT: both means are of h^-1 of the
// quantiles (return units).
template <bool VT>
__global__ void __launch_bounds__(STATS_THREADS)
k_learn_stats_batch_qr(const float* __restrict__ loss, const float* __restrict__ weights, const int64_t* __restrict__ actions,
                       const float* __restrict__ theta, const float* __restrict__ z, const float* __restrict__ q, int B, int A,
                       int N, double* __restrict__ scratch, float eps) {
  __shared__ double s_part[7][STATS_WARPS];
  __shared__ bool s_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int R = RB_MAX_ATOMS / 32;
  double v[7] = {0.0, 0.0, 0.0, 0.0, 0.0, -CUDART_INF, CUDART_INF};
  const int warps = gridDim.x * STATS_WARPS;
  for (int i = blockIdx.x * STATS_WARPS + warp; i < B; i += warps) {
    const int act = (int)actions[i];
    const float* tr = theta + (size_t)i * N;
    const float l = __ldg(loss + i), w = __ldg(weights + i);
    float t[R], x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int c = lane + 32 * r;
      t[r] = (c < N) ? __ldg(tr + c) : 0.0f;
      x[r] = 0.0f;
      if (c < N) {
        x[r] = z ? dueling_q<true>(z + (size_t)i * (N + A * N), A, N, c, act) : __ldg(q + ((size_t)i * A + act) * N + c);
        if constexpr (VT) {
          t[r] = vt_hinv(t[r], eps);
          x[r] = vt_hinv(x[r], eps);
        }
      }
    }
    const float qv = qr_row_mean<R>(x, N), tv = qr_row_mean<R>(t, N);
    v[0] += (double)l;
    v[1] += (double)w * (double)l;
    v[2] += (double)qv;
    v[3] += (double)tv;
    v[5] = fmax(v[5], (double)l);
    v[6] = fmin(v[6], (double)w);
  }
  stats_finish(s_part, s_last, v, B, scratch, true);
}

__global__ void k_learn_stats_record(const double* __restrict__ scratch, const float* __restrict__ grad_norm,
                                     const int32_t* __restrict__ gate, float max_norm, rb_learn_stats_record* __restrict__ ring,
                                     int capacity, int64_t* __restrict__ counter) {
  const float norm = *grad_norm;
  rb_learn_stats_record rec;
  rec.update = *counter;
  rec.loss_mean = (float)scratch[0];
  rec.loss_max = (float)scratch[5];
  rec.objective = (float)scratch[1];
  rec.q_mean = (float)scratch[2];
  rec.target_mean = (float)scratch[3];
  rec.edge_mass = (float)scratch[4];
  rec.weight_min = (float)scratch[6];
  rec.grad_norm = norm;
  rec.clip_coef = fminf(max_norm / (norm + 1e-6f), 1.0f);   // as k_clip_adam / k_peer_adam
  rec.applied = (gate && *gate == 0) ? 0.0f : 1.0f;
  ring[rec.update % capacity] = rec;
  *counter = rec.update + 1;
}

// ================================================================================================
// K6  noisy_resample : factorised Gaussian noise for every NoisyLinear of one net, one launch.
// ================================================================================================
struct NoisyPlan {
  float* w[RB_MAX_NOISY_LAYERS];
  float* b[RB_MAX_NOISY_LAYERS];
  int in_f[RB_MAX_NOISY_LAYERS];
  int out_f[RB_MAX_NOISY_LAYERS];
  int in_off[RB_MAX_NOISY_LAYERS];   // offset of the layer's eps_in in the concatenated normal stream
  int out_off[RB_MAX_NOISY_LAYERS];
  int rows_per_cta[RB_MAX_NOISY_LAYERS];
  int cta_begin[RB_MAX_NOISY_LAYERS + 1];
  int n;
};

constexpr int NOISY_THREADS = 256;

__global__ void __launch_bounds__(NOISY_THREADS)
k_noisy_resample(const __grid_constant__ NoisyPlan plan, const float* __restrict__ x_in, const float* __restrict__ x_out,
                 uint64_t seed, unsigned long long* rng_counter, int prescaled) {
  extern __shared__ __align__(16) float s_in[];  // f(eps_in) of this CTA's layer
  int l = 0;
  while (l + 1 < plan.n && (int)blockIdx.x >= plan.cta_begin[l + 1]) ++l;
  const int in_f = plan.in_f[l], out_f = plan.out_f[l];
  const int tile = blockIdx.x - plan.cta_begin[l];
  const int r0 = tile * plan.rows_per_cta[l], r1 = min(out_f, r0 + plan.rows_per_cta[l]);
  const unsigned long long ctr = rng_counter ? *rng_counter : 0ull;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (x_in) {
    for (int i = tid; i < in_f; i += NOISY_THREADS) {
      const float v = __ldg(x_in + plan.in_off[l] + i);
      s_in[i] = prescaled ? v : scale_noise(v);
    }
  } else {
    // global normal index g = in_off + i ; Philox block g/4 yields normals 4*(g/4) .. +3
    const int g0 = plan.in_off[l], g1 = g0 + in_f;
    for (int blk = g0 / 4 + tid; blk * 4 < g1; blk += NOISY_THREADS) {
      float4 z = normal4(seed, ctr, 0u, (uint32_t)blk);
      float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int g = blk * 4 + q;
        if (g >= g0 && g < g1) s_in[g - g0] = scale_noise(zz[q]);
      }
    }
  }
  __syncthreads();

  float* w = plan.w[l];
  float* bias = plan.b[l];
  const bool vec = (in_f % 4 == 0) && ((reinterpret_cast<uintptr_t>(w) & 15) == 0);
  for (int o = r0 + warp; o < r1; o += NOISY_THREADS / 32) {
    float xo;
    if (x_out) {
      xo = __ldg(x_out + plan.out_off[l] + o);
    } else {
      int g = plan.out_off[l] + o;
      float4 z = normal4(seed, ctr, 1u, (uint32_t)(g >> 2));
      int q = g & 3;
      xo = q == 0 ? z.x : (q == 1 ? z.y : (q == 2 ? z.z : z.w));
    }
    const float eo = (x_out && prescaled) ? xo : scale_noise(xo);
    if (lane == 0) bias[o] = eo;                       // model.py:40
    float* row = w + (size_t)o * in_f;                 // model.py:39 eps_out (outer) eps_in
    if (vec) {
      float4* row4 = reinterpret_cast<float4*>(row);
      const float4* in4 = reinterpret_cast<const float4*>(s_in);
      for (int c = lane; c < in_f / 4; c += 32) {
        float4 e = in4[c];
        __stcs(row4 + c, make_float4(__fmul_rn(eo, e.x), __fmul_rn(eo, e.y), __fmul_rn(eo, e.z), __fmul_rn(eo, e.w)));
      }
    } else {
      for (int c = lane; c < in_f; c += 32) row[c] = __fmul_rn(eo, s_in[c]);
    }
  }
}

// counter bump runs as its own tiny kernel after the resample grid (all CTAs must read the old value)
__global__ void k_bump_counter(unsigned long long* ctr) { *ctr += 1ull; }

// model.py:43-44: W = mu + sigma * eps
__global__ void __launch_bounds__(256)
k_noisy_compose(const float* __restrict__ mu, const float* __restrict__ sigma, const float* __restrict__ eps,
                int64_t count, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if ((count & 3) == 0 && (((uintptr_t)mu | (uintptr_t)sigma | (uintptr_t)eps | (uintptr_t)out) & 15) == 0) {
    const int64_t n4 = count >> 2;
    for (; i < n4; i += stride) {
      float4 m = __ldg(reinterpret_cast<const float4*>(mu) + i), s = __ldg(reinterpret_cast<const float4*>(sigma) + i),
             e = __ldg(reinterpret_cast<const float4*>(eps) + i);
      reinterpret_cast<float4*>(out)[i] =
          make_float4(__fadd_rn(m.x, __fmul_rn(s.x, e.x)), __fadd_rn(m.y, __fmul_rn(s.y, e.y)),
                      __fadd_rn(m.z, __fmul_rn(s.z, e.z)), __fadd_rn(m.w, __fmul_rn(s.w, e.w)));
    }
  } else {
    for (; i < count; i += stride) out[i] = __fadd_rn(mu[i], __fmul_rn(sigma[i], eps[i]));
  }
}

// ================================================================================================
// K7  clip_adam : global-norm clip + Adam on flat buffers (agent.py:97-98), two launches.
// ================================================================================================
constexpr int ADAM_THREADS = 256;
constexpr int ADAM_MAX_CTAS = rbi::SM_COUNT * 8;

__global__ void __launch_bounds__(ADAM_THREADS)
k_sqnorm(const float* __restrict__ grad, int64_t P, float grad_scale, double* __restrict__ partial) {
  __shared__ double s_red[ADAM_THREADS / 32];
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if ((P & 3) == 0 && ((uintptr_t)grad & 15) == 0) {
    for (; i < (P >> 2); i += stride) {
      float4 g = __ldg(reinterpret_cast<const float4*>(grad) + i);
      float a = g.x * grad_scale, b = g.y * grad_scale, c = g.z * grad_scale, d = g.w * grad_scale;
      acc += (double)a * a + (double)b * b + (double)c * c + (double)d * d;
    }
  } else {
    for (; i < P; i += stride) {
      float a = grad[i] * grad_scale;
      acc += (double)a * a;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < ADAM_THREADS / 32; ++w) t += s_red[w];
    partial[blockIdx.x] = t;
  }
}

// sqrt / reciprocal through the SFU approximations (<= 2 ulp): the kernel was partly instruction bound on the
// IEEE div/sqrt sequences (r01 ncu: SM throughput 55 %), and the update tolerates 1e-6 relative error.
__device__ __forceinline__ float fast_sqrt(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float r;
  asm("rcp.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float coef, float b1, float b2,
                                         float step_size, float inv_bc2_sqrt, float eps) {
  g = g * coef;
  m = fmaf(g - m, 1.0f - b1, m);                 // exp_avg.lerp_(grad, 1 - beta1)
  v = fmaf(v, b2, (1.0f - b2) * g * g);          // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
  const float denom = fmaf(fast_sqrt(v), inv_bc2_sqrt, eps);
  p = fmaf(-step_size * m, fast_rcp(denom), p);  // param.addcdiv_(exp_avg, denom, value=-step_size)
}

// rb_clip_adamw's group table, by value: groups tile [0, P) in order, each begins on a multiple of 4
struct AdamGroupPlan {
  rb_adam_group g[RB_MAX_ADAM_GROUPS];
  int n;
};

// rb_clip_adamw: the body below takes one step size, 1 / sqrt(bc2) and count from step_count when GROUPS is false, and per
// group g -- bias corrections from group_steps[g] + 1, decay factor d_g = fl32(1 - lr lambda_g) applied as p = p * d_g
// (rounded on its own, never contracted) before adam_one -- when it is true.  The factors are formed once per CTA into
// shared memory; a float4 finds its group with three compares against the later groups' begins (a begin is a multiple of 4,
// so no float4 straddles two groups).  d_g = 1 for lambda_g = 0 leaves p bitwise as it is.
template <bool GROUPS>
__device__ __forceinline__ void
clip_adam_body(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ exp_avg,
               float* __restrict__ exp_avg_sq, int64_t P, float grad_scale, float max_norm, float lr, float b1, float b2,
               float eps, int64_t* __restrict__ step_count, const double* __restrict__ partial, int n_partial,
               float* __restrict__ norm_out, unsigned int* __restrict__ done_ticket, const int32_t* __restrict__ gate,
               const AdamGroupPlan* plan, int64_t* __restrict__ group_steps) {
  const bool skip = gate && *gate == 0;   // rejected sample batch: no parameter update, no step (see k_tree_sample)
  __shared__ double s_red[ADAM_THREADS / 32];
  __shared__ float s_coef;
  __shared__ float s_step_size[GROUPS ? RB_MAX_ADAM_GROUPS : 1], s_bc2_sqrt[GROUPS ? RB_MAX_ADAM_GROUPS : 1],
      s_decay[GROUPS ? RB_MAX_ADAM_GROUPS : 1];
  __shared__ int64_t s_t[GROUPS ? RB_MAX_ADAM_GROUPS : 1];
  if constexpr (GROUPS) {
    if (threadIdx.x < plan->n) {
      const int k = threadIdx.x;
      const int64_t t = group_steps[k] + 1;
      const double bc1 = 1.0 - pow((double)b1, (double)t);
      const double bc2 = 1.0 - pow((double)b2, (double)t);
      s_step_size[k] = (float)((double)lr / bc1);
      s_bc2_sqrt[k] = (float)(1.0 / sqrt(bc2));
      s_decay[k] = (float)(1.0 - (double)lr * (double)plan->g[k].weight_decay);
      s_t[k] = t;
    }
  }
  // every CTA re-reduces the (few hundred) partial sums in the same order: deterministic, no atomics
  double acc = 0.0;
  for (int i = threadIdx.x; i < n_partial; i += ADAM_THREADS) acc += partial[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < ADAM_THREADS / 32; ++w) t += s_red[w];
    float norm = (float)sqrt(t);
    float c = max_norm / (norm + 1e-6f);         // torch clip_grad_norm_
    s_coef = fminf(c, 1.0f) * grad_scale;
    if (norm_out && blockIdx.x == 0) *norm_out = norm;
  }
  __syncthreads();
  const float coef = s_coef;
  const int64_t step = *step_count + 1;
  float step_size, bc2_sqrt;  // bc2_sqrt is passed to adam_one as the reciprocal
  int64_t lim1 = INT64_MAX, lim2 = INT64_MAX, lim3 = INT64_MAX;   // begins of groups 1..3 (none: never reached)
  if constexpr (GROUPS) {
    if (plan->n > 1) lim1 = plan->g[1].begin;
    if (plan->n > 2) lim2 = plan->g[2].begin;
    if (plan->n > 3) lim3 = plan->g[3].begin;
  } else {
    const double bc1 = 1.0 - pow((double)b1, (double)step);
    const double bc2 = 1.0 - pow((double)b2, (double)step);
    step_size = (float)((double)lr / bc1);
    bc2_sqrt = (float)(1.0 / sqrt(bc2));
  }

  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool vec = (P & 3) == 0 && (((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0;
  if (skip) {
  } else if (vec) {
    for (; i < (P >> 2); i += stride) {
      float4 p = reinterpret_cast<float4*>(param)[i], g = __ldg(reinterpret_cast<const float4*>(grad) + i),
             m = reinterpret_cast<float4*>(exp_avg)[i], v = reinterpret_cast<float4*>(exp_avg_sq)[i];
      if constexpr (GROUPS) {
        const int64_t e = i << 2;
        const int k = (e >= lim1) + (e >= lim2) + (e >= lim3);
        step_size = s_step_size[k];
        bc2_sqrt = s_bc2_sqrt[k];
        const float d = s_decay[k];
        p.x = __fmul_rn(p.x, d); p.y = __fmul_rn(p.y, d); p.z = __fmul_rn(p.z, d); p.w = __fmul_rn(p.w, d);
      }
      adam_one(p.x, g.x, m.x, v.x, coef, b1, b2, step_size, bc2_sqrt, eps);
      adam_one(p.y, g.y, m.y, v.y, coef, b1, b2, step_size, bc2_sqrt, eps);
      adam_one(p.z, g.z, m.z, v.z, coef, b1, b2, step_size, bc2_sqrt, eps);
      adam_one(p.w, g.w, m.w, v.w, coef, b1, b2, step_size, bc2_sqrt, eps);
      reinterpret_cast<float4*>(param)[i] = p;
      reinterpret_cast<float4*>(exp_avg)[i] = m;
      reinterpret_cast<float4*>(exp_avg_sq)[i] = v;
    }
  } else {
    for (; i < P; i += stride) {
      float p = param[i], m = exp_avg[i], v = exp_avg_sq[i];
      if constexpr (GROUPS) {
        const int k = (i >= lim1) + (i >= lim2) + (i >= lim3);
        step_size = s_step_size[k];
        bc2_sqrt = s_bc2_sqrt[k];
        p = __fmul_rn(p, s_decay[k]);
      }
      adam_one(p, grad[i], m, v, coef, b1, b2, step_size, bc2_sqrt, eps);
      param[i] = p;
      exp_avg[i] = m;
      exp_avg_sq[i] = v;
    }
  }
  // every CTA has read *step_count (and the group counts) above; the last one to get here advances them (self-resetting
  // ticket), which saves a dependent 1-thread launch on the critical path
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int t = atomicAdd(done_ticket, 1u);
    if (t == gridDim.x - 1) {
      *done_ticket = 0u;
      if (!skip) {
        *step_count = step;
        if constexpr (GROUPS) {
          for (int k = 0; k < plan->n; ++k) group_steps[k] = s_t[k];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(ADAM_THREADS)
k_clip_adam(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ exp_avg,
            float* __restrict__ exp_avg_sq, int64_t P, float grad_scale, float max_norm, float lr, float b1, float b2,
            float eps, int64_t* __restrict__ step_count, const double* __restrict__ partial, int n_partial,
            float* __restrict__ norm_out, unsigned int* __restrict__ done_ticket, const int32_t* __restrict__ gate) {
  clip_adam_body<false>(param, grad, exp_avg, exp_avg_sq, P, grad_scale, max_norm, lr, b1, b2, eps, step_count, partial,
                        n_partial, norm_out, done_ticket, gate, nullptr, nullptr);
}

__global__ void __launch_bounds__(ADAM_THREADS)
k_clip_adamw(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ exp_avg,
             float* __restrict__ exp_avg_sq, int64_t P, float grad_scale, float max_norm, float lr, float b1, float b2,
             float eps, int64_t* __restrict__ step_count, const double* __restrict__ partial, int n_partial,
             float* __restrict__ norm_out, unsigned int* __restrict__ done_ticket, const int32_t* __restrict__ gate,
             const __grid_constant__ AdamGroupPlan plan, int64_t* __restrict__ group_steps) {
  clip_adam_body<true>(param, grad, exp_avg, exp_avg_sq, P, grad_scale, max_norm, lr, b1, b2, eps, step_count, partial,
                       n_partial, norm_out, done_ticket, gate, &plan, group_steps);
}

int adam_ctas(int64_t P) {
  int64_t want = (P / 4 + ADAM_THREADS - 1) / ADAM_THREADS;
  if (want < 1) want = 1;
  if (want > ADAM_MAX_CTAS) want = ADAM_MAX_CTAS;
  return (int)want;
}

// ================================================================================================
// K8  target_ema : Polyak target update t = fma(tau, p, fl32(1 - tau) * t) on the flat buffers, after clip + Adam.
// ================================================================================================
// Same grid-stride shape as k_clip_adam: float4 when both pointers are 16-byte aligned (plus a scalar tail for n % 4),
// scalar otherwise.  A gate reading 0 (rejected batch) returns before anything is read or written.
__device__ __forceinline__ float ema_one(float t, float p, float tau, float keep) {
  return __fmaf_rn(tau, p, __fmul_rn(keep, t));
}

__global__ void __launch_bounds__(ADAM_THREADS)
k_target_ema(float* __restrict__ target, const float* __restrict__ param, int64_t n, float tau,
             const int32_t* __restrict__ gate) {
  if (gate && *gate == 0) return;
  const float keep = __fsub_rn(1.0f, tau);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if ((((uintptr_t)target | (uintptr_t)param) & 15) == 0) {
    const int64_t n4 = n >> 2;
    for (int64_t i = i0; i < n4; i += stride) {
      float4 t = reinterpret_cast<float4*>(target)[i];
      const float4 p = __ldg(reinterpret_cast<const float4*>(param) + i);
      t = make_float4(ema_one(t.x, p.x, tau, keep), ema_one(t.y, p.y, tau, keep), ema_one(t.z, p.z, tau, keep),
                      ema_one(t.w, p.w, tau, keep));
      reinterpret_cast<float4*>(target)[i] = t;
    }
    const int64_t j = (n4 << 2) + i0;       // the n % 4 elements past the last full float4
    if (j < n) target[j] = ema_one(target[j], param[j], tau, keep);
  } else {
    for (int64_t i = i0; i < n; i += stride) target[i] = ema_one(target[i], param[i], tau, keep);
  }
}

// ================================================================================================
// K9  param_reset : shrink-and-perturb of segments of the flat parameter buffer, theta0 drawn from Philox.
// ================================================================================================
// Grid (x: quads of 4 elements, grid-stride; y: segment).  One Philox4x32-10 call per aligned quad j >> 2 gives the words of
// its four elements; the elements of the quad outside the segment are skipped (padding between tensors is never written).
constexpr uint32_t RESET_STREAM = 0x52534554u;       // "RSET"
constexpr int RESET_THREADS = 256;

struct ResetPlan {
  rb_reset_segment seg[RB_MAX_RESET_SEGMENTS];
};

__global__ void __launch_bounds__(RESET_THREADS)
k_param_reset(float* __restrict__ param, const __grid_constant__ ResetPlan plan, uint64_t seed, uint64_t reset_index) {
  const rb_reset_segment& s = plan.seg[blockIdx.y];
  const int64_t lo = s.offset, hi = s.offset + s.count;
  const float alpha = s.alpha, keep = __fsub_rn(1.0f, s.alpha), bound = s.bound, constant = s.constant;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (lo >> 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; (q << 2) < hi; q += stride) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)reset_index, (uint32_t)(reset_index >> 32), (uint32_t)q, RESET_STREAM),
                                  key);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t j = (q << 2) + e;
      if (j < lo || j >= hi) continue;
      const float u = (float)(w[e] >> 8) * 0x1.0p-24f;
      const float theta0 = __fmaf_rn(bound, __fmaf_rn(2.0f, u, -1.0f), constant);
      param[j] = __fmaf_rn(alpha, param[j], __fmul_rn(keep, theta0));
    }
  }
}

// ================================================================================================
// K10  dormant-neuron scores, mask and ReDo recycling (Sokar et al. 2023) -- all decided and applied on the device.
// ================================================================================================
// k_neuron_scores: sums[c] = sum over (row, position) of act[r][c][p], one CTA per neuron.  Thread t takes the elements
// i = r HW + p with i % 256 == t, in increasing i: fp32 partial sums over chunks of REDO_CHUNK elements, each chunk added to a
// float64 accumulator; the 256 accumulators are summed by a fixed float64 tree in shared memory.  k_bias_grad computes the
// same sum in one CTA per channel too, but carries it in fp32 to the end (200 000 addends at batch 512): the float64 total
// keeps the error to that of one chunk, 63 * 2^-24 relative, whatever R is, and gives the ranks' all-reduce exact addends.
constexpr int REDO_THREADS = 256;
constexpr int REDO_CHUNK = 64;
constexpr int REDO_NEURON_CTAS = 8;                   // CTAs that share one dormant neuron's elements
constexpr uint32_t REDO_STREAM = 0x5245444Fu;        // "REDO": listed with the other stream words above INTS_STREAM

__global__ void __launch_bounds__(REDO_THREADS)
k_neuron_scores(const float* __restrict__ act, int R, int C, int HW, double* __restrict__ sums) {
  __shared__ double s_red[REDO_THREADS];
  const int c = blockIdx.x;
  const int64_t total = (int64_t)R * HW;
  double acc = 0.0;
  float part = 0.0f;
  int in_chunk = 0;
  for (int64_t i = threadIdx.x; i < total; i += REDO_THREADS) {
    const int64_t r = i / HW, p = i - r * HW;
    part = __fadd_rn(part, __ldg(act + (r * C + c) * HW + p));
    if (++in_chunk == REDO_CHUNK) { acc += (double)part; part = 0.0f; in_chunk = 0; }
  }
  acc += (double)part;
  s_red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = REDO_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) s_red[threadIdx.x] += s_red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[c] = s_red[0];
}

struct RedoMaskPlan {
  int32_t n_layers;
  int32_t offset[RB_MAX_REDO_LAYERS];      // first neuron of the layer in sums / mask
  int32_t neurons[RB_MAX_REDO_LAYERS];
  double count[RB_MAX_REDO_LAYERS];        // R HW: activations behind one sum
};

// One CTA per layer.  score s_i = sums[i] / count, mean over the layer summed in float64 in neuron order (thread 0), neuron
// i dormant iff s_i <= tau * mean.  record: int64 {pass index, n_layers, (neurons, dormant) per layer}.
__global__ void __launch_bounds__(REDO_THREADS)
k_redo_mask(const double* __restrict__ sums, const __grid_constant__ RedoMaskPlan plan, float tau, uint8_t* __restrict__ mask,
            long long* __restrict__ record, long long pass_index) {
  __shared__ double s_threshold;
  const int l = blockIdx.x, n = plan.neurons[l];
  const double* s = sums + plan.offset[l];
  uint8_t* m = mask + plan.offset[l];
  const double count = plan.count[l];
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < n; ++i) t += s[i] / count;
    s_threshold = (double)tau * (t / (double)n);
  }
  __syncthreads();
  const double threshold = s_threshold;
  int dormant = 0;
  for (int i0 = 0; i0 < n; i0 += REDO_THREADS) {
    const int i = i0 + threadIdx.x;
    const int d = (i < n) && (s[i] / count <= threshold);
    if (i < n) m[i] = (uint8_t)d;
    dormant += __syncthreads_count(d);
  }
  if (threadIdx.x == 0) {
    record[2 + 2 * l] = n;
    record[3 + 2 * l] = dormant;
    if (l == 0) { record[0] = pass_index; record[1] = plan.n_layers; }
  }
}

struct RedoPlan {
  rb_redo_layer layer[RB_MAX_REDO_LAYERS];
};

// Grid (x: chunk of the neuron's elements, y: neuron, z: layer); a CTA whose neuron is not dormant returns after one mask
// byte.  Incoming element j of a dormant neuron gets theta0(j) -- k_param_reset's formula with REDO_STREAM -- unless the
// upstream neuron it reads from is dormant too: that element is an outgoing element of the upstream neuron and the CTA that
// zeroes it is its only writer.  Every written element's moments become 0.
__global__ void __launch_bounds__(REDO_THREADS)
k_redo_recycle(float* __restrict__ param, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
               const __grid_constant__ RedoPlan plan, const uint8_t* __restrict__ mask, uint64_t seed, uint64_t pass_index) {
  const rb_redo_layer& L = plan.layer[blockIdx.z];
  const int i = blockIdx.y;
  if (i >= L.neurons || !mask[L.mask_offset + i]) return;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const int64_t first = (int64_t)blockIdx.x * REDO_THREADS + threadIdx.x, stride = (int64_t)gridDim.x * REDO_THREADS;
  for (int b = 0; b < L.n_in; ++b) {
    const rb_redo_in& in = L.in[b];
    const uint8_t* up = in.src_span > 0 ? mask + in.src_mask_offset : nullptr;
    for (int64_t e = first; e < in.per_neuron; e += stride) {
      if (up && up[e / in.src_span]) continue;
      const int64_t j = in.offset + (int64_t)i * in.per_neuron + e;
      const uint4 r = philox4x32_10(make_uint4((uint32_t)pass_index, (uint32_t)(pass_index >> 32), (uint32_t)(j >> 2),
                                               REDO_STREAM), key);
      const int q = (int)(j & 3);
      const uint32_t w = q == 0 ? r.x : q == 1 ? r.y : q == 2 ? r.z : r.w;
      const float u = (float)(w >> 8) * 0x1.0p-24f;
      param[j] = __fmaf_rn(in.bound, __fmaf_rn(2.0f, u, -1.0f), in.constant);
      exp_avg[j] = 0.0f;
      exp_avg_sq[j] = 0.0f;
    }
  }
  for (int b = 0; b < L.n_out; ++b) {
    const rb_redo_out& out = L.out[b];
    const int64_t total = out.rows * out.span;
    for (int64_t e = first; e < total; e += stride) {
      const int64_t r = e / out.span, p = e - r * out.span;
      const int64_t j = out.offset + r * out.row_stride + (int64_t)i * out.span + p;
      param[j] = 0.0f;
      exp_avg[j] = 0.0f;
      exp_avg_sq[j] = 0.0f;
    }
  }
}

// The launch of rb_append and rb_append_batch, after each has checked its own arguments.
int append_launch(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep, int32_t* action,
                  float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max, const AppendBatch& ab,
                  rb_stream_t stream, const char* who, bool final_records = false) {
  { ProfScope prof_(RB_K_APPEND, (cudaStream_t)stream);
    if (final_records)
      k_append_batch_final<<<ab.k, APPEND_THREADS, 0, (cudaStream_t)stream>>>(tree, tree_start, size, frames, timestep,
                                                                              action, reward, nonterminal, ring_state,
                                                                              running_max, ab);
    else
      k_append_batch<<<ab.k, APPEND_THREADS, 0, (cudaStream_t)stream>>>(tree, tree_start, size, frames, timestep, action,
                                                                        reward, nonterminal, ring_state, running_max, ab); }
  return check_launch(who);
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int rb_abi_version(void) { return RB_ABI_VERSION; }

int rb_profile_enable(int on) {
  rbi::g_prof_on = on != 0;
  return RB_OK;
}

int rb_profile_collect(int kernel_id, double* total_ms, int* launches) {
  if (kernel_id < 0 || kernel_id >= RB_KERNEL_COUNT || !total_ms || !launches) return fail(RB_ERR_INVAL, "rb_profile_collect: bad argument");
  ProfKernel* k = &rbi::g_prof[kernel_id];
  double t = 0.0;
  for (int i = 0; i < k->used; ++i) {
    float ms = 0.0f;
    cudaError_t e = cudaEventSynchronize(k->e1[i]);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, k->e0[i], k->e1[i]);
    if (e != cudaSuccess) return fail(RB_ERR_CUDA, cudaGetErrorString(e));
    t += ms;
  }
  *total_ms = t;
  *launches = k->used;
  k->used = 0;
  return RB_OK;
}

const char* rb_last_error(void) { return rbi::g_err; }

int rb_tree_update(float* tree, int64_t tree_start, int64_t size, const int64_t* tree_idx, const float* raw_priority,
                   float omega, int omega_is_applied, int B, float* running_max, int32_t* status, const int32_t* gate,
                   rb_stream_t stream) {
  if (!tree || !tree_idx || !raw_priority || !running_max) return fail(RB_ERR_INVAL, "rb_tree_update: null pointer");
  if (B <= 0 || size <= 0 || (size & 1)) return fail(RB_ERR_INVAL, "rb_tree_update: B > 0 and an even size are required");
  if (tree_start + size > ((int64_t)1 << 31)) return fail(RB_ERR_RANGE, "rb_tree_update: tree larger than 2^31 nodes");
  { ProfScope prof_(RB_K_TREE_UPDATE, (cudaStream_t)stream);
    if (B <= 32 && tree_depth(tree_start) <= 30)
      k_tree_update_warp<<<1, 32, 0, (cudaStream_t)stream>>>(tree, tree_start, size, tree_idx, raw_priority, omega,
                                                            omega_is_applied, B, running_max, status, gate);
    else
      k_tree_update<<<1, UPD_THREADS, 0, (cudaStream_t)stream>>>(tree, tree_start, size, tree_idx, raw_priority, omega,
                                                               omega_is_applied, B, running_max, status, gate); }
  return check_launch("rb_tree_update");
}

int rb_tree_find(const float* tree, int64_t tree_start, int64_t size, const double* values, int B, float* probs,
                 int64_t* data_idx, int64_t* tree_idx, rb_stream_t stream) {
  if (!tree || !values || !probs || !data_idx || !tree_idx) return fail(RB_ERR_INVAL, "rb_tree_find: null pointer");
  if (B <= 0 || size <= 0) return fail(RB_ERR_INVAL, "rb_tree_find: B and size must be positive");
  int ctas = (B + 31) / 32;
  if (ctas > rbi::SM_COUNT) ctas = rbi::SM_COUNT;
  { ProfScope prof_(RB_K_TREE_FIND, (cudaStream_t)stream);
    k_tree_find<<<ctas, SAMPLE_THREADS, 0, (cudaStream_t)stream>>>(tree, tree_start, size, values, B, probs, data_idx, tree_idx); }
  return check_launch("rb_tree_find");
}

int rb_tree_sample(const float* tree, int64_t tree_start, int64_t size, const int64_t* ring_state, int n, int history,
                   const double* u01, int u01_attempts, uint64_t seed, uint64_t* rng_counter, int B, float beta,
                   const float* beta_dev, int max_attempts, float* probs, int64_t* data_idx, int64_t* tree_idx,
                   float* weights, int32_t* status, rb_stream_t stream) {
  if (!tree || !ring_state || !probs || !data_idx || !tree_idx || !weights || !status)
    return fail(RB_ERR_INVAL, "rb_tree_sample: null pointer");
  if (B <= 0 || size <= 0 || (size & 1)) return fail(RB_ERR_INVAL, "rb_tree_sample: B > 0 and an even size are required");
  if (u01 == nullptr && rng_counter == nullptr) return fail(RB_ERR_INVAL, "rb_tree_sample: need u01 or rng_counter");
  if ((u01 != nullptr && u01_attempts <= 0) || (u01 == nullptr && max_attempts <= 0))
    return fail(RB_ERR_INVAL, "rb_tree_sample: attempts must be positive");
  { ProfScope prof_(RB_K_TREE_SAMPLE, (cudaStream_t)stream);
    k_tree_sample<<<1, SAMPLE_THREADS, 0, (cudaStream_t)stream>>>(
      tree, tree_start, size, ring_state, n, history, u01, u01_attempts, seed, (unsigned long long*)rng_counter, B, beta,
      beta_dev, max_attempts, probs, data_idx, tree_idx, weights, status); }
  return check_launch("rb_tree_sample");
}

// The grid of a gather over a window of history + n (the k_*_hz kernels take n = n_max and retire the slots the current
// n does not use): (used slots * split, B), each used slot split into `split` parts.
static dim3 gather_grid(int history, int n, int B, int* split) {
  const int used = (history + n < 2 * history) ? history + n : 2 * history;
  // aim for >= 4 CTAs per SM so small batches still cover the machine; a frame is 441 x 16 B
  *split = 1;
  while (*split < 2 && used * B * *split < rbi::SM_COUNT * 2) *split *= 2;  // 221 of 256 threads busy per CTA at split 2
  return dim3(used * *split, B);
}

// the argument checks every gather entry point shares
static int gather_check(const char* who, const uint8_t* frames, const int32_t* timestep, const int32_t* action,
                        const float* reward, const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B,
                        int history, int n, const float* gamma_pow, const float* states, const float* next_states,
                        const int64_t* actions, const float* returns, const float* nonterminals) {
  char what[96];
  if (!frames || !timestep || !action || !reward || !nonterminal || !data_idx || !gamma_pow || !states || !next_states ||
      !actions || !returns || !nonterminals) {
    snprintf(what, sizeof what, "%s: null pointer", who);
    return fail(RB_ERR_INVAL, what);
  }
  if (B <= 0 || history <= 0 || n <= 0 || size <= 0) {
    snprintf(what, sizeof what, "%s: sizes must be positive", who);
    return fail(RB_ERR_INVAL, what);
  }
  if (history + n > RB_MAX_WINDOW) {
    snprintf(what, sizeof what, "%s: history + n exceeds RB_MAX_WINDOW", who);
    return fail(RB_ERR_RANGE, what);
  }
  if (B > 65535) {
    snprintf(what, sizeof what, "%s: B exceeds 65535", who);
    return fail(RB_ERR_RANGE, what);
  }
  return RB_OK;
}

// the augmentation arguments of rb_gather_shift (pad_min 1, intensity 0, one copy), rb_gather_aug and rb_gather_horizon
static int aug_check(const char* who, int pad, int pad_min, float intensity, int m_copies, int k_copies) {
  char what[96];
  if (pad < pad_min || pad > RB_MAX_SHIFT_PAD) {
    snprintf(what, sizeof what, "%s: pad outside [%d, RB_MAX_SHIFT_PAD]", who, pad_min);
    return fail(RB_ERR_RANGE, what);
  }
  if (!(intensity >= 0.0f && intensity <= 0.5f)) {
    snprintf(what, sizeof what, "%s: intensity outside [0, 0.5]", who);
    return fail(RB_ERR_RANGE, what);
  }
  if (m_copies < 1 || m_copies > RB_MAX_AUG_COPIES || k_copies < 1 || k_copies > RB_MAX_AUG_COPIES) {
    snprintf(what, sizeof what, "%s: copies outside [1, RB_MAX_AUG_COPIES]", who);
    return fail(RB_ERR_RANGE, what);
  }
  return RB_OK;
}

int rb_gather(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
              const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n,
              const float* gamma_pow, float* states, float* next_states, int64_t* actions, float* returns,
              float* nonterminals, rb_stream_t stream) {
  const int rc = gather_check("rb_gather", frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n,
                              gamma_pow, states, next_states, actions, returns, nonterminals);
  if (rc != RB_OK) return rc;
  int split;
  const dim3 grid = gather_grid(history, n, B, &split);
  { ProfScope prof_(RB_K_GATHER, (cudaStream_t)stream);
    k_gather<<<grid, GATHER_THREADS, 0, (cudaStream_t)stream>>>(frames, timestep, action, reward, nonterminal, size, data_idx,
                                                              B, history, n, gamma_pow, states, next_states, actions,
                                                              returns, nonterminals, split); }
  return check_launch("rb_gather");
}

int rb_gather_shift(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                    const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n,
                    const float* gamma_pow, float* states, float* next_states, int64_t* actions, float* returns,
                    float* nonterminals, int pad, uint64_t seed, const uint64_t* rng_counter, int32_t* shifts,
                    rb_stream_t stream) {
  const int rc = gather_check("rb_gather_shift", frames, timestep, action, reward, nonterminal, size, data_idx, B, history,
                              n, gamma_pow, states, next_states, actions, returns, nonterminals);
  if (rc != RB_OK) return rc;
  if (!rng_counter || !shifts) return fail(RB_ERR_INVAL, "rb_gather_shift: null pointer");
  const int arc = aug_check("rb_gather_shift", pad, 1, 0.0f, 1, 1);
  if (arc != RB_OK) return arc;
  int split;
  const dim3 grid = gather_grid(history, n, B, &split);
  { ProfScope prof_(RB_K_GATHER_SHIFT, (cudaStream_t)stream);
    k_gather_shift<<<grid, GATHER_THREADS, 0, (cudaStream_t)stream>>>(
      frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n, gamma_pow, states, next_states, actions,
      returns, nonterminals, split, pad, seed, (const unsigned long long*)rng_counter, shifts); }
  return check_launch("rb_gather_shift");
}

int rb_gather_aug(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                  const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n,
                  const float* gamma_pow, float* states, float* next_states, int64_t* actions, float* returns,
                  float* nonterminals, int pad, float intensity, int m_copies, int k_copies, uint64_t seed,
                  const uint64_t* rng_counter, int32_t* shifts, float* scales, rb_stream_t stream) {
  const int rc = gather_check("rb_gather_aug", frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n,
                              gamma_pow, states, next_states, actions, returns, nonterminals);
  if (rc != RB_OK) return rc;
  if (!rng_counter || !shifts || !scales) return fail(RB_ERR_INVAL, "rb_gather_aug: null pointer");
  const int arc = aug_check("rb_gather_aug", pad, 0, intensity, m_copies, k_copies);
  if (arc != RB_OK) return arc;
  if (pad == 0 && intensity == 0.0f && m_copies == 1 && k_copies == 1)
    return fail(RB_ERR_INVAL, "rb_gather_aug: no augmentation requested (that is rb_gather)");
  int split;
  const dim3 grid = gather_grid(history, n, B, &split);
  { ProfScope prof_(RB_K_GATHER_AUG, (cudaStream_t)stream);
    k_gather_aug<<<grid, GATHER_THREADS, 0, (cudaStream_t)stream>>>(
      frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n, gamma_pow, states, next_states, actions,
      returns, nonterminals, split, pad, intensity, m_copies, k_copies, seed, (const unsigned long long*)rng_counter, shifts,
      scales); }
  return check_launch("rb_gather_aug");
}

int rb_horizon_advance(const rb_horizon* table, int T, int64_t* counter, rb_horizon* current, rb_stream_t stream) {
  if (!table || !counter || !current) return fail(RB_ERR_INVAL, "rb_horizon_advance: null pointer");
  if (T < 1 || T > RB_MAX_ANNEAL_STEPS) return fail(RB_ERR_RANGE, "rb_horizon_advance: T outside [1, RB_MAX_ANNEAL_STEPS]");
  k_horizon_advance<<<1, 1, 0, (cudaStream_t)stream>>>(table, T, (long long*)counter, current);
  return check_launch("rb_horizon_advance");
}

}  // extern "C"

// rb_gather_horizon (TRUNC false) and rb_gather_trunc (TRUNC true): the same checks, grid and kernel choice
template <bool TRUNC>
static int horizon_launch(const char* who, const uint8_t* frames, const int32_t* timestep, const int32_t* action,
                          const float* reward, const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B,
                          int history, int n_max, const rb_horizon* current, float* states, float* next_states,
                          int64_t* actions, float* returns, float* nonterminals, int pad, float intensity, int m_copies,
                          int k_copies, uint64_t seed, const uint64_t* rng_counter, int32_t* shifts, float* scales,
                          rb_stream_t stream) {
  char what[96];
  snprintf(what, sizeof what, "%s: null pointer", who);
  if (!current) return fail(RB_ERR_INVAL, what);
  const int rc = gather_check(who, frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max,
                              reinterpret_cast<const float*>(current), states, next_states, actions, returns, nonterminals);
  if (rc != RB_OK) return rc;
  const int arc = aug_check(who, pad, 0, intensity, m_copies, k_copies);
  if (arc != RB_OK) return arc;
  const bool plain = pad == 0 && intensity == 0.0f && m_copies == 1 && k_copies == 1;
  const bool shift = !plain && intensity == 0.0f && m_copies == 1 && k_copies == 1;
  if (!plain && (!rng_counter || !shifts || (!shift && !scales))) return fail(RB_ERR_INVAL, what);
  int split;
  const dim3 grid = gather_grid(history, n_max, B, &split);
  const unsigned long long* ctr = (const unsigned long long*)rng_counter;
  cudaStream_t s = (cudaStream_t)stream;
  // profiled under the id of the gather this launch stands for
  { ProfScope prof_(plain ? RB_K_GATHER : shift ? RB_K_GATHER_SHIFT : RB_K_GATHER_AUG, s);
    if (plain)
      (TRUNC ? k_gather_hz_trunc : k_gather_hz)<<<grid, GATHER_THREADS, 0, s>>>(
        frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max, current, states, next_states,
        actions, returns, nonterminals, split);
    else if (shift)
      (TRUNC ? k_gather_shift_hz_trunc : k_gather_shift_hz)<<<grid, GATHER_THREADS, 0, s>>>(
        frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max, current, states, next_states,
        actions, returns, nonterminals, split, pad, seed, ctr, shifts);
    else
      (TRUNC ? k_gather_aug_hz_trunc : k_gather_aug_hz)<<<grid, GATHER_THREADS, 0, s>>>(
        frames, timestep, action, reward, nonterminal, size, data_idx, B, history, n_max, current, states, next_states,
        actions, returns, nonterminals, split, pad, intensity, m_copies, k_copies, seed, ctr, shifts, scales); }
  return check_launch(who);
}

extern "C" {

int rb_gather_horizon(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                      const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n_max,
                      const rb_horizon* current, float* states, float* next_states, int64_t* actions, float* returns,
                      float* nonterminals, int pad, float intensity, int m_copies, int k_copies, uint64_t seed,
                      const uint64_t* rng_counter, int32_t* shifts, float* scales, rb_stream_t stream) {
  return horizon_launch<false>("rb_gather_horizon", frames, timestep, action, reward, nonterminal, size, data_idx, B,
                               history, n_max, current, states, next_states, actions, returns, nonterminals, pad,
                               intensity, m_copies, k_copies, seed, rng_counter, shifts, scales, stream);
}

int rb_gather_trunc(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                    const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n_max,
                    const rb_horizon* current, float* states, float* next_states, int64_t* actions, float* returns,
                    float* nonterminals, int pad, float intensity, int m_copies, int k_copies, uint64_t seed,
                    const uint64_t* rng_counter, int32_t* shifts, float* scales, rb_stream_t stream) {
  return horizon_launch<true>("rb_gather_trunc", frames, timestep, action, reward, nonterminal, size, data_idx, B,
                              history, n_max, current, states, next_states, actions, returns, nonterminals, pad,
                              intensity, m_copies, k_copies, seed, rng_counter, shifts, scales, stream);
}

int rb_iter_states(const uint8_t* frames, const int32_t* timestep, int64_t size, int64_t first, int count, int history,
                   float* out, rb_stream_t stream) {
  if (!frames || !timestep || !out) return fail(RB_ERR_INVAL, "rb_iter_states: null pointer");
  if (count <= 0 || history <= 0 || history > RB_MAX_WINDOW || count > 65535)
    return fail(RB_ERR_RANGE, "rb_iter_states: count/history out of range");
  dim3 grid(history, count);
  { ProfScope prof_(RB_K_ITER_STATES, (cudaStream_t)stream);
    k_iter_states<<<grid, GATHER_THREADS, 0, (cudaStream_t)stream>>>(frames, timestep, size, first, history, out); }
  return check_launch("rb_iter_states");
}

int rb_append(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep, int32_t* action,
              float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max, const float* state_last_frame,
              int32_t action_value, float reward_value, int terminal, rb_stream_t stream) {
  if (!tree || !frames || !timestep || !action || !reward || !nonterminal || !ring_state || !running_max || !state_last_frame)
    return fail(RB_ERR_INVAL, "rb_append: null pointer");
  if (size <= 0 || (size & 1)) return fail(RB_ERR_INVAL, "rb_append: an even size is required");
  // k_append_batch's limit; a deeper tree holds more than 2^30 transitions (7.6 TB of frames), which no replay reaches
  if (tree_depth(tree_start) > 30) return fail(RB_ERR_RANGE, "rb_append: tree deeper than 30 levels");
  if (((uintptr_t)state_last_frame & 15) != 0) return fail(RB_ERR_INVAL, "rb_append: state_last_frame must be 16-byte aligned");
  AppendBatch ab;
  memset(&ab, 0, sizeof(ab));
  ab.k = 1;
  ab.frame[0] = state_last_frame;
  ab.action[0] = action_value;
  ab.reward[0] = reward_value;
  ab.terminal[0] = terminal ? 1 : 0;
  return append_launch(tree, tree_start, size, frames, timestep, action, reward, nonterminal, ring_state, running_max, ab,
                       stream, "rb_append");
}

}  // extern "C"

// rb_append_batch (final_records false) and rb_append_batch_trunc (true)
static int append_batch_launch(const char* who, bool final_records, float* tree, int64_t tree_start, int64_t size,
                               uint8_t* frames, int32_t* timestep, int32_t* action, float* reward, uint8_t* nonterminal,
                               int64_t* ring_state, float* running_max, const float* const* last_frames,
                               const int32_t* actions, const float* rewards, const int32_t* terminals, int k,
                               rb_stream_t stream) {
  char what[112];
  if (!tree || !frames || !timestep || !action || !reward || !nonterminal || !ring_state || !running_max || !last_frames ||
      !actions || !rewards || !terminals) {
    snprintf(what, sizeof what, "%s: null pointer", who);
    return fail(RB_ERR_INVAL, what);
  }
  if (size <= 0 || (size & 1)) {
    snprintf(what, sizeof what, "%s: an even size is required", who);
    return fail(RB_ERR_INVAL, what);
  }
  if (k <= 0 || k > RB_APPEND_BATCH || k > size) {
    snprintf(what, sizeof what, "%s: 1 <= k <= RB_APPEND_BATCH (and k <= size)", who);
    return fail(RB_ERR_RANGE, what);
  }
  if (tree_depth(tree_start) > 30) {
    snprintf(what, sizeof what, "%s: tree deeper than 30 levels", who);
    return fail(RB_ERR_RANGE, what);
  }
  AppendBatch ab;
  memset(&ab, 0, sizeof(ab));
  ab.k = k;
  for (int j = 0; j < k; ++j) {
    if (!last_frames[j] || ((uintptr_t)last_frames[j] & 15)) {
      snprintf(what, sizeof what, "%s: frames must be non-null and 16-byte aligned", who);
      return fail(RB_ERR_INVAL, what);
    }
    const bool final_record = final_records && terminals[j] == RB_NONTERMINAL_FINAL;
    ab.frame[j] = last_frames[j];
    ab.action[j] = final_record ? 0 : actions[j];
    ab.reward[j] = final_record ? 0.0f : rewards[j];
    ab.terminal[j] = final_record ? RB_NONTERMINAL_FINAL : terminals[j] ? 1 : 0;
  }
  return append_launch(tree, tree_start, size, frames, timestep, action, reward, nonterminal, ring_state, running_max, ab,
                       stream, who, final_records);
}

extern "C" {

int rb_append_batch(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep, int32_t* action,
                    float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max,
                    const float* const* last_frames, const int32_t* actions, const float* rewards, const int32_t* terminals,
                    int k, rb_stream_t stream) {
  return append_batch_launch("rb_append_batch", false, tree, tree_start, size, frames, timestep, action, reward,
                             nonterminal, ring_state, running_max, last_frames, actions, rewards, terminals, k, stream);
}

int rb_append_batch_trunc(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep,
                          int32_t* action, float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max,
                          const float* const* last_frames, const int32_t* actions, const float* rewards,
                          const int32_t* terminals, int k, rb_stream_t stream) {
  return append_batch_launch("rb_append_batch_trunc", true, tree, tree_start, size, frames, timestep, action, reward,
                             nonterminal, ring_state, running_max, last_frames, actions, rewards, terminals, k, stream);
}

int rb_append_bulk_scratch_bytes(int64_t k) {
  if (k <= 0) return 0;
  if (k > ((int64_t)1 << 30)) k = (int64_t)1 << 30;   // rb_append_bulk's largest k (size <= 2^30)
  return (int)(sizeof(int) * ((k + BULK_TILE - 1) / BULK_TILE + 1));
}

int rb_append_bulk(float* tree, int64_t tree_start, int64_t size, uint8_t* frames, int32_t* timestep, int32_t* action,
                   float* reward, uint8_t* nonterminal, int64_t* ring_state, float* running_max, int64_t head,
                   const uint8_t* new_frames, const int32_t* actions, const float* rewards, const uint8_t* flags,
                   int64_t k, void* scratch, int64_t scratch_bytes, rb_stream_t stream) {
  if (!tree || !frames || !timestep || !action || !reward || !nonterminal || !ring_state || !running_max || !new_frames ||
      !actions || !rewards || !flags || !scratch)
    return fail(RB_ERR_INVAL, "rb_append_bulk: null pointer");
  if (size <= 0 || (size & 1)) return fail(RB_ERR_INVAL, "rb_append_bulk: an even size is required");
  if (tree_depth(tree_start) > 30) return fail(RB_ERR_RANGE, "rb_append_bulk: tree deeper than 30 levels");
  if (k < 1 || k > size) return fail(RB_ERR_RANGE, "rb_append_bulk: 1 <= k <= size");
  if (head < 0 || head >= size) return fail(RB_ERR_RANGE, "rb_append_bulk: head outside [0, size)");
  if (scratch_bytes < rb_append_bulk_scratch_bytes(k))
    return fail(RB_ERR_RANGE, "rb_append_bulk: scratch smaller than rb_append_bulk_scratch_bytes(k)");
  cudaStream_t st = (cudaStream_t)stream;
  const int kk = (int)k;   // k <= size <= 2^30
  const int tiles = (kk + BULK_TILE - 1) / BULK_TILE;
  int* tile_reset = static_cast<int*>(scratch);
  { ProfScope prof_(RB_K_APPEND, st);
    // frames: copy-engine copies (device or pinned host source), split at the wrap
    const int64_t n1 = head + k <= size ? k : size - head;
    cudaError_t e = cudaMemcpyAsync(frames + (size_t)head * RB_FRAME_BYTES, new_frames, (size_t)n1 * RB_FRAME_BYTES,
                                    cudaMemcpyDefault, st);
    if (e == cudaSuccess && n1 < k)
      e = cudaMemcpyAsync(frames, new_frames + (size_t)n1 * RB_FRAME_BYTES, (size_t)(k - n1) * RB_FRAME_BYTES,
                          cudaMemcpyDefault, st);
    if (e != cudaSuccess) return fail(RB_ERR_CUDA, cudaGetErrorString(e));
    k_bulk_block_reset<<<tiles, BULK_THREADS, 0, st>>>(flags, kk, tile_reset);
    k_bulk_scan_tiles<<<1, BULK_TOP_THREADS, 0, st>>>(tile_reset, tiles);
    k_bulk_records<<<tiles, BULK_THREADS, 0, st>>>(tree, tree_start, size, timestep, action, reward, nonterminal,
                                                    ring_state, running_max, actions, rewards, flags, kk, tile_reset);
    // a level s above the leaves holds at most (k >> s) + 4 touched nodes; the wide ones get a grid each
    const int L = tree_depth(tree_start);
    int s = 1;
    for (; s <= L && (k >> s) + 4 > 4 * BULK_TOP_THREADS; ++s) {
      const int64_t n = (k >> s) + 4;
      k_bulk_tree_level<<<(unsigned)((n + BULK_THREADS - 1) / BULK_THREADS), BULK_THREADS, 0, st>>>(
          tree, tree_start, size, ring_state, kk, s);
    }
    k_bulk_tree_top<<<1, BULK_TOP_THREADS, 0, st>>>(tree, tree_start, size, ring_state, kk, s, tile_reset, tiles); }
  return check_launch("rb_append_bulk");
}

// The value-rescaled entries' own refusals: support_q (C51) given, 0 <= eps <= 1 (NaN refused).
static int vt_check(const char* name, bool support_q_ok, float eps) {
  char msg[128];
  if (!support_q_ok) {
    snprintf(msg, sizeof msg, "%s: null pointer", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (!(eps >= 0.0f && eps <= 1.0f)) {
    snprintf(msg, sizeof msg, "%s: eps must be in [0, 1]", name);
    return fail(RB_ERR_INVAL, msg);
  }
  return RB_OK;
}

static int null_pointer(const char* name) {
  char msg[128];
  snprintf(msg, sizeof msg, "%s: null pointer", name);
  return fail(RB_ERR_INVAL, msg);
}

// The C51 launchers' shared refusals; a_name / z_name: what the entry calls A and Z in its messages.
static int c51_check(const char* name, bool pointers_ok, int B, int A, int Z, const char* a_name, const char* z_name) {
  if (!pointers_ok) return null_pointer(name);
  char msg[128];
  if (B <= 0 || A <= 0 || Z <= 1) {
    snprintf(msg, sizeof msg, "%s: B, %s > 0 and %s > 1 are required", name, a_name, z_name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (Z > RB_MAX_ATOMS) {
    snprintf(msg, sizeof msg, "%s: %s exceeds RB_MAX_ATOMS", name, z_name);
    return fail(RB_ERR_RANGE, msg);
  }
  return RB_OK;
}

// The averaging launchers' copies range and the fused loss launchers' shared-memory limit.  Those launchers grant the
// dynamic shared memory to both R instantiations: ensure_dynamic_smem skips requests of at most 48 KB without counting the
// kernel's static shared memory, so a launch can depend on a grant a larger request of the other R already made.
static int copies_check(const char* name, int M, int K) {
  if (M < 1 || M > RB_MAX_AUG_COPIES || K < 1 || K > RB_MAX_AUG_COPIES) {
    char msg[128];
    snprintf(msg, sizeof msg, "%s: copies outside [1, RB_MAX_AUG_COPIES]", name);
    return fail(RB_ERR_RANGE, msg);
  }
  return RB_OK;
}

static int smem_check(const char* name, size_t smem, const char* what) {
  if (smem > 200 * 1024) {
    char msg[128];
    snprintf(msg, sizeof msg, "%s: %s", name, what);
    return fail(RB_ERR_RANGE, msg);
  }
  return RB_OK;
}

// The risk entries' own refusals: a known kind; CVaR eta in (0, 1], Wang eta finite (NaN fails every comparison).
static int risk_check(const char* name, int kind, float eta) {
  char msg[128];
  if (kind != RB_RISK_CVAR && kind != RB_RISK_WANG) {
    snprintf(msg, sizeof msg, "%s: risk_kind must be RB_RISK_CVAR or RB_RISK_WANG", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (kind == RB_RISK_CVAR && !(eta > 0.0f && eta <= 1.0f)) {
    snprintf(msg, sizeof msg, "%s: CVaR eta must be in (0, 1]", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (kind == RB_RISK_WANG && !isfinite(eta)) {
    snprintf(msg, sizeof msg, "%s: Wang eta must be finite", name);
    return fail(RB_ERR_INVAL, msg);
  }
  return RB_OK;
}

extern "C++" {   // the shared launchers are templates, which cannot have C linkage
template <bool VT, bool RISK = false>
static int c51_launch(const char* name, const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                      const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                      const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z,
                      float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, const float* support_q, float eps,
                      rb_stream_t stream, int risk_kind = 0, float risk_eta = 0.0f) {
  int rc = VT ? vt_check(name, support_q != nullptr, eps) : RB_OK;
  if (rc == RB_OK)
    rc = c51_check(name, q_online_s && q_online_ns && q_target_ns && actions && returns && nonterminals && weights &&
                   support && loss && grad_q_online_s, B, A, Z, "A", "Z");
  if (rc == RB_OK && RISK) rc = risk_check(name, risk_kind, risk_eta);
  if (rc != RB_OK) return rc;
  constexpr int F = RISK ? RISK_INST : 0;
  const auto k = Z <= 64 ? k_c51<2 | F, VT> : k_c51<4 | F, VT>;
  { ProfScope prof_(RB_K_C51, (cudaStream_t)stream);
    k<<<(B + C51_WARPS - 1) / C51_WARPS, C51_WARPS * 32, 0, (cudaStream_t)stream>>>(
        q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n,
        B, A, Z, loss, grad_q_online_s, m_out, astar_out, support_q, eps, risk_kind, risk_eta); }
  return check_launch(name);
}
}

int rb_c51_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                     const float* returns, const float* nonterminals, const float* weights, const float* support,
                     float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z, float* loss,
                     float* grad_q_online_s, float* m_out, int64_t* astar_out, rb_stream_t stream) {
  return c51_launch<false>("rb_c51_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights,
                           support, vmin, vmax, delta_z, gamma_n, B, A, Z, loss, grad_q_online_s, m_out, astar_out, nullptr,
                           0.0f, stream);
}

int rb_c51_vt_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                        const float* returns, const float* nonterminals, const float* weights, const float* support,
                        float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z, float* loss,
                        float* grad_q_online_s, float* m_out, int64_t* astar_out, const float* support_q, float eps,
                        rb_stream_t stream) {
  return c51_launch<true>("rb_c51_vt_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals,
                          weights, support, vmin, vmax, delta_z, gamma_n, B, A, Z, loss, grad_q_online_s, m_out, astar_out,
                          support_q, eps, stream);
}

int rb_c51_risk_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                          const float* returns, const float* nonterminals, const float* weights, const float* support,
                          float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z, float* loss,
                          float* grad_q_online_s, float* m_out, int64_t* astar_out, int risk_kind, float risk_eta,
                          rb_stream_t stream) {
  return c51_launch<false, true>("rb_c51_risk_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns,
                                 nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, A, Z, loss, grad_q_online_s,
                                 m_out, astar_out, nullptr, 0.0f, stream, risk_kind, risk_eta);
}

static int noisy_launch(float* const* weight_eps, float* const* bias_eps, const int* in_features, const int* out_features,
                        int n_layers, const float* x_in, const float* x_out, uint64_t seed, uint64_t* rng_counter,
                        int prescaled, rb_stream_t stream) {
  if (!weight_eps || !bias_eps || !in_features || !out_features) return fail(RB_ERR_INVAL, "rb_noisy_resample: null pointer");
  if (n_layers <= 0 || n_layers > RB_MAX_NOISY_LAYERS) return fail(RB_ERR_RANGE, "rb_noisy_resample: n_layers out of range");
  if ((x_in == nullptr) != (x_out == nullptr)) return fail(RB_ERR_INVAL, "rb_noisy_resample: give both x_in and x_out or neither");
  if (x_in == nullptr && rng_counter == nullptr) return fail(RB_ERR_INVAL, "rb_noisy_resample: need injected normals or rng_counter");
  NoisyPlan plan;
  memset(&plan, 0, sizeof(plan));
  plan.n = n_layers;
  int in_off = 0, out_off = 0, ctas = 0, max_in = 0;
  for (int l = 0; l < n_layers; ++l) {
    if (!weight_eps[l] || !bias_eps[l] || in_features[l] <= 0 || out_features[l] <= 0)
      return fail(RB_ERR_INVAL, "rb_noisy_resample: bad layer description");
    if (in_features[l] > 57000) return fail(RB_ERR_RANGE, "rb_noisy_resample: in_features exceeds shared-memory staging");
    plan.w[l] = weight_eps[l];
    plan.b[l] = bias_eps[l];
    plan.in_f[l] = in_features[l];
    plan.out_f[l] = out_features[l];
    plan.in_off[l] = in_off;
    plan.out_off[l] = out_off;
    in_off += in_features[l];
    out_off += out_features[l];
    // ~24K weights per CTA, at least 8 rows (one per warp)
    int rows = 24576 / in_features[l];
    if (rows < 8) rows = 8;
    plan.rows_per_cta[l] = rows;
    plan.cta_begin[l] = ctas;
    ctas += (out_features[l] + rows - 1) / rows;
    if (in_features[l] > max_in) max_in = in_features[l];
  }
  plan.cta_begin[n_layers] = ctas;
  const size_t smem = (size_t)max_in * sizeof(float);
  {
    int rc_s = rbi::ensure_dynamic_smem(k_noisy_resample, smem, "rb_noisy_resample");
    if (rc_s != RB_OK) return rc_s;
  }
  { ProfScope prof_(RB_K_NOISY_RESAMPLE, (cudaStream_t)stream);
    k_noisy_resample<<<ctas, NOISY_THREADS, smem, (cudaStream_t)stream>>>(plan, x_in, x_out, seed,
                                                                       (unsigned long long*)rng_counter, prescaled); }
  int rc = check_launch("rb_noisy_resample");
  if (rc != RB_OK) return rc;
  if (x_in == nullptr) {
    k_bump_counter<<<1, 1, 0, (cudaStream_t)stream>>>((unsigned long long*)rng_counter);
    rc = check_launch("rb_noisy_resample(counter)");
  }
  return rc;
}

int rb_noisy_resample(float* const* weight_eps, float* const* bias_eps, const int* in_features, const int* out_features,
                      int n_layers, const float* x_in, const float* x_out, uint64_t seed, uint64_t* rng_counter,
                      rb_stream_t stream) {
  return noisy_launch(weight_eps, bias_eps, in_features, out_features, n_layers, x_in, x_out, seed, rng_counter, 0, stream);
}

int rb_noisy_outer(float* const* weight_eps, float* const* bias_eps, const int* in_features, const int* out_features,
                   int n_layers, const float* f_in, const float* f_out, rb_stream_t stream) {
  if (!f_in || !f_out) return fail(RB_ERR_INVAL, "rb_noisy_outer: null factor vectors");
  return noisy_launch(weight_eps, bias_eps, in_features, out_features, n_layers, f_in, f_out, 0, nullptr, 1, stream);
}

extern "C++" {
template <bool VT, bool RISK = false>
static int c51_dueling_launch(const char* name, const float* z_online, const float* z_target, int actions_n, int atoms,
                              const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                              const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, float* loss,
                              float* dz, float* m_out, int64_t* astar_out, const float* support_q, float eps,
                              rb_stream_t stream, int risk_kind = 0, float risk_eta = 0.0f) {
  const int Z = atoms, A = actions_n;
  int rc = VT ? vt_check(name, support_q != nullptr, eps) : RB_OK;
  if (rc == RB_OK)
    rc = c51_check(name, z_online && z_target && actions && returns && nonterminals && weights && support && loss && dz, B,
                   A, Z, "actions", "atoms");
  if (rc == RB_OK && RISK) rc = risk_check(name, risk_kind, risk_eta);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)(3 * (Z + A * Z) + 3 * Z + A) * sizeof(float);
  rc = smem_check(name, smem, "actions * atoms too large");
  constexpr int F = RISK ? RISK_INST : 0;
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling<2 | F, VT>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling<4 | F, VT>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = Z <= 64 ? k_c51_dueling<2 | F, VT> : k_c51_dueling<4 | F, VT>;
  { ProfScope prof_(RB_K_C51_DUELING, (cudaStream_t)stream);
    k<<<B, C51D_T, smem, (cudaStream_t)stream>>>(z_online, z_target, actions, returns, nonterminals, weights, support, vmin,
                                                 vmax, delta_z, gamma_n, B, A, Z, loss, dz, m_out, astar_out, support_q, eps,
                                                 risk_kind, risk_eta); }
  return check_launch(name);
}
}

int rb_c51_dueling_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                             const float* returns, const float* nonterminals, const float* weights, const float* support,
                             float vmin, float vmax, float delta_z, float gamma_n, int B, float* loss, float* dz, float* m_out,
                             int64_t* astar_out, rb_stream_t stream) {
  return c51_dueling_launch<false>("rb_c51_dueling_loss_grad", z_online, z_target, actions_n, atoms, actions, returns,
                                   nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, loss, dz, m_out,
                                   astar_out, nullptr, 0.0f, stream);
}

int rb_c51_dueling_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                                const float* returns, const float* nonterminals, const float* weights, const float* support,
                                float vmin, float vmax, float delta_z, float gamma_n, int B, float* loss, float* dz,
                                float* m_out, int64_t* astar_out, const float* support_q, float eps, rb_stream_t stream) {
  return c51_dueling_launch<true>("rb_c51_dueling_vt_loss_grad", z_online, z_target, actions_n, atoms, actions, returns,
                                  nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, loss, dz, m_out, astar_out,
                                  support_q, eps, stream);
}

int rb_c51_dueling_risk_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                  const int64_t* actions, const float* returns, const float* nonterminals,
                                  const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                  float gamma_n, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                  int risk_kind, float risk_eta, rb_stream_t stream) {
  return c51_dueling_launch<false, true>("rb_c51_dueling_risk_loss_grad", z_online, z_target, actions_n, atoms, actions,
                                         returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, loss, dz,
                                         m_out, astar_out, nullptr, 0.0f, stream, risk_kind, risk_eta);
}

// The HL-Gauss entries' own refusal: sigma a positive normal fp32 (NaN, +-inf, 0, negatives and subnormals refused).
static int hlg_check(const char* name, float sigma) {
  if (!(sigma >= 1.17549435e-38f && sigma <= 3.40282347e+38f)) {
    char msg[128];
    snprintf(msg, sizeof msg, "%s: sigma must be a positive normal fp32", name);
    return fail(RB_ERR_INVAL, msg);
  }
  return RB_OK;
}

int rb_c51_hlg_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                         const float* returns, const float* nonterminals, const float* weights, const float* support,
                         float vmin, float vmax, float delta_z, float gamma_n, float sigma, int B, int A, int Z,
                         float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, float* y_out,
                         rb_stream_t stream) {
  const char* name = "rb_c51_hlg_loss_grad";
  int rc = c51_check(name, q_online_s && q_online_ns && q_target_ns && actions && returns && nonterminals && weights &&
                     support && loss && grad_q_online_s, B, A, Z, "A", "Z");
  if (rc == RB_OK) rc = hlg_check(name, sigma);
  if (rc != RB_OK) return rc;
  const auto k = Z <= 64 ? k_c51_hlg<2> : k_c51_hlg<4>;
  { ProfScope prof_(RB_K_C51, (cudaStream_t)stream);
    k<<<(B + C51_WARPS - 1) / C51_WARPS, C51_WARPS * 32, 0, (cudaStream_t)stream>>>(
        q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n,
        sigma, B, A, Z, loss, grad_q_online_s, m_out, astar_out, y_out); }
  return check_launch(name);
}

int rb_c51_dueling_hlg_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                 const int64_t* actions, const float* returns, const float* nonterminals,
                                 const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                 float gamma_n, float sigma, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                 float* y_out, rb_stream_t stream) {
  const char* name = "rb_c51_dueling_hlg_loss_grad";
  const int Z = atoms, A = actions_n;
  int rc = c51_check(name, z_online && z_target && actions && returns && nonterminals && weights && support && loss && dz,
                     B, A, Z, "actions", "atoms");
  if (rc == RB_OK) rc = hlg_check(name, sigma);
  if (rc != RB_OK) return rc;
  // k_c51_dueling's size (the kernel leaves its [Z] slot of target logits unused), so both refuse the same shapes
  const size_t smem = (size_t)(3 * (Z + A * Z) + 3 * Z + A) * sizeof(float);
  rc = smem_check(name, smem, "actions * atoms too large");
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling_hlg<2>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling_hlg<4>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = Z <= 64 ? k_c51_dueling_hlg<2> : k_c51_dueling_hlg<4>;
  { ProfScope prof_(RB_K_C51_DUELING, (cudaStream_t)stream);
    k<<<B, C51D_T, smem, (cudaStream_t)stream>>>(z_online, z_target, actions, returns, nonterminals, weights, support, vmin,
                                                 vmax, delta_z, gamma_n, sigma, B, A, Z, loss, dz, m_out, astar_out, y_out); }
  return check_launch(name);
}

// The two-hot entries: the parents' refusals in the parents' order (under VT rb_c51_vt_loss_grad's first), then
// k_c51_twohot / k_c51_dueling_twohot in the parents' launch shapes.
extern "C++" {
template <bool VT>
static int c51_twohot_launch(const char* name, const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                             const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                             const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z,
                             float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, float* y_out,
                             const float* support_q, float eps, rb_stream_t stream) {
  int rc = VT ? vt_check(name, support_q != nullptr, eps) : RB_OK;
  if (rc == RB_OK)
    rc = c51_check(name, q_online_s && q_online_ns && q_target_ns && actions && returns && nonterminals && weights &&
                   support && loss && grad_q_online_s, B, A, Z, "A", "Z");
  if (rc != RB_OK) return rc;
  const auto k = Z <= 64 ? k_c51_twohot<2, VT> : k_c51_twohot<4, VT>;
  { ProfScope prof_(RB_K_C51, (cudaStream_t)stream);
    k<<<(B + C51_WARPS - 1) / C51_WARPS, C51_WARPS * 32, 0, (cudaStream_t)stream>>>(
        q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n,
        B, A, Z, loss, grad_q_online_s, m_out, astar_out, y_out, support_q, eps); }
  return check_launch(name);
}

template <bool VT>
static int c51_dueling_twohot_launch(const char* name, const float* z_online, const float* z_target, int actions_n,
                                     int atoms, const int64_t* actions, const float* returns, const float* nonterminals,
                                     const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                     float gamma_n, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                     float* y_out, const float* support_q, float eps, rb_stream_t stream) {
  const int Z = atoms, A = actions_n;
  int rc = VT ? vt_check(name, support_q != nullptr, eps) : RB_OK;
  if (rc == RB_OK)
    rc = c51_check(name, z_online && z_target && actions && returns && nonterminals && weights && support && loss && dz, B,
                   A, Z, "actions", "atoms");
  if (rc != RB_OK) return rc;
  // k_c51_dueling's size (the kernel leaves its [Z] slot of target logits unused), so both refuse the same shapes
  const size_t smem = (size_t)(3 * (Z + A * Z) + 3 * Z + A) * sizeof(float);
  rc = smem_check(name, smem, "actions * atoms too large");
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling_twohot<2, VT>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling_twohot<4, VT>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = Z <= 64 ? k_c51_dueling_twohot<2, VT> : k_c51_dueling_twohot<4, VT>;
  { ProfScope prof_(RB_K_C51_DUELING, (cudaStream_t)stream);
    k<<<B, C51D_T, smem, (cudaStream_t)stream>>>(z_online, z_target, actions, returns, nonterminals, weights, support, vmin,
                                                 vmax, delta_z, gamma_n, B, A, Z, loss, dz, m_out, astar_out, y_out,
                                                 support_q, eps); }
  return check_launch(name);
}
}

int rb_c51_twohot_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                            const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                            const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z,
                            float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, float* y_out,
                            rb_stream_t stream) {
  return c51_twohot_launch<false>("rb_c51_twohot_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns,
                                  nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, A, Z, loss,
                                  grad_q_online_s, m_out, astar_out, y_out, nullptr, 0.0f, stream);
}

int rb_c51_twohot_vt_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                               const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                               const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int A,
                               int Z, float* loss, float* grad_q_online_s, float* m_out, int64_t* astar_out, float* y_out,
                               const float* support_q, float eps, rb_stream_t stream) {
  return c51_twohot_launch<true>("rb_c51_twohot_vt_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns,
                                 nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, A, Z, loss,
                                 grad_q_online_s, m_out, astar_out, y_out, support_q, eps, stream);
}

int rb_c51_dueling_twohot_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                    const int64_t* actions, const float* returns, const float* nonterminals,
                                    const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                    float gamma_n, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                    float* y_out, rb_stream_t stream) {
  return c51_dueling_twohot_launch<false>("rb_c51_dueling_twohot_loss_grad", z_online, z_target, actions_n, atoms, actions,
                                          returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, loss, dz,
                                          m_out, astar_out, y_out, nullptr, 0.0f, stream);
}

int rb_c51_dueling_twohot_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                       const int64_t* actions, const float* returns, const float* nonterminals,
                                       const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                       float gamma_n, int B, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                       float* y_out, const float* support_q, float eps, rb_stream_t stream) {
  return c51_dueling_twohot_launch<true>("rb_c51_dueling_twohot_vt_loss_grad", z_online, z_target, actions_n, atoms,
                                         actions, returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B,
                                         loss, dz, m_out, astar_out, y_out, support_q, eps, stream);
}

// The CQL entries: the loss entries' shape refusals (c51_check), alpha a positive normal fp32 (NaN, +-inf, 0, negatives
// and subnormals refused), M in [1, RB_MAX_AUG_COPIES], then the shared-memory limit; k_cql_dueling / k_cql with one CTA
// per sample.  A NULL support selects the quantile head.
extern "C++" {
template <bool DUELING>
static int cql_launch(const char* name, const float* rows, const int64_t* actions, const float* weights,
                      const float* support, float alpha, int M, int B, int A, int Z, float* grad, float* gap_out,
                      rb_stream_t stream) {
  int rc = c51_check(name, rows && actions && weights && grad, B, A, Z, "A", "Z");
  if (rc == RB_OK && !(alpha >= FLT_MIN && alpha <= FLT_MAX)) {
    char msg[128];
    snprintf(msg, sizeof msg, "%s: alpha must be a positive finite normal fp32", name);
    rc = fail(RB_ERR_INVAL, msg);
  }
  if (rc == RB_OK) rc = copies_check(name, M, 1);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)((DUELING ? 2 * Z : 0) + 2 * A * Z + 2 * A) * sizeof(float);
  rc = smem_check(name, smem, "A * Z too large");
  const auto k2 = support ? (DUELING ? k_cql_dueling<2, false> : k_cql<2, false>)
                          : (DUELING ? k_cql_dueling<2, true> : k_cql<2, true>);
  const auto k4 = support ? (DUELING ? k_cql_dueling<4, false> : k_cql<4, false>)
                          : (DUELING ? k_cql_dueling<4, true> : k_cql<4, true>);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k2, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k4, smem, name);
  if (rc != RB_OK) return rc;
  { ProfScope prof_(DUELING ? RB_K_C51_DUELING : RB_K_C51, (cudaStream_t)stream);
    (Z <= 64 ? k2 : k4)<<<B, CQL_T, smem, (cudaStream_t)stream>>>(rows, actions, weights, support, alpha, M, B, A, Z, grad,
                                                                  gap_out); }
  return check_launch(name);
}
}

int rb_cql_grad(const float* q_online_s, const int64_t* actions, const float* weights, const float* support, float alpha,
                int M, int B, int A, int Z, float* grad, float* gap_out, rb_stream_t stream) {
  return cql_launch<false>("rb_cql_grad", q_online_s, actions, weights, support, alpha, M, B, A, Z, grad, gap_out, stream);
}

int rb_cql_dueling_grad(const float* z_online, const int64_t* actions, const float* weights, const float* support,
                        float alpha, int M, int B, int A, int Z, float* dz, float* gap_out, rb_stream_t stream) {
  return cql_launch<true>("rb_cql_dueling_grad", z_online, actions, weights, support, alpha, M, B, A, Z, dz, gap_out,
                          stream);
}

extern "C++" {
template <bool VT>
static int c51_dueling_avg_launch(const char* name, const float* z_online, const float* z_target, int actions_n, int atoms,
                                  const int64_t* actions, const float* returns, const float* nonterminals,
                                  const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                  float gamma_n, int B, int M, int K, float* loss, float* dz, float* m_out, int64_t* astar_out,
                                  const float* support_q, float eps, rb_stream_t stream) {
  const int Z = atoms, A = actions_n;
  int rc = VT ? vt_check(name, support_q != nullptr, eps) : RB_OK;
  if (rc == RB_OK)
    rc = c51_check(name, z_online && z_target && actions && returns && nonterminals && weights && support && loss && dz, B,
                   A, Z, "actions", "atoms");
  if (rc == RB_OK) rc = copies_check(name, M, K);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)((M + 2 * K) * (Z + A * Z) + (2 * M + 2 * K + 1) * Z + K * A + M) * sizeof(float);
  rc = smem_check(name, smem, "(M + 2K) * actions * atoms too large");
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling_avg<2, VT>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_c51_dueling_avg<4, VT>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = Z <= 64 ? k_c51_dueling_avg<2, VT> : k_c51_dueling_avg<4, VT>;
  { ProfScope prof_(RB_K_C51_DUELING_AVG, (cudaStream_t)stream);
    k<<<B, C51D_T, smem, (cudaStream_t)stream>>>(z_online, z_target, actions, returns, nonterminals, weights, support, vmin,
                                                 vmax, delta_z, gamma_n, B, A, Z, M, K, loss, dz, m_out, astar_out, support_q,
                                                 eps); }
  return check_launch(name);
}
}

int rb_c51_dueling_avg_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                 const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                                 const float* support, float vmin, float vmax, float delta_z, float gamma_n, int B, int M,
                                 int K, float* loss, float* dz, float* m_out, int64_t* astar_out, rb_stream_t stream) {
  return c51_dueling_avg_launch<false>("rb_c51_dueling_avg_loss_grad", z_online, z_target, actions_n, atoms, actions,
                                       returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, M, K, loss,
                                       dz, m_out, astar_out, nullptr, 0.0f, stream);
}

int rb_c51_dueling_avg_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                    const int64_t* actions, const float* returns, const float* nonterminals,
                                    const float* weights, const float* support, float vmin, float vmax, float delta_z,
                                    float gamma_n, int B, int M, int K, float* loss, float* dz, float* m_out,
                                    int64_t* astar_out, const float* support_q, float eps, rb_stream_t stream) {
  return c51_dueling_avg_launch<true>("rb_c51_dueling_avg_vt_loss_grad", z_online, z_target, actions_n, atoms, actions,
                                      returns, nonterminals, weights, support, vmin, vmax, delta_z, gamma_n, B, M, K, loss,
                                      dz, m_out, astar_out, support_q, eps, stream);
}

int rb_q_values(const float* z, int M, int actions, int atoms, const float* support, float* q, int64_t* best_action,
                float* best_q, rb_stream_t stream) {
  if (!z || !support) return fail(RB_ERR_INVAL, "rb_q_values: null pointer");
  if (!q && !best_action && !best_q) return fail(RB_ERR_INVAL, "rb_q_values: no output requested");
  if (M <= 0 || actions <= 0 || atoms <= 1) return fail(RB_ERR_INVAL, "rb_q_values: M, actions > 0 and atoms > 1 are required");
  if (atoms > RB_MAX_ATOMS) return fail(RB_ERR_RANGE, "rb_q_values: atoms exceeds RB_MAX_ATOMS");
  { ProfScope prof_(RB_K_Q_VALUES, (cudaStream_t)stream);
    k_q_select<false><<<(M + 3) / 4, 128, 0, (cudaStream_t)stream>>>(z, M, actions, atoms, support, q, best_action, best_q, 0,
                                                                    0.0f); }
  return check_launch("rb_q_values");
}

int rb_q_values_risk(const float* z, int M, int actions, int atoms, const float* support, float* q, int64_t* best_action,
                     float* best_q, int risk_kind, float risk_eta, rb_stream_t stream) {
  const char* name = "rb_q_values_risk";
  if (!z || !support) return null_pointer(name);
  char msg[128];
  if (!q && !best_action && !best_q) {
    snprintf(msg, sizeof msg, "%s: no output requested", name);
    return fail(RB_ERR_INVAL, msg);
  }
  int rc = c51_check(name, true, M, actions, atoms, "actions", "atoms");
  if (rc == RB_OK) rc = risk_check(name, risk_kind, risk_eta);
  if (rc != RB_OK) return rc;
  { ProfScope prof_(RB_K_Q_VALUES, (cudaStream_t)stream);
    k_q_select<true><<<(M + 3) / 4, 128, 0, (cudaStream_t)stream>>>(z, M, actions, atoms, support, q, best_action, best_q,
                                                                   risk_kind, risk_eta); }
  return check_launch(name);
}

static int qr_check(const char* name, int B, int A, int N, float kappa) {
  char msg[128];
  if (B <= 0 || A <= 0 || N <= 1) {
    snprintf(msg, sizeof msg, "%s: B, actions > 0 and atoms > 1 are required", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (N > RB_MAX_ATOMS) {
    snprintf(msg, sizeof msg, "%s: atoms exceeds RB_MAX_ATOMS", name);
    return fail(RB_ERR_RANGE, msg);
  }
  if (!(kappa > 0.0f) || !isfinite(kappa)) {
    snprintf(msg, sizeof msg, "%s: kappa must be finite and > 0", name);
    return fail(RB_ERR_INVAL, msg);
  }
  return RB_OK;
}

extern "C++" {
template <bool VT, bool RISK = false>
static int qr_dueling_launch(const char* name, const float* z_online, const float* z_target, int actions_n, int atoms,
                             const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                             float kappa, float gamma_n, int B, float* loss, float* dz, float* theta_out, int64_t* astar_out,
                             float eps, rb_stream_t stream, int risk_kind = 0, float risk_eta = 0.0f) {
  const int N = atoms, A = actions_n;
  int rc = VT ? vt_check(name, true, eps) : RB_OK;
  if (rc == RB_OK && !(z_online && z_target && actions && returns && nonterminals && weights && loss && dz))
    rc = null_pointer(name);
  if (rc == RB_OK) rc = qr_check(name, B, A, N, kappa);
  if (rc == RB_OK && RISK) rc = risk_check(name, risk_kind, risk_eta);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)(3 * (N + A * N) + 4 * N + A) * sizeof(float);
  rc = smem_check(name, smem, "actions * atoms too large");
  constexpr int F = RISK ? RISK_INST : 0;
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_dueling<2 | F, VT>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_dueling<4 | F, VT>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = N <= 64 ? k_qr_dueling<2 | F, VT> : k_qr_dueling<4 | F, VT>;
  { ProfScope prof_(RB_K_C51_DUELING, (cudaStream_t)stream);
    k<<<B, QR_T, smem, (cudaStream_t)stream>>>(z_online, z_target, actions, returns, nonterminals, weights, kappa, gamma_n, B,
                                               A, N, loss, dz, theta_out, astar_out, eps, risk_kind, risk_eta); }
  return check_launch(name);
}
}

int rb_qr_dueling_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                            const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n,
                            int B, float* loss, float* dz, float* theta_out, int64_t* astar_out, rb_stream_t stream) {
  return qr_dueling_launch<false>("rb_qr_dueling_loss_grad", z_online, z_target, actions_n, atoms, actions, returns,
                                  nonterminals, weights, kappa, gamma_n, B, loss, dz, theta_out, astar_out, 0.0f, stream);
}

int rb_qr_dueling_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms, const int64_t* actions,
                               const float* returns, const float* nonterminals, const float* weights, float kappa,
                               float gamma_n, int B, float* loss, float* dz, float* theta_out, int64_t* astar_out, float eps,
                               rb_stream_t stream) {
  return qr_dueling_launch<true>("rb_qr_dueling_vt_loss_grad", z_online, z_target, actions_n, atoms, actions, returns,
                                 nonterminals, weights, kappa, gamma_n, B, loss, dz, theta_out, astar_out, eps, stream);
}

int rb_qr_dueling_risk_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                 const int64_t* actions, const float* returns, const float* nonterminals,
                                 const float* weights, float kappa, float gamma_n, int B, float* loss, float* dz,
                                 float* theta_out, int64_t* astar_out, int risk_kind, float risk_eta, rb_stream_t stream) {
  return qr_dueling_launch<false, true>("rb_qr_dueling_risk_loss_grad", z_online, z_target, actions_n, atoms, actions,
                                        returns, nonterminals, weights, kappa, gamma_n, B, loss, dz, theta_out, astar_out,
                                        0.0f, stream, risk_kind, risk_eta);
}

extern "C++" {
template <bool VT>
static int qr_dueling_avg_launch(const char* name, const float* z_online, const float* z_target, int actions_n, int atoms,
                                 const int64_t* actions, const float* returns, const float* nonterminals,
                                 const float* weights, float kappa, float gamma_n, int B, int M, int K, float* loss,
                                 float* dz, float* theta_out, int64_t* astar_out, float eps, rb_stream_t stream) {
  const int N = atoms, A = actions_n;
  int rc = VT ? vt_check(name, true, eps) : RB_OK;
  if (rc == RB_OK && !(z_online && z_target && actions && returns && nonterminals && weights && loss && dz))
    rc = null_pointer(name);
  if (rc == RB_OK) rc = qr_check(name, B, A, N, kappa);
  if (rc == RB_OK) rc = copies_check(name, M, K);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)((M + 2 * K) * (N + A * N) + (2 * M + 2) * N + K * A + M) * sizeof(float);
  rc = smem_check(name, smem, "(M + 2K) * actions * atoms too large");
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_dueling_avg<2, VT>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_dueling_avg<4, VT>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = N <= 64 ? k_qr_dueling_avg<2, VT> : k_qr_dueling_avg<4, VT>;
  { ProfScope prof_(RB_K_C51_DUELING_AVG, (cudaStream_t)stream);
    k<<<B, QR_T, smem, (cudaStream_t)stream>>>(z_online, z_target, actions, returns, nonterminals, weights, kappa, gamma_n, B,
                                               A, N, M, K, loss, dz, theta_out, astar_out, eps); }
  return check_launch(name);
}
}

int rb_qr_dueling_avg_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                                float kappa, float gamma_n, int B, int M, int K, float* loss, float* dz, float* theta_out,
                                int64_t* astar_out, rb_stream_t stream) {
  return qr_dueling_avg_launch<false>("rb_qr_dueling_avg_loss_grad", z_online, z_target, actions_n, atoms, actions, returns,
                                      nonterminals, weights, kappa, gamma_n, B, M, K, loss, dz, theta_out, astar_out, 0.0f,
                                      stream);
}

int rb_qr_dueling_avg_vt_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                   const int64_t* actions, const float* returns, const float* nonterminals,
                                   const float* weights, float kappa, float gamma_n, int B, int M, int K, float* loss,
                                   float* dz, float* theta_out, int64_t* astar_out, float eps, rb_stream_t stream) {
  return qr_dueling_avg_launch<true>("rb_qr_dueling_avg_vt_loss_grad", z_online, z_target, actions_n, atoms, actions,
                                     returns, nonterminals, weights, kappa, gamma_n, B, M, K, loss, dz, theta_out, astar_out,
                                     eps, stream);
}

extern "C++" {
template <bool VT, bool RISK = false>
static int qr_launch(const char* name, const float* q_online_s, const float* q_online_ns, const float* q_target_ns,
                     const int64_t* actions, const float* returns, const float* nonterminals, const float* weights, float kappa,
                     float gamma_n, int B, int A, int N, float* loss, float* grad_q_online_s, float* theta_out,
                     int64_t* astar_out, float eps, rb_stream_t stream, int risk_kind = 0, float risk_eta = 0.0f) {
  int rc = VT ? vt_check(name, true, eps) : RB_OK;
  if (rc == RB_OK && !(q_online_s && q_online_ns && q_target_ns && actions && returns && nonterminals && weights && loss &&
                       grad_q_online_s))
    rc = null_pointer(name);
  if (rc == RB_OK) rc = qr_check(name, B, A, N, kappa);
  if (rc == RB_OK && RISK) rc = risk_check(name, risk_kind, risk_eta);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)(4 * N + A) * sizeof(float);
  rc = smem_check(name, smem, "too many actions");
  constexpr int F = RISK ? RISK_INST : 0;
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr<2 | F, VT>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr<4 | F, VT>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = N <= 64 ? k_qr<2 | F, VT> : k_qr<4 | F, VT>;
  { ProfScope prof_(RB_K_C51, (cudaStream_t)stream);
    k<<<B, QR_T, smem, (cudaStream_t)stream>>>(q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights,
                                               kappa, gamma_n, B, A, N, loss, grad_q_online_s, theta_out, astar_out, eps,
                                               risk_kind, risk_eta); }
  return check_launch(name);
}
}

int rb_qr_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                    const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n, int B,
                    int A, int N, float* loss, float* grad_q_online_s, float* theta_out, int64_t* astar_out,
                    rb_stream_t stream) {
  return qr_launch<false>("rb_qr_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights,
                          kappa, gamma_n, B, A, N, loss, grad_q_online_s, theta_out, astar_out, 0.0f, stream);
}

int rb_qr_vt_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                       const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n,
                       int B, int A, int N, float* loss, float* grad_q_online_s, float* theta_out, int64_t* astar_out,
                       float eps, rb_stream_t stream) {
  return qr_launch<true>("rb_qr_vt_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals, weights,
                         kappa, gamma_n, B, A, N, loss, grad_q_online_s, theta_out, astar_out, eps, stream);
}

int rb_qr_risk_loss_grad(const float* q_online_s, const float* q_online_ns, const float* q_target_ns, const int64_t* actions,
                         const float* returns, const float* nonterminals, const float* weights, float kappa, float gamma_n,
                         int B, int A, int N, float* loss, float* grad_q_online_s, float* theta_out, int64_t* astar_out,
                         int risk_kind, float risk_eta, rb_stream_t stream) {
  return qr_launch<false, true>("rb_qr_risk_loss_grad", q_online_s, q_online_ns, q_target_ns, actions, returns, nonterminals,
                                weights, kappa, gamma_n, B, A, N, loss, grad_q_online_s, theta_out, astar_out, 0.0f, stream,
                                risk_kind, risk_eta);
}

// The Munchausen entries' own refusals: alpha in [0, 1], tau finite and >= FLT_MIN (a normal fp32), l0 finite and < 0;
// NaN fails every comparison.
static int munchausen_check(const char* name, float alpha, float tau, float l0) {
  char msg[128];
  if (!(alpha >= 0.0f && alpha <= 1.0f)) {
    snprintf(msg, sizeof msg, "%s: alpha must be in [0, 1]", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (!(tau >= FLT_MIN) || !isfinite(tau)) {
    snprintf(msg, sizeof msg, "%s: temperature must be finite and a normal fp32 > 0", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (!(l0 < 0.0f) || !isfinite(l0)) {
    snprintf(msg, sizeof msg, "%s: clip must be finite and < 0", name);
    return fail(RB_ERR_INVAL, msg);
  }
  return RB_OK;
}

int rb_qr_dueling_munchausen_loss_grad(const float* z_online, const float* z_target, int actions_n, int atoms,
                                       const int64_t* actions, const float* returns, const float* nonterminals,
                                       const float* weights, float kappa, float gamma_n, float alpha, float temperature,
                                       float clip, int B, float* loss, float* dz, float* theta_out, float* bonus_out,
                                       rb_stream_t stream) {
  const char* name = "rb_qr_dueling_munchausen_loss_grad";
  const int N = atoms, A = actions_n;
  int rc = RB_OK;
  if (!(z_online && z_target && actions && returns && nonterminals && weights && loss && dz)) rc = null_pointer(name);
  if (rc == RB_OK) rc = qr_check(name, B, A, N, kappa);
  if (rc == RB_OK) rc = munchausen_check(name, alpha, temperature, clip);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)(3 * (N + A * N) + 4 * N + 4 * A) * sizeof(float);
  rc = smem_check(name, smem, "actions * atoms too large");
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_dueling_munchausen<2>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_dueling_munchausen<4>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = N <= 64 ? k_qr_dueling_munchausen<2> : k_qr_dueling_munchausen<4>;
  { ProfScope prof_(RB_K_C51_DUELING, (cudaStream_t)stream);
    k<<<B, QR_T, smem, (cudaStream_t)stream>>>(z_online, z_target, actions, returns, nonterminals, weights, kappa, gamma_n,
                                               alpha, temperature, clip, B, A, N, loss, dz, theta_out, bonus_out); }
  return check_launch(name);
}

int rb_qr_munchausen_loss_grad(const float* q_online_s, const float* q_target_s, const float* q_target_ns,
                               const int64_t* actions, const float* returns, const float* nonterminals, const float* weights,
                               float kappa, float gamma_n, float alpha, float temperature, float clip, int B, int A, int N,
                               float* loss, float* grad_q_online_s, float* theta_out, float* bonus_out, rb_stream_t stream) {
  const char* name = "rb_qr_munchausen_loss_grad";
  int rc = RB_OK;
  if (!(q_online_s && q_target_s && q_target_ns && actions && returns && nonterminals && weights && loss && grad_q_online_s))
    rc = null_pointer(name);
  if (rc == RB_OK) rc = qr_check(name, B, A, N, kappa);
  if (rc == RB_OK) rc = munchausen_check(name, alpha, temperature, clip);
  if (rc != RB_OK) return rc;
  const size_t smem = (size_t)(4 * N + 4 * A) * sizeof(float);
  rc = smem_check(name, smem, "too many actions");
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_munchausen<2>, smem, name);
  if (rc == RB_OK) rc = rbi::ensure_dynamic_smem(k_qr_munchausen<4>, smem, name);
  if (rc != RB_OK) return rc;
  const auto k = N <= 64 ? k_qr_munchausen<2> : k_qr_munchausen<4>;
  { ProfScope prof_(RB_K_C51, (cudaStream_t)stream);
    k<<<B, QR_T, smem, (cudaStream_t)stream>>>(q_online_s, q_target_s, q_target_ns, actions, returns, nonterminals, weights,
                                               kappa, gamma_n, alpha, temperature, clip, B, A, N, loss, grad_q_online_s,
                                               theta_out, bonus_out); }
  return check_launch(name);
}

extern "C++" {
template <bool VT, bool RISK = false>
static int qr_q_values_launch(const char* name, const float* z, int M, int actions, int atoms, float* q,
                              int64_t* best_action, float* best_q, float eps, rb_stream_t stream, int risk_kind = 0,
                              float risk_eta = 0.0f) {
  int rc = VT ? vt_check(name, true, eps) : RB_OK;
  if (rc != RB_OK) return rc;
  if (!z) return null_pointer(name);
  char msg[128];
  if (!q && !best_action && !best_q) {
    snprintf(msg, sizeof msg, "%s: no output requested", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (M <= 0 || actions <= 0 || atoms <= 1) {
    snprintf(msg, sizeof msg, "%s: M, actions > 0 and atoms > 1 are required", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (atoms > RB_MAX_ATOMS) {
    snprintf(msg, sizeof msg, "%s: atoms exceeds RB_MAX_ATOMS", name);
    return fail(RB_ERR_RANGE, msg);
  }
  rc = RISK ? risk_check(name, risk_kind, risk_eta) : RB_OK;
  if (rc != RB_OK) return rc;
  { ProfScope prof_(RB_K_Q_VALUES, (cudaStream_t)stream);
    k_qr_select<VT, RISK><<<(M + 3) / 4, 128, 0, (cudaStream_t)stream>>>(z, M, actions, atoms, q, best_action, best_q, eps,
                                                                         risk_kind, risk_eta); }
  return check_launch(name);
}
}

int rb_qr_q_values(const float* z, int M, int actions, int atoms, float* q, int64_t* best_action, float* best_q,
                   rb_stream_t stream) {
  return qr_q_values_launch<false>("rb_qr_q_values", z, M, actions, atoms, q, best_action, best_q, 0.0f, stream);
}

int rb_qr_vt_q_values(const float* z, int M, int actions, int atoms, float* q, int64_t* best_action, float* best_q,
                      float eps, rb_stream_t stream) {
  return qr_q_values_launch<true>("rb_qr_vt_q_values", z, M, actions, atoms, q, best_action, best_q, eps, stream);
}

int rb_qr_q_values_risk(const float* z, int M, int actions, int atoms, float* q, int64_t* best_action, float* best_q,
                        int risk_kind, float risk_eta, rb_stream_t stream) {
  return qr_q_values_launch<false, true>("rb_qr_q_values_risk", z, M, actions, atoms, q, best_action, best_q, 0.0f, stream,
                                         risk_kind, risk_eta);
}

static int stats_batch_check(const float* loss, const float* weights, const int64_t* actions, const float* m,
                             const float* support, const float* z, const float* q, int B, int A, int Z, const double* scratch) {
  if (!loss || !weights || !actions || !m || !support || !scratch) return fail(RB_ERR_INVAL, "rb_learn_stats: null pointer");
  if ((z == nullptr) == (q == nullptr)) return fail(RB_ERR_INVAL, "rb_learn_stats: give exactly one of z and q");
  if (B <= 0 || A <= 0 || Z <= 1) return fail(RB_ERR_INVAL, "rb_learn_stats: B, A > 0 and Z > 1 are required");
  if (Z > RB_MAX_ATOMS) return fail(RB_ERR_RANGE, "rb_learn_stats: Z exceeds RB_MAX_ATOMS");
  return RB_OK;
}

static int stats_record_check(const double* scratch, const float* grad_norm, const rb_learn_stats_record* ring, int capacity,
                              const int64_t* counter) {
  if (!scratch || !grad_norm || !ring || !counter) return fail(RB_ERR_INVAL, "rb_learn_stats: null pointer");
  if (capacity <= 0) return fail(RB_ERR_RANGE, "rb_learn_stats: the ring needs a positive capacity");
  return RB_OK;
}

int rb_learn_stats_scratch_elems(void) { return STATS_SCRATCH; }

int rb_learn_stats_batch(const float* loss, const float* weights, const int64_t* actions, const float* m, const float* support,
                         const float* z, const float* q, int B, int A, int Z, double* scratch, rb_stream_t stream) {
  int rc = stats_batch_check(loss, weights, actions, m, support, z, q, B, A, Z, scratch);
  if (rc != RB_OK) return rc;
  int ctas = (B + STATS_WARPS - 1) / STATS_WARPS;
  if (ctas > STATS_MAX_CTAS) ctas = STATS_MAX_CTAS;
  { ProfScope prof_(RB_K_LEARN_STATS, (cudaStream_t)stream);
    k_learn_stats_batch<<<ctas, STATS_THREADS, 0, (cudaStream_t)stream>>>(loss, weights, actions, m, support, z, q, B, A, Z,
                                                                          scratch); }
  return check_launch("rb_learn_stats_batch");
}

extern "C++" {
template <bool VT>
static int stats_batch_qr_launch(const char* name, const float* loss, const float* weights, const int64_t* actions,
                                 const float* theta, const float* z, const float* q, int B, int A, int N, double* scratch,
                                 float eps, rb_stream_t stream) {
  int rc = VT ? vt_check(name, true, eps) : RB_OK;
  if (rc != RB_OK) return rc;
  if (!loss || !weights || !actions || !theta || !scratch) return null_pointer(name);
  char msg[128];
  if ((z == nullptr) == (q == nullptr)) {
    snprintf(msg, sizeof msg, "%s: give exactly one of z and q", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (B <= 0 || A <= 0 || N <= 1) {
    snprintf(msg, sizeof msg, "%s: B, A > 0 and N > 1 are required", name);
    return fail(RB_ERR_INVAL, msg);
  }
  if (N > RB_MAX_ATOMS) {
    snprintf(msg, sizeof msg, "%s: N exceeds RB_MAX_ATOMS", name);
    return fail(RB_ERR_RANGE, msg);
  }
  int ctas = (B + STATS_WARPS - 1) / STATS_WARPS;
  if (ctas > STATS_MAX_CTAS) ctas = STATS_MAX_CTAS;
  { ProfScope prof_(RB_K_LEARN_STATS, (cudaStream_t)stream);
    k_learn_stats_batch_qr<VT><<<ctas, STATS_THREADS, 0, (cudaStream_t)stream>>>(loss, weights, actions, theta, z, q, B, A,
                                                                                 N, scratch, eps); }
  return check_launch(name);
}
}

int rb_learn_stats_batch_qr(const float* loss, const float* weights, const int64_t* actions, const float* theta, const float* z,
                            const float* q, int B, int A, int N, double* scratch, rb_stream_t stream) {
  return stats_batch_qr_launch<false>("rb_learn_stats_batch_qr", loss, weights, actions, theta, z, q, B, A, N, scratch, 0.0f,
                                      stream);
}

int rb_learn_stats_batch_qr_vt(const float* loss, const float* weights, const int64_t* actions, const float* theta,
                               const float* z, const float* q, int B, int A, int N, double* scratch, float eps,
                               rb_stream_t stream) {
  return stats_batch_qr_launch<true>("rb_learn_stats_batch_qr_vt", loss, weights, actions, theta, z, q, B, A, N, scratch, eps,
                                     stream);
}

int rb_learn_stats_write(const double* scratch, const float* grad_norm, const int32_t* gate, float max_norm,
                         rb_learn_stats_record* ring, int capacity, int64_t* counter, rb_stream_t stream) {
  int rc = stats_record_check(scratch, grad_norm, ring, capacity, counter);
  if (rc != RB_OK) return rc;
  { ProfScope prof_(RB_K_LEARN_STATS, (cudaStream_t)stream);
    k_learn_stats_record<<<1, 1, 0, (cudaStream_t)stream>>>(scratch, grad_norm, gate, max_norm, ring, capacity, counter); }
  return check_launch("rb_learn_stats_write");
}

int rb_learn_stats(const float* loss, const float* weights, const int64_t* actions, const float* m, const float* support,
                   const float* z, const float* q, int B, int A, int Z, const float* grad_norm, const int32_t* gate,
                   float max_norm, double* scratch, rb_learn_stats_record* ring, int capacity, int64_t* counter,
                   rb_stream_t stream) {
  int rc = stats_batch_check(loss, weights, actions, m, support, z, q, B, A, Z, scratch);
  if (rc == RB_OK) rc = stats_record_check(scratch, grad_norm, ring, capacity, counter);
  if (rc != RB_OK) return rc;
  rc = rb_learn_stats_batch(loss, weights, actions, m, support, z, q, B, A, Z, scratch, stream);
  if (rc != RB_OK) return rc;
  return rb_learn_stats_write(scratch, grad_norm, gate, max_norm, ring, capacity, counter, stream);
}

int rb_noisy_compose(const float* mu, const float* sigma, const float* eps, int64_t count, float* out, rb_stream_t stream) {
  if (!mu || !sigma || !eps || !out) return fail(RB_ERR_INVAL, "rb_noisy_compose: null pointer");
  if (count <= 0) return fail(RB_ERR_INVAL, "rb_noisy_compose: count must be positive");
  int64_t ctas = (count / 4 + 255) / 256;
  if (ctas < 1) ctas = 1;
  if (ctas > rbi::SM_COUNT * 8) ctas = rbi::SM_COUNT * 8;
  { ProfScope prof_(RB_K_NOISY_COMPOSE, (cudaStream_t)stream);
    k_noisy_compose<<<(int)ctas, 256, 0, (cudaStream_t)stream>>>(mu, sigma, eps, count, out); }
  return check_launch("rb_noisy_compose");
}

int rb_clip_adam_scratch_elems(void) { return ADAM_MAX_CTAS + 1; }  // partial sums + one ticket word (zero-initialised by the caller)

int rb_clip_adam(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t P, float grad_scale,
                 float max_norm, float lr, float beta1, float beta2, float eps, int64_t* step_count, double* partial_sums,
                 float* norm_out, const int32_t* gate, rb_stream_t stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || !step_count || !partial_sums)
    return fail(RB_ERR_INVAL, "rb_clip_adam: null pointer");
  if (P <= 0) return fail(RB_ERR_INVAL, "rb_clip_adam: P must be positive");
  const int ctas = adam_ctas(P);
  { ProfScope prof_(RB_K_SQNORM, (cudaStream_t)stream);
    k_sqnorm<<<ctas, ADAM_THREADS, 0, (cudaStream_t)stream>>>(grad, P, grad_scale, partial_sums); }
  int rc = check_launch("rb_clip_adam(norm)");
  if (rc != RB_OK) return rc;
  { ProfScope prof_(RB_K_CLIP_ADAM, (cudaStream_t)stream);
    k_clip_adam<<<ctas, ADAM_THREADS, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, P, grad_scale, max_norm, lr,
                                                               beta1, beta2, eps, step_count, partial_sums, ctas, norm_out,
                                                               reinterpret_cast<unsigned int*>(partial_sums + ADAM_MAX_CTAS), gate); }
  return check_launch("rb_clip_adam");
}

int rb_clip_adamw(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t P, float grad_scale,
                  float max_norm, float lr, float beta1, float beta2, float eps, const rb_adam_group* groups, int n_groups,
                  int64_t* step_count, int64_t* group_steps, double* partial_sums, float* norm_out, const int32_t* gate,
                  rb_stream_t stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq || !groups || !step_count || !group_steps || !partial_sums)
    return fail(RB_ERR_INVAL, "rb_clip_adamw: null pointer");
  if (P <= 0) return fail(RB_ERR_INVAL, "rb_clip_adamw: P must be positive");
  if (n_groups < 1 || n_groups > RB_MAX_ADAM_GROUPS)
    return fail(RB_ERR_RANGE, "rb_clip_adamw: n_groups outside [1, RB_MAX_ADAM_GROUPS]");
  AdamGroupPlan plan;
  memset(&plan, 0, sizeof(plan));
  plan.n = n_groups;
  int64_t end = 0;
  for (int k = 0; k < n_groups; ++k) {
    const rb_adam_group& g = groups[k];
    if (g.begin != end || g.end <= g.begin || g.end > P)
      return fail(RB_ERR_RANGE, "rb_clip_adamw: groups must tile [0, P) in order, each non-empty");
    if (g.begin % 4) return fail(RB_ERR_RANGE, "rb_clip_adamw: a group must begin on a multiple of 4");
    int rc = rbi::adamw_decay_check(lr, g.weight_decay,"rb_clip_adamw: weight_decay must be finite, >= 0 and lr * weight_decay < 1");
    if (rc != RB_OK) return rc;
    plan.g[k] = g;
    end = g.end;
  }
  if (end != P) return fail(RB_ERR_RANGE, "rb_clip_adamw: groups must tile [0, P) in order, each non-empty");
  const int ctas = adam_ctas(P);
  { ProfScope prof_(RB_K_SQNORM, (cudaStream_t)stream);
    k_sqnorm<<<ctas, ADAM_THREADS, 0, (cudaStream_t)stream>>>(grad, P, grad_scale, partial_sums); }
  int rc = check_launch("rb_clip_adamw(norm)");
  if (rc != RB_OK) return rc;
  { ProfScope prof_(RB_K_CLIP_ADAM, (cudaStream_t)stream);
    k_clip_adamw<<<ctas, ADAM_THREADS, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, P, grad_scale, max_norm,
                                                                lr, beta1, beta2, eps, step_count, partial_sums, ctas,
                                                                norm_out,
                                                                reinterpret_cast<unsigned int*>(partial_sums + ADAM_MAX_CTAS),
                                                                gate, plan, group_steps); }
  return check_launch("rb_clip_adamw");
}

int rb_target_ema(float* target, const float* param, int64_t n, float tau, const int32_t* gate, rb_stream_t stream) {
  if (!target || !param) return fail(RB_ERR_INVAL, "rb_target_ema: null pointer");
  if (n < 0) return fail(RB_ERR_INVAL, "rb_target_ema: n must not be negative");
  if (!(tau > 0.0f && tau <= 1.0f)) return fail(RB_ERR_RANGE, "rb_target_ema: tau outside (0, 1]");
  const uintptr_t t0 = (uintptr_t)target, p0 = (uintptr_t)param, bytes = (uintptr_t)n * sizeof(float);
  if (n > 0 && t0 < p0 + bytes && p0 < t0 + bytes) return fail(RB_ERR_INVAL, "rb_target_ema: target and param overlap");
  if (n == 0) return RB_OK;
  const int ctas = adam_ctas(n);
  { ProfScope prof_(RB_K_TARGET_EMA, (cudaStream_t)stream);
    k_target_ema<<<ctas, ADAM_THREADS, 0, (cudaStream_t)stream>>>(target, param, n, tau, gate); }
  return check_launch("rb_target_ema");
}

int rb_param_reset(float* param, int64_t n, const rb_reset_segment* segs, int n_segs, uint64_t seed, uint64_t reset_index,
                   rb_stream_t stream) {
  if (!param || !segs) return fail(RB_ERR_INVAL, "rb_param_reset: null pointer");
  if (n_segs < 1 || n_segs > RB_MAX_RESET_SEGMENTS)
    return fail(RB_ERR_RANGE, "rb_param_reset: n_segs outside [1, RB_MAX_RESET_SEGMENTS]");
  ResetPlan plan;
  memset(&plan, 0, sizeof(plan));
  int64_t end = 0, widest = 0;
  for (int i = 0; i < n_segs; ++i) {
    const rb_reset_segment& s = segs[i];
    if (s.count <= 0 || s.offset < end || s.offset > n - s.count)
      return fail(RB_ERR_RANGE, "rb_param_reset: segment empty, outside [0, n), unsorted or overlapping");
    if (!(s.bound >= 0.0f && s.bound <= FLT_MAX) || !(s.constant >= 0.0f && s.constant <= FLT_MAX))
      return fail(RB_ERR_RANGE, "rb_param_reset: bound and constant must be finite and non-negative");
    if (!(s.alpha >= 0.0f && s.alpha <= 1.0f)) return fail(RB_ERR_RANGE, "rb_param_reset: alpha outside [0, 1]");
    plan.seg[i] = s;
    end = s.offset + s.count;
    const int64_t quads = ((end - 1) >> 2) - (s.offset >> 2) + 1;
    if (quads > widest) widest = quads;
  }
  int64_t ctas = (widest + RESET_THREADS - 1) / RESET_THREADS;
  if (ctas > rbi::SM_COUNT * 4) ctas = rbi::SM_COUNT * 4;
  dim3 grid((unsigned)ctas, (unsigned)n_segs);
  { ProfScope prof_(RB_K_PARAM_RESET, (cudaStream_t)stream);
    k_param_reset<<<grid, RESET_THREADS, 0, (cudaStream_t)stream>>>(param, plan, seed, reset_index); }
  return check_launch("rb_param_reset");
}

int rb_neuron_scores(const float* act, int R, int C, int HW, double* sums, rb_stream_t stream) {
  if (!act || !sums) return fail(RB_ERR_INVAL, "rb_neuron_scores: null pointer");
  if (R <= 0 || C <= 0 || HW <= 0) return fail(RB_ERR_INVAL, "rb_neuron_scores: R, C and HW must be positive");
  k_neuron_scores<<<C, REDO_THREADS, 0, (cudaStream_t)stream>>>(act, R, C, HW, sums);
  return check_launch("rb_neuron_scores");
}

int rb_redo_mask(const double* sums, const rb_redo_scored* layers, int n_layers, float tau, uint8_t* mask, int64_t* record,
                 int64_t pass_index, rb_stream_t stream) {
  if (!sums || !layers || !mask || !record) return fail(RB_ERR_INVAL, "rb_redo_mask: null pointer");
  if (n_layers < 1 || n_layers > RB_MAX_REDO_LAYERS)
    return fail(RB_ERR_RANGE, "rb_redo_mask: n_layers outside [1, RB_MAX_REDO_LAYERS]");
  if (!(tau >= 0.0f && tau <= 1.0f)) return fail(RB_ERR_RANGE, "rb_redo_mask: tau outside [0, 1]");
  if (pass_index < 0) return fail(RB_ERR_RANGE, "rb_redo_mask: pass_index must not be negative");
  RedoMaskPlan plan;
  memset(&plan, 0, sizeof(plan));
  plan.n_layers = n_layers;
  int64_t end = 0;
  for (int l = 0; l < n_layers; ++l) {
    const rb_redo_scored& s = layers[l];
    if (s.neurons <= 0 || s.offset < end || (int64_t)s.offset + s.neurons > INT32_MAX)
      return fail(RB_ERR_RANGE, "rb_redo_mask: layer empty, unsorted or overlapping");
    if (!(s.count >= 1.0 && s.count <= 9007199254740992.0))
      return fail(RB_ERR_RANGE, "rb_redo_mask: count must be in [1, 2^53]");
    plan.offset[l] = s.offset; plan.neurons[l] = s.neurons; plan.count[l] = s.count;
    end = (int64_t)s.offset + s.neurons;
  }
  k_redo_mask<<<n_layers, REDO_THREADS, 0, (cudaStream_t)stream>>>(sums, plan, tau, mask, (long long*)record,
                                                                   (long long)pass_index);
  return check_launch("rb_redo_mask");
}

int rb_redo_recycle(float* param, float* exp_avg, float* exp_avg_sq, int64_t n, const rb_redo_layer* layers, int n_layers,
                    const uint8_t* mask, uint64_t seed, uint64_t pass_index, rb_stream_t stream) {
  if (!param || !exp_avg || !exp_avg_sq || !layers || !mask) return fail(RB_ERR_INVAL, "rb_redo_recycle: null pointer");
  if (n_layers < 1 || n_layers > RB_MAX_REDO_LAYERS)
    return fail(RB_ERR_RANGE, "rb_redo_recycle: n_layers outside [1, RB_MAX_REDO_LAYERS]");
  RedoPlan plan;
  memset(&plan, 0, sizeof(plan));
  // extents [begin, end) of every incoming block and of every outgoing block: each kind must be disjoint within itself (an
  // incoming block may be another layer's outgoing block: the kernel gives such an element to the zeroing writer)
  int64_t in_ext[RB_MAX_REDO_LAYERS * RB_MAX_REDO_BLOCKS][2], out_ext[RB_MAX_REDO_LAYERS * RB_MAX_REDO_BLOCKS][2];
  int n_in = 0, n_out = 0, widest = 0;
  for (int l = 0; l < n_layers; ++l) {
    const rb_redo_layer& L = layers[l];
    if (L.neurons <= 0 || L.mask_offset < 0 || (int64_t)L.mask_offset + L.neurons > INT32_MAX)
      return fail(RB_ERR_RANGE, "rb_redo_recycle: layer empty or mask range invalid");
    if (L.n_in < 1 || L.n_in > RB_MAX_REDO_BLOCKS || L.n_out < 0 || L.n_out > RB_MAX_REDO_BLOCKS)
      return fail(RB_ERR_RANGE, "rb_redo_recycle: n_in outside [1, RB_MAX_REDO_BLOCKS] or n_out outside [0, RB_MAX_REDO_BLOCKS]");
    for (int b = 0; b < L.n_in; ++b) {
      const rb_redo_in& in = L.in[b];
      if (in.per_neuron <= 0 || in.offset < 0 || in.per_neuron > n / L.neurons || in.offset > n - in.per_neuron * L.neurons)
        return fail(RB_ERR_RANGE, "rb_redo_recycle: incoming block empty or outside [0, n)");
      if (!(in.bound >= 0.0f && in.bound <= FLT_MAX) || !(in.constant >= 0.0f && in.constant <= FLT_MAX))
        return fail(RB_ERR_RANGE, "rb_redo_recycle: bound and constant must be finite and non-negative");
      if (in.src_span < 0 || (in.src_span > 0 && in.per_neuron % in.src_span))
        return fail(RB_ERR_RANGE, "rb_redo_recycle: src_span must be 0 or divide per_neuron");
      if (in.src_span > 0) {   // the upstream mask range must be exactly one layer's
        bool found = false;
        for (int u = 0; u < n_layers; ++u)
          found = found || (u != l && layers[u].mask_offset == in.src_mask_offset &&
                            layers[u].neurons == in.per_neuron / in.src_span);
        if (!found) return fail(RB_ERR_RANGE, "rb_redo_recycle: src_mask_offset and src_span name no layer of the table");
      }
      in_ext[n_in][0] = in.offset; in_ext[n_in][1] = in.offset + in.per_neuron * L.neurons; ++n_in;
    }
    for (int b = 0; b < L.n_out; ++b) {
      const rb_redo_out& out = L.out[b];
      if (out.rows <= 0 || out.span <= 0 || out.offset < 0 || out.span > n / L.neurons ||
          out.row_stride < out.span * L.neurons || out.row_stride > n || out.rows > n / out.row_stride + 1 ||
          out.offset > n - ((out.rows - 1) * out.row_stride + out.span * L.neurons))
        return fail(RB_ERR_RANGE, "rb_redo_recycle: outgoing block empty, rows overlapping or outside [0, n)");
      out_ext[n_out][0] = out.offset;
      out_ext[n_out][1] = out.offset + (out.rows - 1) * out.row_stride + out.span * L.neurons; ++n_out;
    }
    plan.layer[l] = L;
    if (L.neurons > widest) widest = L.neurons;
  }
  for (int a = 0; a < n_layers; ++a)
    for (int b = a + 1; b < n_layers; ++b)
      if (layers[a].mask_offset < layers[b].mask_offset + layers[b].neurons &&
          layers[b].mask_offset < layers[a].mask_offset + layers[a].neurons)
        return fail(RB_ERR_RANGE, "rb_redo_recycle: mask ranges of two layers overlap");
  for (int a = 0; a < n_in; ++a)
    for (int b = a + 1; b < n_in; ++b)
      if (in_ext[a][0] < in_ext[b][1] && in_ext[b][0] < in_ext[a][1])
        return fail(RB_ERR_RANGE, "rb_redo_recycle: incoming blocks overlap");
  for (int a = 0; a < n_out; ++a)
    for (int b = a + 1; b < n_out; ++b)
      if (out_ext[a][0] < out_ext[b][1] && out_ext[b][0] < out_ext[a][1])
        return fail(RB_ERR_RANGE, "rb_redo_recycle: outgoing blocks overlap");
  if (widest > 65535) return fail(RB_ERR_RANGE, "rb_redo_recycle: more than 65535 neurons in a layer");
  dim3 grid(REDO_NEURON_CTAS, (unsigned)widest, (unsigned)n_layers);
  k_redo_recycle<<<grid, REDO_THREADS, 0, (cudaStream_t)stream>>>(param, exp_avg, exp_avg_sq, plan, mask, seed, pass_index);
  return check_launch("rb_redo_recycle");
}

}  // extern "C"
