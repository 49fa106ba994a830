// rb_peer.cu -- fused gradient exchange + optimiser over NVLink peer memory (multi-GPU learners, sm_90a).
//
// Replaces  ncclAllReduce(flat_grad) ; k_sqnorm ; k_clip_adam (replicated on every rank)  by
//   k_peer_reduce : reduce-scatter done with peer LOADS -- rank r sums its 1/W part of a SEGMENT of every rank's
//                   gradient buffer (fixed rank order: deterministic), keeps the sum locally and accumulates the squared
//                   norm of what it owns.  The flat buffer is exchanged as up to two segments so that the noisy-head
//                   segment (99 % of the bytes, final after k_head_bwd1) crosses NVLink on a side stream WHILE the conv
//                   backward is still running; the small conv segment follows when that is done;
//   k_peer_adam   : clip coefficient from the W per-rank partial norms, Adam on the owned parts only (the moments are
//                   sharded: 1/W of the optimiser traffic per GPU), all-gather done with peer STORES -- the updated
//                   parameters are written straight into every rank's flat parameter buffer;
//   k_peer_fence  : waits until every rank's parts have landed here (and therefore every rank is done reading this
//                   rank's gradients), so plain stream order protects the next forward / backward.
// Cross-GPU ordering uses monotonically increasing epoch flags in peer-visible memory (st.release.sys /
// ld.acquire.sys); nothing spins on the host.  All buffers handed in as `peer_*[rank]` pointers must be mapped on
// every GPU (torch symmetric memory in rainbow_b200/peer.py).
//
// tests/test_gpu_peer_f64.py checks every stage against a float64 reference, W = 1..8 ranks emulated on one GPU.

#include <cuda_runtime.h>
#include <stdint.h>

#include "rainbow_b200.h"
#include "rb_internal.cuh"

namespace {

constexpr int PEER_THREADS = 256;
constexpr int PEER_MAX_CTAS = 592;   // grid-stride cap; the scratch holds one partial per CTA
constexpr int PEER_SEGS = 2;

// flag blocks of one rank (uint64[4][W]): [0] / [1] = "rank q's gradients of segment 0 / 1 are complete",
// [2] = "rank q's partial squared norm is published", [3] = "rank q's parameter parts have been stored here"
constexpr int FLAG_NORM = 2, FLAG_PARAM = 3;

struct PeerBufs {
  const float* grad[RB_MAX_PEERS];   // every rank's flat gradient buffer (read)
  float* param[RB_MAX_PEERS];        // every rank's flat parameter buffer (written)
  uint64_t* flags[RB_MAX_PEERS];     // every rank's flag block
  double* norms[RB_MAX_PEERS];       // every rank's norm block: double[W]
  int world, rank;
};

struct Segs {   // segment s covers flat elements [begin[s], begin[s] + len[s]); rank r owns part r of len[s] / W elements
  int64_t begin[PEER_SEGS], len[PEER_SEGS];
  int n;
};

__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// one thread per CTA waits until the W local flags of `block` reach `epoch`, then the CTA proceeds
__device__ __forceinline__ void wait_flags(const uint64_t* local_flags, int block, int world, uint64_t epoch) {
  if (threadIdx.x == 0) {
    for (int q = 0; q < world; ++q)
      while (ld_acquire_sys(local_flags + block * world + q) < epoch) __nanosleep(64);
  }
  __syncthreads();
}

// Phase 1 (per segment): announce "my gradients of this segment are complete" to every rank, wait for everybody's
// announcement, then reduce the owned part over all ranks with peer loads.  Grid-stride over the part; per-CTA partial of
// the squared norm, summed in CTA order by the last CTA to finish (deterministic) into seg_norm[seg].
__global__ void __launch_bounds__(PEER_THREADS)
k_peer_reduce(const __grid_constant__ PeerBufs pb, const uint64_t* __restrict__ epoch_ptr, int seg, int64_t seg_begin,
              int64_t part, float grad_scale, float* __restrict__ gred, double* __restrict__ cta_partial,
              unsigned int* __restrict__ ticket, double* __restrict__ seg_norm) {
  __shared__ double s_red[PEER_THREADS / 32];
  const uint64_t epoch = *epoch_ptr + 1;
  const int W = pb.world, r = pb.rank;
  if (blockIdx.x == 0 && threadIdx.x < W) st_release_sys(pb.flags[threadIdx.x] + seg * W + r, epoch);
  wait_flags(pb.flags[r], seg, W, epoch);
  const int64_t base = seg_begin + (int64_t)r * part;
  double acc = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n4 = part >> 2;
  constexpr int UN = 4;   // grid-stride iterations whose peer loads are all issued before any is consumed (few CTAs, deep queues)
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < n4; i0 += stride * UN) {
    float4 g[UN][RB_MAX_PEERS];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int64_t i = i0 + u * stride;
#pragma unroll
      for (int p = 0; p < RB_MAX_PEERS; ++p)
        if (p < W && i < n4) g[u][p] = *reinterpret_cast<const float4*>(pb.grad[p] + base + 4 * i);
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < n4) {
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int p = 0; p < RB_MAX_PEERS; ++p)   // fixed rank order: deterministic
          if (p < W) { s.x += g[u][p].x; s.y += g[u][p].y; s.z += g[u][p].z; s.w += g[u][p].w; }
        s.x *= grad_scale; s.y *= grad_scale; s.z *= grad_scale; s.w *= grad_scale;
        reinterpret_cast<float4*>(gred)[i] = s;
        acc += (double)s.x * s.x + (double)s.y * s.y + (double)s.z * s.z + (double)s.w * s.w;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < PEER_THREADS / 32; ++w) t += s_red[w];
    cta_partial[blockIdx.x] = t;
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) {  // last CTA: squared norm of this rank's part of the segment
      *ticket = 0u;
      __threadfence();
      double n2 = 0.0;
      for (unsigned int c = 0; c < gridDim.x; ++c) n2 += __ldcg(cta_partial + c);
      seg_norm[seg] = n2;
    }
  }
}

// Phase 2: publish this rank's partial norm, global norm -> clip -> Adam on the owned parts -> parameter parts stored
// into every rank's buffer.
// one 16-byte store that the NVSwitch replicates into every rank's copy of the buffer (NVLS multicast mapping)
__device__ __forceinline__ void multimem_st4(float* mc_addr, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

struct SegDecay {   // rb_peer_adamw_gather: lambda of each segment
  float wd[PEER_SEGS];
};

// GROUPS (rb_peer_adamw_gather): the bias corrections of segment s come from seg_steps[s] + 1 instead of step_count + 1,
// and p = p * fl32(1 - lr lambda_s), rounded on its own, before the moments; the last CTA advances seg_steps too.
template <bool GROUPS>
__device__ __forceinline__ void
peer_adam_body(const PeerBufs& pb, const Segs& sg, uint64_t* __restrict__ epoch_ptr, const float* __restrict__ gred,
               float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, const double* __restrict__ seg_norm,
               float max_norm, float lr, float b1, float b2, float eps, int64_t* __restrict__ step_count,
               float* __restrict__ norm_out, unsigned int* __restrict__ ticket, float* __restrict__ mc_param,
               const SegDecay* decay, int64_t* __restrict__ seg_steps) {
  const uint64_t epoch = *epoch_ptr + 1;
  const int W = pb.world, r = pb.rank;
  if (blockIdx.x == 0 && threadIdx.x < W) {   // this rank's share of the squared norm, to every rank
    double mine = 0.0;
    for (int s = 0; s < sg.n; ++s) mine += seg_norm[s];
    const int q = threadIdx.x;
    pb.norms[q][r] = mine;
    __threadfence_system();
    st_release_sys(pb.flags[q] + FLAG_NORM * W + r, epoch);
  }
  wait_flags(pb.flags[r], FLAG_NORM, W, epoch);
  double n2 = 0.0;
  for (int q = 0; q < W; ++q) n2 += pb.norms[r][q];  // same order on every rank -> identical coefficient everywhere
  const float norm = (float)sqrt(n2);
  const float coef = fminf(max_norm / (norm + 1e-6f), 1.0f);
  if (norm_out && blockIdx.x == 0 && threadIdx.x == 0) *norm_out = norm;
  const int64_t step = *step_count + 1;
  float step_size, inv_bc2_sqrt, d = 1.0f;
  if constexpr (!GROUPS) {
    step_size = (float)((double)lr / (1.0 - pow((double)b1, (double)step)));
    inv_bc2_sqrt = (float)(1.0 / sqrt(1.0 - pow((double)b2, (double)step)));
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t shard_off = 0;   // offset of the segment's part inside gred / exp_avg / exp_avg_sq
  for (int s = 0; s < sg.n; ++s) {
    const int64_t part = sg.len[s] / W, base = sg.begin[s] + (int64_t)r * part;
    const float* my_param = pb.param[r] + base;
    if constexpr (GROUPS) {
      const int64_t t = seg_steps[s] + 1;
      step_size = (float)((double)lr / (1.0 - pow((double)b1, (double)t)));
      inv_bc2_sqrt = (float)(1.0 / sqrt(1.0 - pow((double)b2, (double)t)));
      d = (float)(1.0 - (double)lr * (double)decay->wd[s]);
    }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (part >> 2); i += stride) {
      float4 p = reinterpret_cast<const float4*>(my_param)[i];
      const float4 g = reinterpret_cast<const float4*>(gred + shard_off)[i];
      float4 m = reinterpret_cast<float4*>(exp_avg + shard_off)[i], v = reinterpret_cast<float4*>(exp_avg_sq + shard_off)[i];
      float* pp = &p.x; const float* gg = &g.x; float* mm = &m.x; float* vv = &v.x;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if constexpr (GROUPS) pp[c] = __fmul_rn(pp[c], d);
        const float gc = gg[c] * coef;
        mm[c] = fmaf(gc - mm[c], 1.0f - b1, mm[c]);
        vv[c] = fmaf(vv[c], b2, (1.0f - b2) * gc * gc);
        pp[c] = pp[c] - step_size * (mm[c] / (sqrtf(vv[c]) * inv_bc2_sqrt + eps));
      }
      reinterpret_cast<float4*>(exp_avg + shard_off)[i] = m;
      reinterpret_cast<float4*>(exp_avg_sq + shard_off)[i] = v;
      if (mc_param) {   // all-gather in the switch: ONE multicast store lands in every rank's parameter buffer
        multimem_st4(mc_param + base + 4 * i, p);
      } else {
#pragma unroll
        for (int q = 0; q < RB_MAX_PEERS; ++q)   // all-gather by peer stores
          if (q < W) reinterpret_cast<float4*>(pb.param[q] + base)[i] = p;
      }
    }
    shard_off += part;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) {  // last CTA: this rank's parts are in place on every rank
      *ticket = 0u;
      __threadfence_system();
      for (int q = 0; q < W; ++q) st_release_sys(pb.flags[q] + FLAG_PARAM * W + r, epoch);
      *step_count = step;
      if constexpr (GROUPS) {
        for (int s = 0; s < sg.n; ++s) seg_steps[s] += 1;   // every CTA read them before its ticket
      }
    }
  }
}

__global__ void __launch_bounds__(PEER_THREADS)
k_peer_adam(const __grid_constant__ PeerBufs pb, const __grid_constant__ Segs sg, uint64_t* __restrict__ epoch_ptr,
            const float* __restrict__ gred, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
            const double* __restrict__ seg_norm, float max_norm, float lr, float b1, float b2, float eps,
            int64_t* __restrict__ step_count, float* __restrict__ norm_out, unsigned int* __restrict__ ticket,
            float* __restrict__ mc_param) {
  peer_adam_body<false>(pb, sg, epoch_ptr, gred, exp_avg, exp_avg_sq, seg_norm, max_norm, lr, b1, b2, eps, step_count,
                        norm_out, ticket, mc_param, nullptr, nullptr);
}

__global__ void __launch_bounds__(PEER_THREADS)
k_peer_adamw(const __grid_constant__ PeerBufs pb, const __grid_constant__ Segs sg, uint64_t* __restrict__ epoch_ptr,
             const float* __restrict__ gred, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
             const double* __restrict__ seg_norm, float max_norm, float lr, float b1, float b2, float eps,
             int64_t* __restrict__ step_count, float* __restrict__ norm_out, unsigned int* __restrict__ ticket,
             float* __restrict__ mc_param, const __grid_constant__ SegDecay decay, int64_t* __restrict__ seg_steps) {
  peer_adam_body<true>(pb, sg, epoch_ptr, gred, exp_avg, exp_avg_sq, seg_norm, max_norm, lr, b1, b2, eps, step_count,
                       norm_out, ticket, mc_param, &decay, seg_steps);
}

// Phase 3: every rank's parts have arrived here (so every rank has also finished reading our gradients); advance the epoch.
__global__ void k_peer_fence(const __grid_constant__ PeerBufs pb, uint64_t* __restrict__ epoch_ptr) {
  const uint64_t epoch = *epoch_ptr + 1;
  wait_flags(pb.flags[pb.rank], FLAG_PARAM, pb.world, epoch);
  if (threadIdx.x == 0) *epoch_ptr = epoch;
}

int fill_bufs(PeerBufs* pb, const float* const* peer_grad, float* const* peer_param, uint64_t* const* peer_flags,
              double* const* peer_norms, int world, int rank, const char* who) {
  if (!peer_flags || (!peer_grad && !peer_param)) return rbi::fail(RB_ERR_INVAL, who);
  if (world < 1 || world > RB_MAX_PEERS || rank < 0 || rank >= world) return rbi::fail(RB_ERR_RANGE, "rb_peer: bad world/rank");
  pb->world = world;
  pb->rank = rank;
  for (int q = 0; q < RB_MAX_PEERS; ++q) {
    const bool in = q < world;
    if (in && (!peer_flags[q] || (peer_grad && !peer_grad[q]) || (peer_param && !peer_param[q]) || (peer_norms && !peer_norms[q])))
      return rbi::fail(RB_ERR_INVAL, "rb_peer: null peer buffer");
    pb->grad[q] = (in && peer_grad) ? peer_grad[q] : nullptr;
    pb->param[q] = (in && peer_param) ? peer_param[q] : nullptr;
    pb->flags[q] = in ? peer_flags[q] : nullptr;
    pb->norms[q] = (in && peer_norms) ? peer_norms[q] : nullptr;
  }
  return RB_OK;
}

int ctas_for(int64_t part) {
  int64_t want = (part / 4 + PEER_THREADS - 1) / PEER_THREADS;
  return (int)(want < 1 ? 1 : (want > PEER_MAX_CTAS ? PEER_MAX_CTAS : want));
}
// The reduce-scatter runs BESIDE the conv backward, whose library kernels (dgrad_engine: 512-thread CTAs that take a whole
// SM's register file) cannot start on an SM that holds even one of our CTAs: one CTA per SM would make the dgrad chain
// wait for the reduce to finish.  64 CTAs x 256 threads x 4 x W 16-byte peer loads in flight (2 MB at W = 2) keep NVLink
// busy and leave the other SMs to the backward.
int reduce_ctas_for(int64_t part) {
  const int c = ctas_for(part);
  return c > 64 ? 64 : c;
}

// scratch layout: per segment PEER_MAX_CTAS doubles of CTA partials, then double seg_norm[PEER_SEGS], then tickets
double* scratch_partials(void* scratch, int seg) { return reinterpret_cast<double*>(scratch) + (size_t)seg * PEER_MAX_CTAS; }
double* scratch_seg_norm(void* scratch) { return reinterpret_cast<double*>(scratch) + (size_t)PEER_SEGS * PEER_MAX_CTAS; }
unsigned int* scratch_tickets(void* scratch) { return reinterpret_cast<unsigned int*>(scratch_seg_norm(scratch) + PEER_SEGS); }

}  // namespace

extern "C" {

int rb_peer_scratch_bytes(void) { return (int)((PEER_SEGS * PEER_MAX_CTAS + PEER_SEGS) * sizeof(double) + 64); }

int rb_peer_reduce(const float* const* peer_grad, uint64_t* const* peer_flags, int world, int rank, int seg, int64_t seg_begin,
                   int64_t seg_len, float grad_scale, float* gred_part, const uint64_t* epoch, void* scratch,
                   rb_stream_t stream) {
  if (!peer_grad || !gred_part || !epoch || !scratch) return rbi::fail(RB_ERR_INVAL, "rb_peer_reduce: null pointer");
  if (seg < 0 || seg >= PEER_SEGS) return rbi::fail(RB_ERR_RANGE, "rb_peer_reduce: segment id must be 0 or 1");
  PeerBufs pb;
  int rc = fill_bufs(&pb, peer_grad, nullptr, peer_flags, nullptr, world, rank, "rb_peer_reduce: null pointer");
  if (rc != RB_OK) return rc;
  if (seg_begin < 0 || seg_len <= 0 || seg_len % (4 * (int64_t)world) || seg_begin % 4)
    return rbi::fail(RB_ERR_INVAL, "rb_peer_reduce: segment must start on a multiple of 4 and hold a multiple of 4 * world elements");
  const int64_t part = seg_len / world;
  k_peer_reduce<<<reduce_ctas_for(part), PEER_THREADS, 0, (cudaStream_t)stream>>>(pb, epoch, seg, seg_begin, part, grad_scale, gred_part,
                                                                         scratch_partials(scratch, seg),
                                                                         scratch_tickets(scratch) + seg, scratch_seg_norm(scratch));
  return rbi::check_launch("rb_peer_reduce");
}

// The checks rb_peer_adam_gather and rb_peer_adamw_gather share, and the launch parameters they derive.
static int peer_gather_setup(PeerBufs* pb, Segs* sg, int64_t* biggest, float* const* peer_param, uint64_t* const* peer_flags,
                             double* const* peer_norms, int world, int rank, int n_seg, const int64_t* seg_begin,
                             const int64_t* seg_len, const float* gred, float* exp_avg, float* exp_avg_sq,
                             int64_t* step_count, uint64_t* epoch, void* scratch) {
  if (!peer_param || !peer_norms || !seg_begin || !seg_len || !gred || !exp_avg || !exp_avg_sq || !step_count || !epoch || !scratch)
    return rbi::fail(RB_ERR_INVAL, "rb_peer_adam_gather: null pointer");
  if (n_seg < 1 || n_seg > PEER_SEGS) return rbi::fail(RB_ERR_RANGE, "rb_peer_adam_gather: 1 or 2 segments");
  int rc = fill_bufs(pb, nullptr, peer_param, peer_flags, peer_norms, world, rank, "rb_peer_adam_gather: null pointer");
  if (rc != RB_OK) return rc;
  sg->n = n_seg;
  *biggest = 0;
  for (int s = 0; s < PEER_SEGS; ++s) {
    sg->begin[s] = s < n_seg ? seg_begin[s] : 0;
    sg->len[s] = s < n_seg ? seg_len[s] : 0;
    if (s < n_seg && (seg_begin[s] < 0 || seg_len[s] <= 0 || seg_len[s] % (4 * (int64_t)world) || seg_begin[s] % 4))
      return rbi::fail(RB_ERR_INVAL, "rb_peer_adam_gather: bad segment");
    if (sg->len[s] / world > *biggest) *biggest = sg->len[s] / world;
  }
  return RB_OK;
}

int rb_peer_adam_gather(float* const* peer_param, uint64_t* const* peer_flags, double* const* peer_norms, int world, int rank,
                        int n_seg, const int64_t* seg_begin, const int64_t* seg_len, const float* gred, float* exp_avg,
                        float* exp_avg_sq, float max_norm, float lr, float beta1, float beta2, float eps, int64_t* step_count,
                        uint64_t* epoch, void* scratch, float* norm_out, float* multicast_param, rb_stream_t stream) {
  PeerBufs pb;
  Segs sg;
  int64_t biggest;
  int rc = peer_gather_setup(&pb, &sg, &biggest, peer_param, peer_flags, peer_norms, world, rank, n_seg, seg_begin, seg_len,
                             gred, exp_avg, exp_avg_sq, step_count, epoch, scratch);
  if (rc != RB_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  k_peer_adam<<<ctas_for(biggest), PEER_THREADS, 0, st>>>(pb, sg, epoch, gred, exp_avg, exp_avg_sq, scratch_seg_norm(scratch), max_norm,
                                                        lr, beta1, beta2, eps, step_count, norm_out,
                                                        scratch_tickets(scratch) + PEER_SEGS, multicast_param);
  rc = rbi::check_launch("rb_peer_adam_gather(adam)");
  if (rc != RB_OK) return rc;
  k_peer_fence<<<1, 32, 0, st>>>(pb, epoch);
  return rbi::check_launch("rb_peer_adam_gather(fence)");
}

int rb_peer_adamw_gather(float* const* peer_param, uint64_t* const* peer_flags, double* const* peer_norms, int world, int rank,
                         int n_seg, const int64_t* seg_begin, const int64_t* seg_len, const float* seg_weight_decay,
                         const float* gred, float* exp_avg, float* exp_avg_sq, float max_norm, float lr, float beta1,
                         float beta2, float eps, int64_t* step_count, int64_t* seg_steps, uint64_t* epoch, void* scratch,
                         float* norm_out, float* multicast_param, rb_stream_t stream) {
  if (!seg_weight_decay || !seg_steps) return rbi::fail(RB_ERR_INVAL, "rb_peer_adamw_gather: null pointer");
  PeerBufs pb;
  Segs sg;
  int64_t biggest;
  int rc = peer_gather_setup(&pb, &sg, &biggest, peer_param, peer_flags, peer_norms, world, rank, n_seg, seg_begin, seg_len,
                             gred, exp_avg, exp_avg_sq, step_count, epoch, scratch);
  if (rc != RB_OK) return rc;
  SegDecay decay;
  for (int s = 0; s < PEER_SEGS; ++s) {
    decay.wd[s] = s < n_seg ? seg_weight_decay[s] : 0.0f;
    rc = rbi::adamw_decay_check(lr, decay.wd[s],
                                "rb_peer_adamw_gather: weight_decay must be finite, >= 0 and lr * weight_decay < 1");
    if (rc != RB_OK) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
  k_peer_adamw<<<ctas_for(biggest), PEER_THREADS, 0, st>>>(pb, sg, epoch, gred, exp_avg, exp_avg_sq, scratch_seg_norm(scratch),
                                                         max_norm, lr, beta1, beta2, eps, step_count, norm_out,
                                                         scratch_tickets(scratch) + PEER_SEGS, multicast_param, decay,
                                                         seg_steps);
  rc = rbi::check_launch("rb_peer_adamw_gather(adam)");
  if (rc != RB_OK) return rc;
  k_peer_fence<<<1, 32, 0, st>>>(pb, epoch);
  return rbi::check_launch("rb_peer_adamw_gather(fence)");
}

int rb_peer_clip_adam(const float* const* peer_grad, float* const* peer_param, uint64_t* const* peer_flags,
                      double* const* peer_norms, int world, int rank, int64_t P, float* gred, float* exp_avg,
                      float* exp_avg_sq, float grad_scale, float max_norm, float lr, float beta1, float beta2, float eps,
                      int64_t* step_count, uint64_t* epoch, void* scratch, float* norm_out, rb_stream_t stream) {
  if (P <= 0 || P % (4 * (int64_t)(world > 0 ? world : 1))) return rbi::fail(RB_ERR_INVAL, "rb_peer_clip_adam: P must be a multiple of 4 * world");
  int rc = rb_peer_reduce(peer_grad, peer_flags, world, rank, 0, 0, P, grad_scale, gred, epoch, scratch, stream);
  if (rc != RB_OK) return rc;
  const int64_t b = 0, l = P;
  return rb_peer_adam_gather(peer_param, peer_flags, peer_norms, world, rank, 1, &b, &l, gred, exp_avg, exp_avg_sq, max_norm, lr,
                             beta1, beta2, eps, step_count, epoch, scratch, norm_out, nullptr, stream);
}

}  // extern "C"
