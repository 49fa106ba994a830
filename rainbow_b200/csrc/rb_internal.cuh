// rb_internal.cuh -- helpers shared by the translation units of librainbow_b200.so (not installed).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "rainbow_b200.h"

namespace rbi {

// Streaming multiprocessors of the target GPU (H100 SXM).  Grid sizes and split-K factors are derived from it at compile
// time rather than queried, so that the summation order of split reductions -- and hence the results -- does not depend
// on the device a run happens to land on.
constexpr int SM_COUNT = 132;

// ---- error reporting (state lives in rb_kernels.cu) -------------------------------------------
char* err_buffer();  // thread-local, 256 bytes

inline int fail(int code, const char* what) {
  snprintf(err_buffer(), 256, "%s", what);
  return code;
}

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    snprintf(err_buffer(), 256, "%s: %s", what, cudaGetErrorString(e));
    return RB_ERR_CUDA;
  }
  return RB_OK;
}

// ---- AdamW's decoupled weight decay (rb_clip_adamw, rb_peer_adamw_gather) ---------------------
// lambda finite and >= 0, fl32(lr) fl32(lambda) < 1: the factor fl32(1 - lr lambda) the kernels multiply p by is in (0, 1]
inline int adamw_decay_check(float lr, float weight_decay, const char* who) {
  if (!(weight_decay >= 0.0f && weight_decay <= 3.402823466e38f) || !((double)lr * (double)weight_decay < 1.0))
    return fail(RB_ERR_RANGE, who);
  return RB_OK;
}

// ---- opt-in to more than 48 KB of dynamic shared memory, once per (device, kernel, size) ---------------
// cudaFuncSetAttribute is not a stream operation; calling it again and again (e.g. while a CUDA graph is being
// captured) is avoided by remembering the largest size already granted per device.
struct SmemGrant {
  const void* fn;
  int dev;
  size_t bytes;
};
SmemGrant* smem_grants();   // table of 256 entries, zero-initialised (defined in rb_kernels.cu)

template <typename Kernel>
inline int ensure_dynamic_smem(Kernel kernel, size_t bytes, const char* who) {
  if (bytes <= 48 * 1024) return RB_OK;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(RB_ERR_CUDA, who);
  const void* fn = reinterpret_cast<const void*>(kernel);
  SmemGrant* t = smem_grants();
  int slot = -1;
  for (int i = 0; i < 256; ++i) {
    if (t[i].fn == fn && t[i].dev == dev) {
      if (t[i].bytes >= bytes) return RB_OK;
      slot = i;
      break;
    }
    if (t[i].fn == nullptr) {
      slot = i;
      break;
    }
  }
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    snprintf(err_buffer(), 256, "%s: %s", who, cudaGetErrorString(e));
    return RB_ERR_CUDA;
  }
  if (slot >= 0) {
    t[slot].fn = fn;
    t[slot].dev = dev;
    t[slot].bytes = bytes;
  }
  return RB_OK;
}

// ---- optional per-kernel timing: CUDA events recorded on the launching stream around a launch ----
constexpr int PROF_SLOTS = 2048;
struct ProfKernel {
  cudaEvent_t e0[PROF_SLOTS], e1[PROF_SLOTS];
  int created = 0, used = 0;
};
bool& prof_on();
ProfKernel* prof_table();  // [RB_KERNEL_COUNT]

struct ProfScope {
  cudaStream_t st;
  ProfKernel* k = nullptr;
  ProfScope(int id, cudaStream_t stream) : st(stream) {
    if (!prof_on()) return;
    ProfKernel* pk = &prof_table()[id];
    if (pk->used >= PROF_SLOTS) return;
    if (pk->used >= pk->created) {
      cudaEventCreate(&pk->e0[pk->created]);
      cudaEventCreate(&pk->e1[pk->created]);
      pk->created++;
    }
    k = pk;
    cudaEventRecord(k->e0[k->used], st);
  }
  ~ProfScope() {
    if (k) {
      cudaEventRecord(k->e1[k->used], st);
      k->used++;
    }
  }
};

// ---- tensor-core layer 1 of the fused head (rb_head_tc.cu), called from rb_head_forward -----------------------------
void head_fc1_tc_splits(int K1, int H, int* S, int* kt_per);
bool head_fc1_tc_ok(int K1, int H, int m_lo, int m_hi);
int head_fc1_tc(const float* const* w_mu, const float* const* w_sig, const float* const* b_mu, const float* const* b_sig,
                const float* const* ei, const float* const* eo, int K1, int H, const float* x_lo, int m_lo, const float* x_hi,
                int m_hi, float* part, float* h, cudaStream_t st);

// ---- Philox4x32-10 counter-based RNG (Salmon et al. 2011) -------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

// 53-bit unit uniform in [0,1) from two 32-bit words (same construction as numpy's random_sample).
__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
  return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0);
}

// Box-Muller: two 32-bit words -> two standard normals.
__device__ __forceinline__ float2 box_muller(uint32_t a, uint32_t b) {
  float u1 = ((float)a + 1.0f) * 2.3283064365386963e-10f;  // (0,1]
  float u2 = (float)b * 2.3283064365386963e-10f;           // [0,1)
  float r = sqrtf(-2.0f * logf(u1));
  float s, c;
  sincospif(2.0f * u2, &s, &c);
  return make_float2(r * c, r * s);
}

// Normals 4*idx4 .. 4*idx4+3 of stream `which` (0 = eps_in, 1 = eps_out) for draw `ctr`.
__device__ __forceinline__ float4 normal4(uint64_t seed, unsigned long long ctr, uint32_t which, uint32_t idx4) {
  uint4 r = philox4x32_10(make_uint4((uint32_t)ctr, (uint32_t)(ctr >> 32), idx4, 0x4E4F4953u + which),
                          make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  float2 a = box_muller(r.x, r.y), b = box_muller(r.z, r.w);
  return make_float4(a.x, a.y, b.x, b.y);
}

// model.py:32-34: f(x) = sign(x) * sqrt(|x|)
__device__ __forceinline__ float scale_noise(float x) {
  float s = (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f);
  return __fmul_rn(s, __fsqrt_rn(fabsf(x)));
}

}  // namespace rbi
