/*
 * rb_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C, scalar-loop restatement of the Kaixhin/Rainbow learner hot path
 * (reference commit 1745b184), used ONLY as the checker in tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
 * Nothing under rainbow_b200/ may import, link or call this file.
 *
 * Parity status: the reference ships no tests or golden vectors for this path
 * ("parity unpinned" by the reference itself).  This oracle is pinned instead
 * against outputs of the UNMODIFIED reference modules imported from
 * /root/reference in the build container: see oracle/gen_golden.py (generator)
 * and tests/golden/ (npz) (committed vectors); tests/test_oracle_golden.py
 * checks every function below against them.
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -fPIC -shared (see Makefile).
 * -ffp-contract=off matters: the reference evaluates every float op separately
 * (numpy / ATen eager), so no FMA contraction is allowed here either.
 *
 * Each function cites the reference lines it restates (paths relative to the
 * reference repo root).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define FRAME_BYTES 7056 /* 84*84, memory.py:7 */

/* Python-style modulo (result has the sign of the divisor); memory.py:86,131 */
static int64_t pymod(int64_t a, int64_t m) {
  int64_t r = a % m;
  return r < 0 ? r + m : r;
}

/* ------------------------------------------------------------------------- */
/* Sum tree                                                                   */
/* ------------------------------------------------------------------------- */

/* memory.py:17 -- leaves start at 2**ceil(log2(size)) - 1 */
int64_t orc_tree_start(int64_t size) {
  int64_t p = 1;
  while (p < size) p <<= 1;
  return p - 1;
}

/* memory.py:158 -- np.power(priorities, omega) on float32.
 * numpy evaluates float32 ** python-float in float32 (powf); for omega == 0.5
 * the result is bit-identical to sqrtf (SURVEY.md 8(a) A9 probe, re-checked by
 * the golden test). */
void orc_pow_priorities(const float* raw, float omega, int B, float* out) {
  for (int i = 0; i < B; ++i) out[i] = (omega == 0.5f) ? sqrtf(raw[i]) : powf(raw[i], omega);
}

/* memory.py:44-48 (update) + :28-33 (_propagate) + :23-25 (_update_nodes).
 * Leaf scatter in index order (duplicates: last write wins), then one
 * level at a time every touched parent is recomputed as fl32(left + right).
 * `values` are already exponentiated.  *max_io follows memory.py:47-48. */
void orc_tree_update(float* tree, const int64_t* idx, const float* values, int B, float* max_io) {
  int64_t* node = (int64_t*)malloc(sizeof(int64_t) * (size_t)B);
  float vmax = values[0];
  for (int i = 0; i < B; ++i) {
    tree[idx[i]] = values[i];
    node[i] = idx[i];
    if (values[i] > vmax) vmax = values[i];
  }
  /* all idx sit on the leaf level, so all walks have the same length */
  while (node[0] != 0) {
    for (int i = 0; i < B; ++i) {
      int64_t p = (node[i] - 1) / 2;
      tree[p] = tree[2 * p + 1] + tree[2 * p + 2];
      node[i] = p;
    }
  }
  if (vmax > *max_io) *max_io = vmax;
  free(node);
}

/* memory.py:51-54 (_update_index) + :36-41 (_propagate_index) */
void orc_tree_set_leaf(float* tree, int64_t tree_index, float value) {
  tree[tree_index] = value;
  int64_t i = tree_index;
  while (i != 0) {
    int64_t p = (i - 1) / 2;
    tree[p] = tree[2 * p + 1] + tree[2 * p + 2];
    i = p;
  }
}

/* memory.py:64-82 (find/_retrieve), one sample at a time.
 * Residual is float64, nodes float32; strict '>' sends the walk right.
 * On the level above the leaves both child indices are clipped to the last
 * array element (memory.py:70-71).  Returns 0. */
int orc_tree_find(const float* tree, int64_t tree_start, int64_t size, const double* values, int B,
                  float* probs, int64_t* data_idx, int64_t* tree_idx) {
  const int64_t len = tree_start + size;
  for (int k = 0; k < B; ++k) {
    double v = values[k];
    int64_t i = 0;
    while (i < tree_start) {
      int64_t cl = 2 * i + 1, cr = 2 * i + 2;
      if (cl >= tree_start) {
        if (cl > len - 1) cl = len - 1;
        if (cr > len - 1) cr = len - 1;
      }
      float left = tree[cl];
      if (v > (double)left) {
        v = v - (double)left;
        i = cr;
      } else {
        i = cl;
      }
    }
    probs[k] = tree[i];
    tree_idx[k] = i;
    data_idx[k] = i - tree_start;
  }
  return 0;
}

/* memory.py:125-129 -- stratified sample points from unit uniforms.
 * segment_length is float32 (numpy 2: np.float32 / int), widened to float64
 * for both the draw (RandomState.uniform = low + (high-low)*u) and the
 * segment starts (int64 arange * np.float32 -> float64). */
void orc_segment_samples(float p_total, int B, const double* u01, double* samples) {
  float seg = p_total / (float)B;
  double segd = (double)seg;
  for (int k = 0; k < B; ++k) {
    double draw = 0.0 + segd * u01[k];
    double start = (double)k * segd;
    samples[k] = draw + start;
  }
}

/* memory.py:131 -- whole-batch validity.  Returns 1 when every sample passes. */
int orc_batch_valid(const int64_t* data_idx, const float* probs, int B, int64_t head, int64_t capacity,
                    int n, int history) {
  for (int k = 0; k < B; ++k) {
    if (!(pymod(head - data_idx[k], capacity) > n)) return 0;
    if (!(pymod(data_idx[k] - head, capacity) >= history)) return 0;
    if (!(probs[k] != 0.0f)) return 0;
  }
  return 1;
}

/* memory.py:151-154 -- importance-sampling weights, all float32:
 * p = prob/total ; w = (count*p)**(-beta) ; w /= max(w). */
void orc_is_weights(const float* probs, float p_total, int64_t count, float beta, int B, float* weights) {
  float wmax = -INFINITY;
  float nb = -beta;
  for (int k = 0; k < B; ++k) {
    float p = probs[k] / p_total;
    float w = powf((float)count * p, nb);
    weights[k] = w;
    if (w > wmax) wmax = w;
  }
  for (int k = 0; k < B; ++k) weights[k] = weights[k] / wmax;
}

/* ------------------------------------------------------------------------- */
/* Transition ring (structure-of-arrays restatement of Transition_dtype)      */
/* ------------------------------------------------------------------------- */

/* memory.py:106 -- state[-1].mul(255).to(uint8): float32 product, then a
 * truncating cast. */
void orc_quantise_frame(const float* frame, uint8_t* out) {
  for (int i = 0; i < FRAME_BYTES; ++i) {
    float x = frame[i] * 255.0f;
    out[i] = (uint8_t)(int)x;
  }
}

/* memory.py:111-121 (_get_transitions) + :134-145 (_get_samples_from_segments
 * tail).  Window = H+n records around each sampled index, indices wrap
 * (memory.py:86); records are blanked when they belong to another episode
 * (memory.py:114-120); blank record = zero frame, action 0, reward 0,
 * nonterminal False (memory.py:8).
 * Outputs: states/next_states f32 [B,H,84*84] (= u8 / 255, true division),
 * actions i64[B], returns f32[B] (left-to-right f32 dot with gamma_pow, as
 * torch.matmul produces here -- pinned by the golden test), nonterminals f32[B]. */
void orc_gather(const uint8_t* frames, const int32_t* timestep, const int32_t* action, const float* reward,
                const uint8_t* nonterminal, int64_t size, const int64_t* data_idx, int B, int history, int n,
                const float* gamma_pow, float* states, float* next_states, int64_t* actions, float* returns,
                float* nonterminals) {
  const int W = history + n;
  int64_t* pos = (int64_t*)malloc(sizeof(int64_t) * (size_t)W);
  int* first = (int*)malloc(sizeof(int) * (size_t)W);
  int* blank = (int*)malloc(sizeof(int) * (size_t)W);
  for (int b = 0; b < B; ++b) {
    for (int s = 0; s < W; ++s) {
      pos[s] = pymod(data_idx[b] - (history - 1) + s, size);
      first[s] = timestep[pos[s]] == 0;
      blank[s] = 0;
    }
    for (int t = history - 2; t >= 0; --t) blank[t] = blank[t + 1] || first[t + 1];
    for (int t = history; t < W; ++t) blank[t] = blank[t - 1] || first[t];
    for (int h = 0; h < history; ++h) {
      float* dst = states + ((size_t)b * history + h) * FRAME_BYTES;
      float* dstn = next_states + ((size_t)b * history + h) * FRAME_BYTES;
      const uint8_t* src = frames + (size_t)pos[h] * FRAME_BYTES;
      const uint8_t* srcn = frames + (size_t)pos[n + h] * FRAME_BYTES;
      for (int i = 0; i < FRAME_BYTES; ++i) {
        dst[i] = blank[h] ? 0.0f : (float)src[i] / 255.0f;
        dstn[i] = blank[n + h] ? 0.0f : (float)srcn[i] / 255.0f;
      }
    }
    actions[b] = blank[history - 1] ? 0 : (int64_t)action[pos[history - 1]];
    float acc = 0.0f;
    for (int k = 0; k < n; ++k) {
      int s = history - 1 + k;
      float r = blank[s] ? 0.0f : reward[pos[s]];
      acc = acc + r * gamma_pow[k];
    }
    returns[b] = acc;
    nonterminals[b] = blank[W - 1] ? 0.0f : (nonterminal[pos[W - 1]] ? 1.0f : 0.0f);
  }
  free(pos);
  free(first);
  free(blank);
}

/* memory.py:166-178 -- validation iterator state at position `cur`:
 * H records ending at cur (negative indices wrap like numpy), backward-only
 * blanking.  out f32 [H,84*84]. */
void orc_iter_state(const uint8_t* frames, const int32_t* timestep, int64_t size, int64_t cur, int history,
                    float* out) {
  int first[64], blank[64];
  int64_t pos[64];
  for (int s = 0; s < history; ++s) {
    pos[s] = pymod(cur - (history - 1) + s, size);
    first[s] = timestep[pos[s]] == 0;
    blank[s] = 0;
  }
  for (int t = history - 2; t >= 0; --t) blank[t] = blank[t + 1] || first[t + 1];
  for (int s = 0; s < history; ++s) {
    const uint8_t* src = frames + (size_t)pos[s] * FRAME_BYTES;
    for (int i = 0; i < FRAME_BYTES; ++i) out[(size_t)s * FRAME_BYTES + i] = blank[s] ? 0.0f : (float)src[i] / 255.0f;
  }
}

/* ------------------------------------------------------------------------- */
/* Learner: double-DQN + C51 projection + IS-weighted cross-entropy           */
/* ------------------------------------------------------------------------- */

static void softmax_row(const float* x, int Z, float* p, float* logp) {
  float mx = x[0];
  for (int z = 1; z < Z; ++z)
    if (x[z] > mx) mx = x[z];
  float sum = 0.0f;
  for (int z = 0; z < Z; ++z) {
    p[z] = expf(x[z] - mx);
    sum += p[z];
  }
  float lsum = logf(sum);
  for (int z = 0; z < Z; ++z) {
    p[z] = p[z] / sum;
    if (logp) logp[z] = (x[z] - mx) - lsum;
  }
}

/* agent.py:66-96 given the three PRE-softmax logit tensors [B,A,Z]
 * (model.py:75 `q`), i.e. with the softmax halves of model.py:76-79 folded in.
 *   - agent.py:67      log p(s_t, a_t)        (log-softmax row of the online net)
 *   - agent.py:71-73   a* = argmax_a sum_z support_z * p_online(s_{t+n}, a, z)
 *   - agent.py:75-76   p_target(s_{t+n}, a*, .)
 *   - agent.py:79-80   Tz = R + (nonterminal * gamma^n) * support, clamped
 *   - agent.py:82-86   b, l, u with the two fix-ups (second sees updated l)
 *   - agent.py:89-92   m: all l-side terms in atom order, then all u-side terms
 *   - agent.py:94      loss_i = -sum_z m * logp
 *   - agent.py:96      d/dq[i,a_i,z] of mean_i(w_i*loss_i) = (w_i/B) * (p*sum(m) - m)
 * Outputs: loss[B], grad[B,A,Z] (zero off the taken action), m[B,Z] (may be NULL),
 * astar[B] (may be NULL). */
void orc_c51(const float* q_on_s, const float* q_on_ns, const float* q_tg_ns, const int64_t* actions,
             const float* returns, const float* nonterminals, const float* weights, const float* support,
             float vmin, float vmax, float delta_z, float gamma_n, int B, int A, int Z, float* loss, float* grad,
             float* m_out, int64_t* astar_out) {
  float* p = (float*)malloc(sizeof(float) * (size_t)Z * 6);
  float* logp = p + Z;
  float* pt = p + 2 * Z;
  float* bb = p + 3 * Z;
  float* m = p + 4 * Z;
  float* tmp = p + 5 * Z;
  int64_t* l = (int64_t*)malloc(sizeof(int64_t) * (size_t)Z * 2);
  int64_t* u = l + Z;
  for (int i = 0; i < B; ++i) {
    /* double-DQN action selection with the online net */
    int best = 0;
    float best_ev = -INFINITY;
    for (int a = 0; a < A; ++a) {
      softmax_row(q_on_ns + ((size_t)i * A + a) * Z, Z, tmp, NULL);
      float ev = 0.0f;
      for (int z = 0; z < Z; ++z) ev += support[z] * tmp[z];
      if (ev > best_ev) {
        best_ev = ev;
        best = a;
      }
    }
    if (astar_out) astar_out[i] = best;
    softmax_row(q_tg_ns + ((size_t)i * A + best) * Z, Z, pt, NULL);
    const int64_t act = actions[i];
    softmax_row(q_on_s + ((size_t)i * A + act) * Z, Z, p, logp);
    /* projection */
    float scale = nonterminals[i] * gamma_n;
    for (int z = 0; z < Z; ++z) {
      float tz = returns[i] + scale * support[z];
      if (tz < vmin) tz = vmin;
      if (tz > vmax) tz = vmax;
      float b = (tz - vmin) / delta_z;
      int64_t lo = (int64_t)floorf(b), up = (int64_t)ceilf(b);
      if (up > 0 && lo == up) lo -= 1;
      if (lo < Z - 1 && lo == up) up += 1;
      bb[z] = b;
      l[z] = lo;
      u[z] = up;
      m[z] = 0.0f;
    }
    for (int z = 0; z < Z; ++z) m[l[z]] += pt[z] * ((float)u[z] - bb[z]);
    /* fp32 rounding can put b just past Z - 1 at Tz = Vmax (e.g. Z 62 with V +-1): u = Z, outside m.  That
     * contribution, pt * (b - l), is within the rounding of b; it is dropped, as the kernel drops it. */
    for (int z = 0; z < Z; ++z)
      if (u[z] < Z) m[u[z]] += pt[z] * (bb[z] - (float)l[z]);
    float ce = 0.0f, msum = 0.0f;
    for (int z = 0; z < Z; ++z) {
      ce += m[z] * logp[z];
      msum += m[z];
    }
    loss[i] = -ce;
    if (m_out) memcpy(m_out + (size_t)i * Z, m, sizeof(float) * (size_t)Z);
    float* g = grad + (size_t)i * A * Z;
    for (int j = 0; j < A * Z; ++j) g[j] = 0.0f;
    float wi = weights[i] / (float)B;
    for (int z = 0; z < Z; ++z) g[(size_t)act * Z + z] = wi * (p[z] * msum - m[z]);
  }
  free(p);
  free(l);
}

/* ------------------------------------------------------------------------- */
/* NoisyLinear noise                                                          */
/* ------------------------------------------------------------------------- */

/* model.py:32-40 -- f(x) = sign(x)*sqrt(|x|) on the raw normals, then
 * weight_epsilon = f(x_out) (outer) f(x_in), bias_epsilon = f(x_out). */
void orc_noisy(const float* x_in, const float* x_out, int in_f, int out_f, float* w_eps, float* b_eps) {
  float* fi = (float*)malloc(sizeof(float) * (size_t)in_f);
  for (int i = 0; i < in_f; ++i) {
    float s = (x_in[i] > 0.0f) ? 1.0f : ((x_in[i] < 0.0f) ? -1.0f : 0.0f);
    fi[i] = s * sqrtf(fabsf(x_in[i]));
  }
  for (int o = 0; o < out_f; ++o) {
    float s = (x_out[o] > 0.0f) ? 1.0f : ((x_out[o] < 0.0f) ? -1.0f : 0.0f);
    float fo = s * sqrtf(fabsf(x_out[o]));
    b_eps[o] = fo;
    for (int i = 0; i < in_f; ++i) w_eps[(size_t)o * in_f + i] = fo * fi[i];
  }
  free(fi);
}

/* ------------------------------------------------------------------------- */
/* Optimiser step (agent.py:97-98): clip_grad_norm_ + Adam, flat buffers      */
/* ------------------------------------------------------------------------- */

/* torch.nn.utils.clip_grad_norm_(params, max_norm): total L2 norm over all
 * grads, coef = max_norm / (norm + 1e-6) clamped to 1.  Then torch.optim.Adam
 * (betas 0.9/0.999, no weight decay, no amsgrad):
 *   m = b1*m + (1-b1)*g ; v = b2*v + (1-b2)*g*g ;
 *   p -= (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
 * `step` is the 1-based step count AFTER this update.  Returns the pre-clip norm. */
float orc_clip_adam(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t P, float max_norm,
                    float lr, float beta1, float beta2, float eps, int64_t step) {
  double acc = 0.0;
  for (int64_t i = 0; i < P; ++i) acc += (double)grad[i] * (double)grad[i];
  float norm = (float)sqrt(acc);
  float coef = max_norm / (norm + 1e-6f);
  if (coef > 1.0f) coef = 1.0f;
  double bc1 = 1.0 - pow((double)beta1, (double)step);
  double bc2 = 1.0 - pow((double)beta2, (double)step);
  float step_size = (float)((double)lr / bc1);
  float bc2_sqrt = (float)sqrt(bc2);
  for (int64_t i = 0; i < P; ++i) {
    float g = grad[i] * coef;
    grad[i] = g;
    float m = exp_avg[i] + (g - exp_avg[i]) * (1.0f - beta1); /* torch: lerp_(grad, 1-beta1) */
    float v = exp_avg_sq[i] * beta2 + (1.0f - beta2) * g * g;
    exp_avg[i] = m;
    exp_avg_sq[i] = v;
    float denom = sqrtf(v) / bc2_sqrt + eps;
    param[i] = param[i] - step_size * (m / denom);
  }
  return norm;
}
