// rl_kernels.cuh -- trajectory post-processing, sampling and loss kernels (HBM / latency bound).
//   gae_kernel                : xt/agent/ppo/ppo.py:77-106       one warp per env, affine reverse scan
//   sample_kernel<DIST>       : xt/model/tf_dist.py:63-130       Categorical (Gumbel-max) / DiagGaussian draw + log-prob
//   ppo_loss_kernel           : xt/model/ppo/__init__.py:4-25    Categorical loss + dlogits/dv, block-reduced loss
//   ppo_gauss_loss_kernel     : xt/model/ppo/__init__.py:4-25    DiagGaussian loss + dmean/dv, ordered dlog_std and loss
//   vtrace_kernel             : xt/model/impala/vtrace.py:39-115 + impala_cnn_opt.py:299-351
//   dqn_loss_kernel           : xt/algorithm/dqn/dqn.py:79-97 + Keras mse (double DQN, n-step discount, Huber)
//   nstep_kernel              : n-step returns of a device-resident rollout buffer
//   heads_kernel<LOSS>        : both dense heads + the per-sample loss of LOSS + their backward, one warp per sample
//   infer_heads_kernel<DIST>  : both dense heads + the draw of DIST (rollout inference), one warp per sample
//   dueling_fwd / dgrad       : the dueling combine layer
//   IMPALA Keras, MuZero      : softmax_rows, impala_keras_*, mse_loss; mz_*
// The per-sample rules (categorical_draw / gaussian_draw, ppo_categorical_row, ppo_gauss_row, dqn_td_target / td_loss)
// are written once: the standalone kernels of the layer-by-layer path and the fused heads kernels both call them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gemm_f32.cuh"

namespace xtb {

constexpr int MAX_ADIM = 32;

__device__ inline float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-level sum -> one atomicAdd per block
__device__ inline void block_atomic_add(float v, float* out) {
  __shared__ float red[32];
  v = warp_sum(v);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    int nw = (blockDim.x + 31) >> 5;
    float s = lane < nw ? red[lane] : 0.f;
    s = warp_sum(s);
    if (lane == 0) atomicAdd(out, s);
  }
}

// ------------------------------------------------------------------------------------------
// GAE.  adv_t = delta_t + c_t * adv_{t+1},  c_t = (1-done_t)*gamma*lam, adv_T = 0.
// Each lane owns `chunk` consecutive steps; per-lane affine map (a,b): adv_in -> a*adv_in+b is
// composed right-to-left, exclusive-scanned across lanes with shuffles, then replayed.
// ------------------------------------------------------------------------------------------
__global__ void gae_kernel(const float* __restrict__ value, const float* __restrict__ reward,
                           const uint8_t* __restrict__ done, int n_env, int T, float gamma, float lam,
                           int sign_clip, float* __restrict__ adv, float* __restrict__ old_v,
                           float* __restrict__ target_v) {
  pdl_wait(); pdl_trigger();
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= n_env) return;
  const float* V = value + (long long)warp * (T + 1);
  const float* R = reward + (long long)warp * T;
  const uint8_t* D = done + (long long)warp * T;
  float* A = adv + (long long)warp * T;
  float* OV = old_v + (long long)warp * T;
  float* TV = target_v + (long long)warp * T;
  int chunk = (T + 31) / 32;
  int t0 = lane * chunk, t1 = min(T, t0 + chunk);
  // pass 1: compose the chunk's affine map, walking backwards
  float a = 1.f, b = 0.f;
  for (int t = t1 - 1; t >= t0; --t) {
    float r = R[t];
    if (sign_clip) r = (r > 0.f) ? 1.f : ((r < 0.f) ? -1.f : 0.f);
    float disc = D[t] ? 0.f : gamma;
    float delta = r + disc * V[t + 1] - V[t];
    float c = disc * lam;
    // adv_t = delta + c*adv_{t+1};  adv_{t+1} = a*x + b  =>  adv_t = (c*a)*x + (delta + c*b)
    b = delta + c * b;
    a = c * a;
  }
  // suffix scan over lanes: incoming value for lane l = result of lanes l+1..31 applied to 0
  // inclusive suffix composition F_l = f_l o F_{l+1}
  float fa = a, fb = b;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float oa = __shfl_down_sync(0xffffffffu, fa, o);
    float ob = __shfl_down_sync(0xffffffffu, fb, o);
    if (lane + o < 32) {  // F = F o other : x -> fa*(oa*x+ob)+fb
      fb = fa * ob + fb;
      fa = fa * oa;
    }
  }
  float incoming = __shfl_down_sync(0xffffffffu, fb, 1);  // F_{l+1}(0) = fb_{l+1}
  if (lane == 31) incoming = 0.f;
  // pass 2: replay
  float nxt = incoming;
  for (int t = t1 - 1; t >= t0; --t) {
    float r = R[t];
    if (sign_clip) r = (r > 0.f) ? 1.f : ((r < 0.f) ? -1.f : 0.f);
    float disc = D[t] ? 0.f : gamma;
    float v = V[t];
    float delta = r + disc * V[t + 1] - v;
    float ad = delta + disc * lam * nxt;
    A[t] = ad;
    OV[t] = v;
    TV[t] = ad + v;
    nxt = ad;
  }
}

// ------------------------------------------------------------------------------------------
// Philox4x32-10
// ------------------------------------------------------------------------------------------
__device__ inline void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; i++) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

// Categorical draw of sample b (xt/model/tf_dist.py:89-130): Gumbel-max over its logits lg[0..A), A <= n (n: the
// size of a register array, whose loops are unrolled, or A).  Uniform i is u[i] when u is set, else a word of
// Philox4x32-10 on counter (b, i / 4, offset) mapped into (0, 1).  The first maximum wins, like np.argmax.  Writes the
// action to action[b] and, when head_out is set, the logits to its row b; returns the action's log-probability.
template <class LG>
__device__ __forceinline__ float categorical_draw(const LG& lg, int n, int A, const float* u, int b, uint64_t seed,
                                                  uint64_t offset, int32_t* action, float* head_out) {
  if (head_out) {
#pragma unroll
    for (int i = 0; i < n; i++) if (i < A) head_out[(long long)b * A + i] = lg[i];
  }
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < n; i++) if (i < A) mx = fmaxf(mx, lg[i]);
  float z = 0.f;
#pragma unroll
  for (int i = 0; i < n; i++) if (i < A) z += expf(lg[i] - mx);
  const float lz = logf(z);
  float best = -INFINITY; int bi = 0;
  uint32_t c[4] = {0, 0, 0, 0};
#pragma unroll
  for (int i = 0; i < n; i++) {
    if (i < A) {
      float ui;
      if (u) {
        ui = u[i];
      } else {
        if ((i & 3) == 0) {
          c[0] = (uint32_t)b; c[1] = (uint32_t)(i >> 2);
          c[2] = (uint32_t)(offset & 0xffffffffu); c[3] = (uint32_t)(offset >> 32);
          philox4x32_10(c, (uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32));
        }
        ui = (float)(c[i & 3] >> 8) * 5.9604644775390625e-08f + 2.98023223876953125e-08f;
      }
      const float s = lg[i] - logf(-logf(ui));
      if (s > best) { best = s; bi = i; }
    }
  }
  float la = 0.f;
#pragma unroll
  for (int i = 0; i < n; i++) if (i == bi) la = lg[i];
  action[b] = bi;
  return la - mx - lz;
}

__global__ void bump_counter_kernel(unsigned long long* ctr, int add) {
  pdl_wait(); pdl_trigger(); *ctr += (unsigned long long)add; }

__global__ void argmax_kernel(const float* __restrict__ q, int B, int A, int32_t* __restrict__ action) {
  pdl_wait(); pdl_trigger();
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* l = q + (long long)b * A;
  float best = l[0]; int bi = 0;
  for (int i = 1; i < A; i++) if (l[i] > best) { best = l[i]; bi = i; }
  action[b] = bi;
}

// ------------------------------------------------------------------------------------------
// PPO loss + gradient wrt (logits, v).  One thread per sample.
// ------------------------------------------------------------------------------------------
struct PpoHyperDev { float clip_ratio, ent_coef, vf_clip, critic_coef; };

// The clipped surrogate and the clipped value loss of one sample, whatever the action distribution: surr, dsurr =
// d surr / d logp_a (through s1 when s1 <= s2, else through the clip: zero outside the range), critic = the critic
// term of the loss, dv = d loss / d v.
struct PpoClipTerms { float surr, dsurr, critic, dv; };
__device__ __forceinline__ PpoClipTerms ppo_clip_terms(float logp_a, float old_logp, float ad, float vv, float ov, float R,
                                                       const PpoHyperDev& hp, float inv_count) {
  const float ratio = expf(logp_a - old_logp);
  const float s1 = ratio * ad;
  const float s2 = fminf(fmaxf(ratio, 1.f - hp.clip_ratio), 1.f + hp.clip_ratio) * ad;
  const float surr = fminf(s1, s2);
  const float dsurr = (s1 <= s2) ? ratio * ad
                                 : ((ratio >= 1.f - hp.clip_ratio && ratio <= 1.f + hp.clip_ratio) ? ratio * ad : 0.f);
  const float l1 = (vv - R) * (vv - R);
  const float vc = ov + fminf(fmaxf(vv - ov, -hp.vf_clip), hp.vf_clip);
  const float l2 = (vc - R) * (vc - R);
  const float dvl = (l1 >= l2) ? 2.f * (vv - R) : ((vv - ov >= -hp.vf_clip && vv - ov <= hp.vf_clip) ? 2.f * (vc - R) : 0.f);
  return {surr, dsurr, hp.critic_coef * 0.5f * fmaxf(l1, l2), hp.critic_coef * 0.5f * dvl * inv_count};
}

// Categorical PPO loss of sample b: actor loss with entropy + clipped critic loss (xt/model/ppo/__init__.py:4-25) on
// its logits lg[0..A), A <= n (as in categorical_draw), and value vv; the rollout row is r = idx ? idx[b] : b.  Fills
// dl[i] = d loss / d logit_i (0 for A <= i < n) and dv = d loss / d v; returns the sample's loss term.
template <class LG, class DL>
__device__ __forceinline__ float ppo_categorical_row(const LG& lg, int n, int A, float vv, const int32_t* idx, int b,
                                                     const int32_t* action, const float* old_logp, const float* adv,
                                                     const float* old_v, const float* target_v, const PpoHyperDev& hp,
                                                     float inv_count, DL& dl, float& dv) {
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < n; i++) if (i < A) mx = fmaxf(mx, lg[i]);
  float z = 0.f;
#pragma unroll
  for (int i = 0; i < n; i++) if (i < A) z += expf(lg[i] - mx);
  const float lz = logf(z);
  float H = 0.f;
#pragma unroll
  for (int i = 0; i < n; i++) if (i < A) { const float rl = lg[i] - mx; H += (expf(rl) / z) * (lz - rl); }
  const int r = idx ? idx[b] : b;
  const int ac = action[r];
  float logp_a = 0.f;
#pragma unroll
  for (int i = 0; i < n; i++) if (i == ac) logp_a = lg[i] - mx - lz;
  const PpoClipTerms c = ppo_clip_terms(logp_a, old_logp[r], adv[r], vv, old_v[r], target_v[r], hp, inv_count);
  dv = c.dv;
#pragma unroll
  for (int i = 0; i < n; i++) {
    float d = 0.f;
    if (i < A) {   // d logp_a / d l_i = [i == a] - p_i,  d H / d l_i = -p_i (logp_i + H)
      const float rl = lg[i] - mx, p = expf(rl) / z;
      d = (-c.dsurr * (((i == ac) ? 1.f : 0.f) - p) + hp.ent_coef * p * (rl - lz + H)) * inv_count;
    }
    dl[i] = d;
  }
  return (-c.surr - hp.ent_coef * H + c.critic) * inv_count;
}

__global__ void ppo_loss_kernel(const float* __restrict__ logits, const float* __restrict__ v,
                                const int32_t* __restrict__ idx, const int32_t* __restrict__ action,
                                const float* __restrict__ old_logp, const float* __restrict__ adv,
                                const float* __restrict__ old_v, const float* __restrict__ target_v,
                                int B, int A, PpoHyperDev hp, float inv_count,
                                float* __restrict__ dlogits, float* __restrict__ dv,
                                float* __restrict__ loss_out) {
  pdl_wait(); pdl_trigger();
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  float lsum = 0.f;
  if (b < B) {
    float* dl = dlogits + (long long)b * A;
    lsum = ppo_categorical_row(logits + (long long)b * A, A, A, v[b], idx, b, action, old_logp, adv, old_v, target_v, hp,
                               inv_count, dl, dv[b]);
  }
  block_atomic_add(lsum, loss_out);
}

// ------------------------------------------------------------------------------------------
// V-trace + IMPALA loss.  One warp per trajectory, lanes own consecutive time chunks.
// loss = sum xent*pg_adv + 0.25*sum (vs-V)^2 - 0.01*sum H    (sums, not means)
// ------------------------------------------------------------------------------------------
__device__ inline void softmax_stats(const float* l, int A, float& mx, float& lz) {
  mx = -INFINITY;
  for (int i = 0; i < A; i++) mx = fmaxf(mx, l[i]);
  float z = 0.f;
  for (int i = 0; i < A; i++) z += expf(l[i] - mx);
  lz = logf(z);
}

__global__ void vtrace_kernel(const float* __restrict__ tp_logits, const float* __restrict__ baseline,
                              const float* __restrict__ bp_logits, const int32_t* __restrict__ action,
                              const uint8_t* __restrict__ done, const float* __restrict__ reward,
                              int n_traj, int S, int A, float gamma, float* __restrict__ dlogits,
                              float* __restrict__ dbaseline, float* __restrict__ vs_out,
                              float* __restrict__ pg_out, float* __restrict__ loss_out) {
  pdl_wait(); pdl_trigger();
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  float lsum = 0.f;
  if (warp < n_traj) {
    const long long base = (long long)warp * S;
    const int T = S - 1;                       // drop_last
    const float boot = baseline[base + S - 1];
    int chunk = (T + 31) / 32;
    int t0 = lane * chunk, t1 = min(T, t0 + chunk);
    // pass 1: chunk affine map of acc_t = delta_t + (disc_t*c_t)*acc_{t+1}
    float a = 1.f, b = 0.f;
    for (int t = t1 - 1; t >= t0; --t) {
      long long n = base + t;
      float mx, lz, bmx, blz;
      softmax_stats(tp_logits + n * A, A, mx, lz);
      softmax_stats(bp_logits + n * A, A, bmx, blz);
      int ac = action[n];
      float tlp = tp_logits[n * A + ac] - mx - lz;
      float blp = bp_logits[n * A + ac] - bmx - blz;
      float rho = expf(tlp - blp);
      float crho = fminf(1.f, rho), cs = fminf(1.f, rho);
      float disc = done[n] ? 0.f : gamma;
      float r = fminf(fmaxf(reward[n], -1.f), 1.f);
      float V = baseline[n];
      float Vn = (t == T - 1) ? boot : baseline[n + 1];
      float delta = crho * (r + disc * Vn - V);
      float c = disc * cs;
      b = delta + c * b;
      a = c * a;
    }
    float fa = a, fb = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float oa = __shfl_down_sync(0xffffffffu, fa, o);
      float ob = __shfl_down_sync(0xffffffffu, fb, o);
      if (lane + o < 32) { fb = fa * ob + fb; fa = fa * oa; }
    }
    float incoming = __shfl_down_sync(0xffffffffu, fb, 1);
    if (lane == 31) incoming = 0.f;
    // vs of the first step of the next lane's chunk (needed for pg_adv at our last step)
    // vs_{t1} = V_{t1} + acc_{t1};  acc_{t1} == incoming.
    float acc_next = incoming;
    for (int t = t1 - 1; t >= t0; --t) {
      long long n = base + t;
      float mx, lz, bmx, blz;
      const float* tl = tp_logits + n * A;
      softmax_stats(tl, A, mx, lz);
      softmax_stats(bp_logits + n * A, A, bmx, blz);
      int ac = action[n];
      float tlp = tl[ac] - mx - lz;
      float blp = bp_logits[n * A + ac] - bmx - blz;
      float rho = expf(tlp - blp);
      float crho = fminf(1.f, rho), cs = fminf(1.f, rho), cpg = fminf(1.f, rho);
      float disc = done[n] ? 0.f : gamma;
      float r = fminf(fmaxf(reward[n], -1.f), 1.f);
      float V = baseline[n];
      float Vn = (t == T - 1) ? boot : baseline[n + 1];
      float vs_next = (t == T - 1) ? boot : (Vn + acc_next);
      float delta = crho * (r + disc * Vn - V);
      float acc = delta + disc * cs * acc_next;
      float vs = V + acc;
      float pg = cpg * (r + disc * vs_next - V);
      if (vs_out) vs_out[n] = vs;
      if (pg_out) pg_out[n] = pg;
      // entropy and grads
      float H = 0.f;
      for (int i = 0; i < A; i++) { float lp = tl[i] - mx - lz; H -= expf(lp) * lp; }
      for (int i = 0; i < A; i++) {
        float lp = tl[i] - mx - lz;
        float p = expf(lp);
        float d = pg * (p - ((i == ac) ? 1.f : 0.f)) + 0.01f * p * (lp + H);
        dlogits[n * A + i] = d;
      }
      dbaseline[n] = 0.5f * (V - vs);
      lsum += (-tlp) * pg + 0.25f * (vs - V) * (vs - V) - 0.01f * H;
      acc_next = acc;
    }
    if (lane == 0) {
      long long n = base + S - 1;
      for (int i = 0; i < A; i++) dlogits[n * A + i] = 0.f;
      dbaseline[n] = 0.f;
      if (vs_out) vs_out[n] = 0.f;
      if (pg_out) pg_out[n] = 0.f;
    }
  }
  block_atomic_add(lsum, loss_out);
}

// ------------------------------------------------------------------------------------------
// DQN TD target + loss gradient.  Reference semantics (xt/algorithm/dqn/dqn.py:79-97 + Keras 'mse', mean over B*A):
// y = r (+ gamma * max_a' Q_target(s') unless done), loss = mean (Q - y)^2 over B*A with only the taken action non-zero.
// Extensions named by BASELINE.json's north_star, off by default:
//   disc != NULL : per-sample bootstrap discount (gamma^n of an n-step return built by nstep_kernel; 0 = terminated)
//   huber > 0    : Huber loss with that delta instead of the squared error (gradient clip(diff, -delta, delta))
//   idx != NULL  : action / reward / done / disc are indexed through idx (minibatch rows of a replay ring)
// ------------------------------------------------------------------------------------------
// TD target of sample b, rollout row r: the max over the next-state Q row b of the target net (qn_o set: double DQN,
// the target net's Q at the online net's argmax, the first maximum winning) bootstraps the reward unless done[r]
__device__ __forceinline__ float dqn_td_target(const float* qn_t, const float* qn_o, const float* reward, const uint8_t* done,
                                               const float* disc, float gamma, int b, int r, int A) {
  const float* t = qn_t + (long long)b * A;
  float mq;
  if (qn_o) {
    const float* o = qn_o + (long long)b * A;
    float best = o[0]; int bi = 0;
    for (int i = 1; i < A; i++) if (o[i] > best) { best = o[i]; bi = i; }
    mq = t[bi];
  } else {
    mq = t[0];
    for (int i = 1; i < A; i++) mq = fmaxf(mq, t[i]);
  }
  const float g = disc ? disc[r] : gamma;
  return done[r] ? reward[r] : reward[r] + g * mq;
}

// loss of the TD error diff = Q(s, a) - y (the squared error, or with huber > 0 the Huber loss of that delta);
// grad = d loss / d diff
__device__ __forceinline__ float td_loss(float diff, float huber, float& grad) {
  float l;
  if (huber > 0.f) {
    const float ad = fabsf(diff);
    l = ad <= huber ? 0.5f * diff * diff : huber * (ad - 0.5f * huber);
    grad = fminf(fmaxf(diff, -huber), huber);
  } else { l = diff * diff; grad = 2.f * diff; }
  return l;
}

__global__ void dqn_loss_kernel(const float* __restrict__ q, const float* __restrict__ qn_t,
                                const float* __restrict__ qn_o, const int32_t* __restrict__ idx,
                                const int32_t* __restrict__ action, const float* __restrict__ reward,
                                const uint8_t* __restrict__ done, const float* __restrict__ disc,
                                int B, int A, float gamma, float huber, float inv_count, float* __restrict__ dq,
                                float* __restrict__ y_out, float* __restrict__ loss_out) {
  pdl_wait(); pdl_trigger();
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  float lsum = 0.f;
  if (b < B) {
    const int r = idx ? idx[b] : b;
    const float y = dqn_td_target(qn_t, qn_o, reward, done, disc, gamma, b, r, A);
    const int a = action[r];
    float grad;
    const float l = td_loss(q[(long long)b * A + a] - y, huber, grad);
    for (int i = 0; i < A; i++) dq[(long long)b * A + i] = (i == a) ? grad * inv_count : 0.f;
    if (y_out) y_out[b] = y;
    lsum = l * inv_count;
  }
  block_atomic_add(lsum, loss_out);
}

// n-step returns over env-major trajectories [E][T] (north_star: "n-step TD-target kernel over a device-resident rollout
// buffer"): R_t = sum_{k<m} gamma^k r_{t+k}, m = steps until the first done (inclusive) or n or the end of the segment;
// disc_t = gamma^m, or 0 when the window ended in a terminal step; last_t = t + m - 1 (row whose next-state bootstraps);
// done_n_t = 1 when the window contains a terminal step.  One thread per (env, t); rows of a warp are consecutive t.
__global__ void nstep_kernel(const float* __restrict__ reward, const uint8_t* __restrict__ done, int E, int T, int n, float gamma,
                             float* __restrict__ ret, float* __restrict__ disc, int32_t* __restrict__ last, uint8_t* __restrict__ done_n) {
  pdl_wait(); pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= E * T) return;
  const int e = i / T, t = i - e * T;
  float acc = 0.f, g = 1.f;
  int k = 0; bool term = false;
  for (; k < n && t + k < T; k++) {
    acc = fmaf(g, reward[e * T + t + k], acc);
    g *= gamma;
    if (done[e * T + t + k]) { term = true; k++; break; }
  }
  ret[i] = acc;
  disc[i] = term ? 0.f : g;
  last[i] = i + k - 1;
  done_n[i] = term ? 1 : 0;
}

// ------------------------------------------------------------------------------------------
// Fused PPO heads: pi/v dense heads + categorical loss + their backward in ONE kernel (K4/K7 of the
// kernel work-list: the logits never leave the chip between the head GEMM and the loss).
//   logits = h_pi @ Wpi + bpi,  v = h_v @ Wv + bv            (xt/model/model_utils.py:63-65)
//   loss, dlogits, dv                                        (xt/model/ppo/__init__.py:4-25)
//   dWpi,dbpi,dWv,dbv += ...   (atomics into the flat gradient bucket)
//   g(h) = (dlogits @ Wpi^T [+ dv * Wv^T]) * act'(h)         -> gradient wrt the hidden pre-activation
// One warp per sample, lane owns hidden units lane, lane+32, ...  (K <= 32*HEAD_KPL, A <= HEAD_AMAX)
// The same kernel runs the dueling DQN TD step: the K x A head is the "value" stream, the K x 1 head the "adv" stream
// (xt/model/dqn/dqn_cnn.py:53-58); only the per-sample loss differs, so it is the LOSS template policy.
// ------------------------------------------------------------------------------------------
// template: HEAD_KPL hidden units per lane (K <= 32*HEAD_KPL), HEAD_AMAX >= A

struct PpoHeadsArgs {
  const float* h_pi; const float* h_v;     // [B,K] hidden activations (may alias)
  float* g_pi; float* g_v;                 // [B,K] gradient wrt hidden pre-activation (may alias)
  __nv_bfloat16* gp_hi; long long gp_lo; __nv_bfloat16* gv_hi; long long gv_lo;   // their batch-planar bf16 planes (bp_gemm.cuh), may be NULL
  int pitch;                               // rows per feature chunk of those planes
  const float* w_pi; const float* b_pi; const float* w_v; const float* b_v;
  // Parameter-gradient partial sums, one slab of `slab` floats per block, reduced afterwards in block order by
  // bp::grad_reduce_kernel (no atomics: the step is bitwise reproducible).  Slab layout (K hidden units, A actions):
  // [dW_pi K*A | dW_v K | dbh_pi K | dbh_v K | db_pi A | db_v 1 | loss 1 (| dlog_std A: LOSS::kLogStd)]; dbh_* = bias
  // gradients of the layers that produced h_pi / h_v (column sums of g).
  float* part; int slab;
  const int32_t* idx; const int32_t* action; const float* old_logp; const float* adv; const float* old_v; const float* target_v;
  float* logits_out; float* v_out;
  int B, K, A, act_pi, act_v, shared;
  PpoHyperDev hp; float inv_count;
  // dueling TD step (DuelingTdLoss): as dqn_loss_kernel, with q = the combine of the two heads; action / reward / done /
  // disc are indexed through idx.  loss_in: the loss already accumulated (added once, by sample 0, so the ordered
  // reduction of the loss slot writes loss_in + this step's loss).
  const float* qn_t; const float* qn_o; const float* reward; const uint8_t* done; const float* disc; const float* loss_in;
  float gamma, huber;
  // Gaussian PPO (PpoGaussLoss): float behaviour actions [N, A] indexed through idx, and the A floats of pi_logstd
  const float* action_f; const float* log_std;
};

// Per-sample loss policies of heads_kernel.  acc[0..A) = h . W_pi (no bias), acc[HEAD_AMAX] = h . W_v; every lane holds
// the same values.  Fill dl[i] = dloss/d(pi head output i), dv = dloss/d(v head output) (0 for i >= A) and, on lane 0,
// add the sample's loss to lsum and the bias gradients to dbp / dbv.  A policy with kLogStd also adds, on lane 0, the
// gradient wrt the state-independent log_std to dls (an extra A slab floats); the others leave dls alone.
// PPO: ppo_categorical_row on logits = acc[0..A) + b_pi, v = acc[HEAD_AMAX] + b_v.
struct PpoLoss {
  static constexpr bool kLogStd = false;
  template <int HEAD_AMAX>
  static __device__ __forceinline__ void sample(const PpoHeadsArgs& a, int b, int lane, const float (&acc)[HEAD_AMAX + 1],
                                                float (&dl)[HEAD_AMAX], float& dv, float& lsum, float (&dbp)[HEAD_AMAX],
                                                float& dbv, float (&)[HEAD_AMAX]) {
    const int A = a.A;
    float lg[HEAD_AMAX];
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) lg[i] = (i < A) ? acc[i] + a.b_pi[i] : -INFINITY;
    const float vv = acc[HEAD_AMAX] + a.b_v[0];
    const float l = ppo_categorical_row(lg, HEAD_AMAX, A, vv, a.idx, b, a.action, a.old_logp, a.adv, a.old_v, a.target_v, a.hp,
                                        a.inv_count, dl, dv);
    if (lane == 0) {
      lsum += l;
      if (a.logits_out) for (int i = 0; i < A; i++) a.logits_out[(long long)b * A + i] = lg[i];
      if (a.v_out) a.v_out[b] = vv;
      dbv += dv;
#pragma unroll
      for (int i = 0; i < HEAD_AMAX; i++) dbp[i] += dl[i];
    }
  }
};

// Dueling DQN TD step: value = pi head [A], adv = v head [1], q = adv + (value - mean_a value) (xt/model/dqn/dqn_mlp.py:80-87),
// then dqn_td_target and td_loss, as in dqn_loss_kernel.  Only the taken action carries gradient, g = c e_a, so
// dvalue = c (e_a - 1/A) and dadv = c.
struct DuelingTdLoss {
  static constexpr bool kLogStd = false;
  template <int HEAD_AMAX>
  static __device__ __forceinline__ void sample(const PpoHeadsArgs& a, int b, int lane, const float (&acc)[HEAD_AMAX + 1],
                                                float (&dl)[HEAD_AMAX], float& dv, float& lsum, float (&dbp)[HEAD_AMAX],
                                                float& dbv, float (&)[HEAD_AMAX]) {
    const int A = a.A;
    float val[HEAD_AMAX], s = 0.f;
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) { val[i] = (i < A) ? acc[i] + a.b_pi[i] : 0.f; s += val[i]; }
    const float adv = acc[HEAD_AMAX] + a.b_v[0], mean = s / A;
    const int r = a.idx ? a.idx[b] : b;
    const int ac = a.action[r];
    float q_a = 0.f;
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) if (i == ac) q_a = adv + (val[i] - mean);
    const float y = dqn_td_target(a.qn_t, a.qn_o, a.reward, a.done, a.disc, a.gamma, b, r, A);
    float grad;
    const float l = td_loss(q_a - y, a.huber, grad);
    const float c = grad * a.inv_count, cm = c / A;
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) dl[i] = (i < A) ? ((i == ac) ? c : 0.f) - cm : 0.f;
    dv = c;
    if (lane == 0) {
      lsum += l * a.inv_count;
      if (b == 0) lsum += *a.loss_in;
      dbv += dv;
#pragma unroll
      for (int i = 0; i < HEAD_AMAX; i++) dbp[i] += dl[i];
    }
  }
};

template <class LOSS, int HEAD_KPL, int HEAD_AMAX>
__global__ void __launch_bounds__(256) heads_kernel(PpoHeadsArgs a) {
  pdl_wait(); pdl_trigger();
  extern __shared__ float sh_dw[];          // [nwarp][nacc] per-warp partial sums in slab layout
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int K = a.K, A = a.A, kpl = K / 32;
  const int nacc = K * A + 3 * K + A + 2 + (LOSS::kLogStd ? A : 0);
  float wpi[HEAD_KPL][HEAD_AMAX], wv[HEAD_KPL];
  float dwp[HEAD_KPL][HEAD_AMAX], dwv[HEAD_KPL];
#pragma unroll
  for (int j = 0; j < HEAD_KPL; j++) {
    wv[j] = 0.f; dwv[j] = 0.f;
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) { wpi[j][i] = 0.f; dwp[j][i] = 0.f; }
    if (j < kpl) {
      int k = lane + 32 * j;
      wv[j] = a.w_v[k];
#pragma unroll
      for (int i = 0; i < HEAD_AMAX; i++) if (i < A) wpi[j][i] = a.w_pi[k * A + i];
    }
  }
  float dbp[HEAD_AMAX], dls[HEAD_AMAX]; float dbv = 0.f, lsum = 0.f;
  float bh_pi[HEAD_KPL], bh_v[HEAD_KPL];
#pragma unroll
  for (int j = 0; j < HEAD_KPL; j++) { bh_pi[j] = 0.f; bh_v[j] = 0.f; }
#pragma unroll
  for (int i = 0; i < HEAD_AMAX; i++) { dbp[i] = 0.f; dls[i] = 0.f; }
  for (int b = blockIdx.x * nwarp + warp; b < a.B; b += gridDim.x * nwarp) {
    float hp_[HEAD_KPL], hv_[HEAD_KPL];
    float acc[HEAD_AMAX + 1];
#pragma unroll
    for (int i = 0; i <= HEAD_AMAX; i++) acc[i] = 0.f;
#pragma unroll
    for (int j = 0; j < HEAD_KPL; j++) {
      hp_[j] = 0.f; hv_[j] = 0.f;
      if (j < kpl) {
        int k = lane + 32 * j;
        hp_[j] = a.h_pi[(long long)b * K + k];
        hv_[j] = a.shared ? hp_[j] : a.h_v[(long long)b * K + k];
#pragma unroll
        for (int i = 0; i < HEAD_AMAX; i++) acc[i] = fmaf(hp_[j], wpi[j][i], acc[i]);
        acc[HEAD_AMAX] = fmaf(hv_[j], wv[j], acc[HEAD_AMAX]);
      }
    }
#pragma unroll
    for (int i = 0; i <= HEAD_AMAX; i++) acc[i] = warp_sum(acc[i]);
    // ---- loss + d(head outputs): every lane computes the same values
    float dl[HEAD_AMAX], dv;
    LOSS::template sample<HEAD_AMAX>(a, b, lane, acc, dl, dv, lsum, dbp, dbv, dls);
    // ---- head weight gradients (registers) and gradient wrt the hidden units
#pragma unroll
    for (int j = 0; j < HEAD_KPL; j++) {
      if (j < kpl) {
        int k = lane + 32 * j;
        float gp = 0.f;
#pragma unroll
        for (int i = 0; i < HEAD_AMAX; i++) { dwp[j][i] = fmaf(hp_[j], dl[i], dwp[j][i]); gp = fmaf(dl[i], wpi[j][i], gp); }
        dwv[j] = fmaf(hv_[j], dv, dwv[j]);
        float gv = dv * wv[j];
        long long eo = (long long)b * K + k;
        if (a.shared) {
          float r = (gp + gv) * act_grad_from_out(a.act_pi, hp_[j]);
          a.g_pi[eo] = r; f32_store_plane(a.gp_hi, a.gp_lo, ((long long)(k >> 3) * a.pitch + b) * 8 + (k & 7), r);
          bh_pi[j] += r;
        } else {
          float r1 = gp * act_grad_from_out(a.act_pi, hp_[j]), r2 = gv * act_grad_from_out(a.act_v, hv_[j]);
          a.g_pi[eo] = r1; f32_store_plane(a.gp_hi, a.gp_lo, ((long long)(k >> 3) * a.pitch + b) * 8 + (k & 7), r1);
          a.g_v[eo] = r2; f32_store_plane(a.gv_hi, a.gv_lo, ((long long)(k >> 3) * a.pitch + b) * 8 + (k & 7), r2);
          bh_pi[j] += r1; bh_v[j] += r2;
        }
      }
    }
  }
  // plane rows [B, round16(B)) are read by the weight-gradient K loop (16 samples per MMA step): keep them zero
  for (int b = a.B + blockIdx.x * nwarp + warp; b < ((a.B + 15) & ~15); b += gridDim.x * nwarp) {
#pragma unroll
    for (int j = 0; j < HEAD_KPL; j++) {
      if (j < kpl) {
        int k = lane + 32 * j;
        long long e = ((long long)(k >> 3) * a.pitch + b) * 8 + (k & 7);
        f32_store_plane(a.gp_hi, a.gp_lo, e, 0.f);
        if (!a.shared) f32_store_plane(a.gv_hi, a.gv_lo, e, 0.f);
      }
    }
  }
  // ---- every warp parks its sums in its own row; the rows are added in warp order and written to this block's slab
  float* row = sh_dw + (size_t)warp * nacc;
#pragma unroll
  for (int j = 0; j < HEAD_KPL; j++) {
    if (j < kpl) {
      int k = lane + 32 * j;
#pragma unroll
      for (int i = 0; i < HEAD_AMAX; i++) if (i < A) row[k * A + i] = dwp[j][i];
      row[K * A + k] = dwv[j];
      row[K * A + K + k] = bh_pi[j];
      row[K * A + 2 * K + k] = a.shared ? 0.f : bh_v[j];
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) if (i < A) row[K * A + 3 * K + i] = dbp[i];
    row[K * A + 3 * K + A] = dbv;
    row[K * A + 3 * K + A + 1] = lsum;
    if (LOSS::kLogStd) {
#pragma unroll
      for (int i = 0; i < HEAD_AMAX; i++) if (i < A) row[K * A + 3 * K + A + 2 + i] = dls[i];
    }
  }
  __syncthreads();
  float* out = a.part + (size_t)blockIdx.x * a.slab;
  for (int e = threadIdx.x; e < nacc; e += blockDim.x) {
    float t = sh_dw[e];
    for (int w = 1; w < nwarp; w++) t += sh_dw[(size_t)w * nacc + e];
    out[e] = t;
  }
}

// Dueling combine layer (XTB_DUELING), one warp per sample: q = adv + (value - mean_a value) (xt/model/dqn/dqn_mlp.py:80-87)
__global__ void __launch_bounds__(256) dueling_fwd_kernel(const float* __restrict__ value, const float* __restrict__ adv, int B, int A,
                                                          float* __restrict__ q) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31, b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* v = value + (long long)b * A;
  float s = 0.f;
  for (int i = lane; i < A; i += 32) s += v[i];
  const float mean = warp_sum(s) / A, ad = adv[b];
  for (int i = lane; i < A; i += 32) q[(long long)b * A + i] = ad + (v[i] - mean);
}
// Its data gradient, g = dloss/dq: gvalue = (g - mean_a g) * act'(value), gadv = sum_a g * act'(adv), written or, when
// acc_v / acc_a is set, added to what another consumer of that tensor already wrote.
__global__ void __launch_bounds__(256) dueling_dgrad_kernel(const float* __restrict__ g, const float* __restrict__ value,
                                                            const float* __restrict__ adv, int B, int A, int act_v, int act_a,
                                                            int acc_v, int acc_a, float* __restrict__ gvalue, float* __restrict__ gadv) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31, b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* gr = g + (long long)b * A;
  float s = 0.f;
  for (int i = lane; i < A; i += 32) s += gr[i];
  s = warp_sum(s);
  const float mean = s / A;
  for (int i = lane; i < A; i += 32) {
    const long long e = (long long)b * A + i;
    const float r = (gr[i] - mean) * act_grad_from_out(act_v, value[e]);
    gvalue[e] = acc_v ? gvalue[e] + r : r;
  }
  if (lane == 0) {
    const float r = s * act_grad_from_out(act_a, adv[b]);
    gadv[b] = acc_a ? gadv[b] + r : r;
  }
}

// ------------------------------------------------------------------------------------------
// Diagonal Gaussian policy of PPO (xt/model/tf_dist.py:49-86, xt/model/ppo/ppo.py:75-83): mean = pi_latent [B, A],
// log_std = the A floats of the pi_logstd variable, std = exp(log_std).
// ------------------------------------------------------------------------------------------
constexpr float kHalfLog2Pi = 0.918938533204672742f;     // 0.5 log(2 pi)
constexpr float kGaussEntConst = 1.418938533204672742f;  // 0.5 (log(2 pi) + 1)

// standard normals n[0..4) of sample b, dimensions 4g..4g+3: one Philox call (counter (b, g, offset), the uniform
// mapping of categorical_draw, never 0 or 1) and Box-Muller on the two pairs of its words
__device__ inline void gauss_normals4(int b, int g, uint64_t seed, uint64_t offset, float (&n)[4]) {
  uint32_t c[4] = {(uint32_t)b, (uint32_t)g, (uint32_t)(offset & 0xffffffffu), (uint32_t)(offset >> 32)};
  philox4x32_10(c, (uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32));
#pragma unroll
  for (int p = 0; p < 2; p++) {
    const float u0 = (float)(c[2 * p] >> 8) * 5.9604644775390625e-08f + 2.98023223876953125e-08f;
    const float u1 = (float)(c[2 * p + 1] >> 8) * 5.9604644775390625e-08f + 2.98023223876953125e-08f;
    const float r = sqrtf(-2.f * logf(u0));
    float s, co;
    sincospif(2.f * u1, &s, &co);
    n[2 * p] = r * co; n[2 * p + 1] = r * s;
  }
}

// DiagGaussianDist.sample + log_prob of sample b (xt/model/tf_dist.py:63-66, 85-86) with mean m[0..A), A <= n (as in
// categorical_draw): x_i = m_i + exp(log_std_i) n_i, n_i = nrm[i] when nrm is set, else normal i % 4 of gauss_normals4 at
// counter (b, i / 4, offset).  Writes x to row b of action and, when head_out is set, the mean to its row b; returns
// logp = -neglog_prob(x), computed from x.
template <class M>
__device__ __forceinline__ float gaussian_draw(const M& m, int n, int A, const float* log_std, const float* nrm, int b,
                                               uint64_t seed, uint64_t offset, float* action, float* head_out) {
  float q = 0.f, sls = 0.f, n4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < n; i++) {
    if (i < A) {
      float nv;
      if (nrm) {
        nv = nrm[i];
      } else {
        if ((i & 3) == 0) gauss_normals4(b, i >> 2, seed, offset, n4);
        nv = (i & 3) == 0 ? n4[0] : (i & 3) == 1 ? n4[1] : (i & 3) == 2 ? n4[2] : n4[3];
      }
      const float ls = log_std[i], sd = expf(ls);
      const float x = m[i] + sd * nv;
      const float z = (x - m[i]) / sd;
      q += z * z; sls += ls;
      action[(long long)b * A + i] = x;
      if (head_out) head_out[(long long)b * A + i] = m[i];
    }
  }
  return -((kHalfLog2Pi * (float)A + 0.5f * q) + sls);
}

// Gaussian PPO loss of one sample: actor loss with entropy + clipped critic loss (xt/model/ppo/__init__.py:4-25) on its
// mean m[0..A), A <= N, value vv and log_std[0..A).  x = the behaviour action of rollout row r; with std = exp(log_std)
// and z_i = (x_i - m_i) / std_i:
//   dlogp/dmean_i = z_i / std_i,  dlogp/dlog_std_i = z_i^2 - 1,  dH/dlog_std_i = 1
// Writes dm[i] = d loss / d mean_i for i < A, adds the sample's d loss / d log_std_i to dls[i] when add_ls is set, sets
// dv = d loss / d v and returns the sample's loss term.
template <int N, class M, class DM>
__device__ __forceinline__ float ppo_gauss_row(const M& m, const float* log_std, int A, float vv, int r, const float* action,
                                               const float* old_logp, const float* adv, const float* old_v, const float* target_v,
                                               const PpoHyperDev& hp, float inv_count, DM& dm, float (&dls)[N], bool add_ls,
                                               float& dv) {
  const float* x = action + (long long)r * A;
  float sd[N], z[N], q = 0.f, sls = 0.f, H = 0.f;
#pragma unroll
  for (int i = 0; i < N; i++) {
    sd[i] = 1.f; z[i] = 0.f;
    if (i < A) {
      const float ls = log_std[i];
      const float mi = m[i];
      sd[i] = expf(ls);
      z[i] = (x[i] - mi) / sd[i];
      q += z[i] * z[i]; sls += ls; H += ls + kGaussEntConst;
    }
  }
  const float logp_a = -((kHalfLog2Pi * (float)A + 0.5f * q) + sls);
  const PpoClipTerms c = ppo_clip_terms(logp_a, old_logp[r], adv[r], vv, old_v[r], target_v[r], hp, inv_count);
  dv = c.dv;
#pragma unroll
  for (int i = 0; i < N; i++) if (i < A) dm[i] = -c.dsurr * (z[i] / sd[i]) * inv_count;
#pragma unroll
  for (int i = 0; i < N; i++) if (i < A && add_ls) dls[i] += (-c.dsurr * (z[i] * z[i] - 1.f) - hp.ent_coef) * inv_count;
  return (-c.surr - hp.ent_coef * H + c.critic) * inv_count;
}

// ppo_gauss_row over a minibatch, one block, a thread per sample: dmean / dv per sample; dlog_std and the loss are
// summed over the samples in a fixed order (warp butterflies, then the warps in order), so the result is reproducible.
// AMAX >= A.
constexpr int GAUSS_LOSS_THREADS = 256;
template <int AMAX>
__global__ void __launch_bounds__(GAUSS_LOSS_THREADS)
ppo_gauss_loss_kernel(const float* __restrict__ mean, const float* __restrict__ v, const float* __restrict__ log_std,
                      const int32_t* __restrict__ idx, const float* __restrict__ action, const float* __restrict__ old_logp,
                      const float* __restrict__ adv, const float* __restrict__ old_v, const float* __restrict__ target_v,
                      int B, int A, PpoHyperDev hp, float inv_count, float* __restrict__ dmean, float* __restrict__ dv,
                      float* __restrict__ dlog_std, float* __restrict__ loss_out) {
  pdl_wait(); pdl_trigger();
  __shared__ float red[GAUSS_LOSS_THREADS / 32][AMAX + 1];
  float acc[AMAX];
#pragma unroll
  for (int i = 0; i < AMAX; i++) acc[i] = 0.f;
  float lsum = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float* dm = dmean + (long long)b * A;
    lsum += ppo_gauss_row(mean + (long long)b * A, log_std, A, v[b], idx ? idx[b] : b, action, old_logp, adv, old_v, target_v, hp,
                          inv_count, dm, acc, true, dv[b]);
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  lsum = warp_sum(lsum);
  if (lane == 0) red[w][AMAX] = lsum;
#pragma unroll
  for (int i = 0; i < AMAX; i++) {
    const float s = warp_sum(acc[i]);
    if (lane == 0) red[w][i] = s;
  }
  __syncthreads();
  if ((int)threadIdx.x <= AMAX && ((int)threadIdx.x < A || (int)threadIdx.x == AMAX)) {
    float s = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); k++) s += red[k][threadIdx.x];
    if ((int)threadIdx.x == AMAX) *loss_out += s;
    else dlog_std[threadIdx.x] = s;
  }
}

// heads_kernel policy of the Gaussian PPO step: ppo_gauss_row on mean = acc[0..A) + b_pi and v = acc[HEAD_AMAX] + b_v;
// lane 0 adds the per-sample log_std gradient to dls (the extra A slab floats, reduced in block order).
struct PpoGaussLoss {
  static constexpr bool kLogStd = true;
  template <int HEAD_AMAX>
  static __device__ __forceinline__ void sample(const PpoHeadsArgs& a, int b, int lane, const float (&acc)[HEAD_AMAX + 1],
                                                float (&dl)[HEAD_AMAX], float& dv, float& lsum, float (&dbp)[HEAD_AMAX],
                                                float& dbv, float (&dls)[HEAD_AMAX]) {
    const int A = a.A;
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) dl[i] = 0.f;
    const int r = a.idx ? a.idx[b] : b;
    float mean[HEAD_AMAX];
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) mean[i] = (i < A) ? acc[i] + a.b_pi[i] : 0.f;
    const float vv = acc[HEAD_AMAX] + a.b_v[0];
    const float l = ppo_gauss_row(mean, a.log_std, A, vv, r, a.action_f, a.old_logp, a.adv, a.old_v, a.target_v, a.hp, a.inv_count,
                                  dl, dls, lane == 0, dv);
    if (lane == 0) {
      lsum += l;
      if (a.v_out) a.v_out[b] = vv;
      dbv += dv;
#pragma unroll
      for (int i = 0; i < HEAD_AMAX; i++) {
        if (a.logits_out && i < A) a.logits_out[(long long)b * A + i] = mean[i];
        dbp[i] += dl[i];
      }
    }
  }
};

// Action distributions of the PPO pipeline.  Action: the action element, one per sample (Categorical: int32 [B]) or A
// per sample (DiagGaussian: float [B, A]); kLogStd: the policy owns the log_std parameters; Loss: its heads_kernel
// policy; draw: its draw of sample b from the pi head's output (logits / mean) with noise row nz (uniforms / standard
// normals) or, when nz is NULL, Philox at offset.  infer: the same draw in infer_heads_kernel, on the head sums acc (as
// in heads_kernel) plus b_pi; returns logp.
struct Categorical {
  using Action = int32_t;
  using Loss = PpoLoss;
  static constexpr bool kLogStd = false;
  __host__ __device__ static constexpr int action_width(int) { return 1; }
  template <int HEAD_AMAX>
  static __device__ __forceinline__ float infer(const float (&acc)[HEAD_AMAX + 1], const float* b_pi, const float*, int b, int A,
                                                uint64_t seed, uint64_t offset, int32_t* action, float* head_out) {
    float lg[HEAD_AMAX];
#pragma unroll
    for (int i = 0; i < HEAD_AMAX; i++) lg[i] = (i < A) ? acc[i] + b_pi[i] : -INFINITY;
    return categorical_draw(lg, HEAD_AMAX, A, nullptr, b, seed, offset, action, head_out);
  }
  template <class H>
  static __device__ __forceinline__ float draw(const H& head, int n, int A, const float*, const float* nz, int b, uint64_t seed,
                                               uint64_t offset, int32_t* action, float* head_out) {
    return categorical_draw(head, n, A, nz, b, seed, offset, action, head_out);
  }
};

struct DiagGaussian {
  using Action = float;
  using Loss = PpoGaussLoss;
  static constexpr bool kLogStd = true;
  __host__ __device__ static constexpr int action_width(int A) { return A; }
  template <int HEAD_AMAX>
  static __device__ __forceinline__ float infer(const float (&acc)[HEAD_AMAX + 1], const float* b_pi, const float* log_std, int b,
                                                int A, uint64_t seed, uint64_t offset, float* action, float* head_out) {
    struct {   // mean i, formed where gaussian_draw reads it
      const float (&acc)[HEAD_AMAX + 1]; const float* b_pi;
      __device__ float operator[](int i) const { return acc[i] + b_pi[i]; }
    } mean{acc, b_pi};
    return gaussian_draw(mean, HEAD_AMAX, A, log_std, nullptr, b, seed, offset, action, head_out);
  }
  template <class H>
  static __device__ __forceinline__ float draw(const H& head, int n, int A, const float* log_std, const float* nz, int b,
                                               uint64_t seed, uint64_t offset, float* action, float* head_out) {
    return gaussian_draw(head, n, A, log_std, nz, b, seed, offset, action, head_out);
  }
};

// One thread per sample: the draw of DIST from the pi head's output pi [B, A] with noise [B, A] if set, else Philox at
// `offset`, or at *offset_dev + t_add when offset_dev is set (the device-resident counter of rollout inference, so that
// CUDA-graph replays draw fresh noise).  log_std: DiagGaussian only.  v_out != NULL: the value head output is copied out
// alongside.
template <class DIST>
__global__ void sample_kernel(const float* __restrict__ pi, const float* __restrict__ log_std, int B, int A,
                              const float* __restrict__ noise, uint64_t seed, uint64_t offset,
                              const unsigned long long* __restrict__ offset_dev, int t_add,
                              typename DIST::Action* __restrict__ action, float* __restrict__ logp,
                              const float* __restrict__ v_in, float* __restrict__ v_out) {
  pdl_wait(); pdl_trigger();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (offset_dev) offset = (uint64_t)(*offset_dev) + (uint64_t)t_add;
  logp[b] = DIST::draw(pi + (long long)b * A, A, A, log_std, noise ? noise + (long long)b * A : nullptr, b, seed, offset, action,
                       nullptr);
  if (v_out) v_out[b] = v_in[b];
}

// Inference heads of PPO: the pi head (logits / mean) and the value head of one dense layer each, then the draw of
// DIST at Philox offset *offset_dev + t_add (the device-resident counter of rollout inference), in one kernel, one warp
// per sample.  log_std: DiagGaussian only.
template <class DIST, int HEAD_KPL, int HEAD_AMAX>
__global__ void __launch_bounds__(256)
infer_heads_kernel(const float* __restrict__ h_pi, const float* __restrict__ h_v, const float* __restrict__ w_pi,
                   const float* __restrict__ b_pi, const float* __restrict__ w_v, const float* __restrict__ b_v,
                   const float* __restrict__ log_std, int B, int K, int A, uint64_t seed,
                   const unsigned long long* __restrict__ offset_dev, int t_add, typename DIST::Action* __restrict__ action,
                   float* __restrict__ logp, float* __restrict__ v_out, float* __restrict__ head_out) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int kpl = K / 32;
  const uint64_t offset = (uint64_t)(*offset_dev) + (uint64_t)t_add;
  for (int b = blockIdx.x * nwarp + warp; b < B; b += gridDim.x * nwarp) {
    float acc[HEAD_AMAX + 1];
#pragma unroll
    for (int i = 0; i <= HEAD_AMAX; i++) acc[i] = 0.f;
#pragma unroll
    for (int j = 0; j < HEAD_KPL; j++) {
      if (j < kpl) {
        int k = lane + 32 * j;
        float hp = h_pi[(long long)b * K + k], hv = h_v[(long long)b * K + k];
#pragma unroll
        for (int i = 0; i < HEAD_AMAX; i++) if (i < A) acc[i] = fmaf(hp, w_pi[k * A + i], acc[i]);
        acc[HEAD_AMAX] = fmaf(hv, w_v[k], acc[HEAD_AMAX]);
      }
    }
#pragma unroll
    for (int i = 0; i <= HEAD_AMAX; i++) acc[i] = warp_sum(acc[i]);
    if (lane == 0) {
      logp[b] = DIST::template infer<HEAD_AMAX>(acc, b_pi, log_std, b, A, seed, offset, action, head_out);
      v_out[b] = acc[HEAD_AMAX] + b_v[0];
    }
  }
}

// ------------------------------------------------------------------------------------------
// IMPALA (xt/algorithm/impala/impala.py + xt/model/impala/impala_mlp.py, impala_cnn.py): the learner-side V-trace
// variant and the Keras softmax policy-gradient loss.
// ------------------------------------------------------------------------------------------
// probs = softmax(logits) row by row (the `output_actions` softmax of predict)
__global__ void softmax_rows_kernel(const float* __restrict__ logits, int B, int A, float* __restrict__ probs) {
  pdl_wait(); pdl_trigger();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* l = logits + (long long)b * A;
  float mx, lz;
  softmax_stats(l, A, mx, lz);
  for (int i = 0; i < A; i++) probs[(long long)b * A + i] = expf(l[i] - mx - lz);
}

// rho_t = min(1, exp(log(sum p_target y + 1e-10) - log(sum p_behav y + 1e-10)))   (impala.py:150-155, 186-189)
__device__ inline float keras_rho(const float* tl, const float* bp, const float* y, int A) {
  float mx, lz;
  softmax_stats(tl, A, mx, lz);
  float pt = 0.f, pb = 0.f;
  for (int i = 0; i < A; i++) { pt += expf(tl[i] - mx - lz) * y[i]; pb += bp[i] * y[i]; }
  return fminf(1.f, expf(logf(pt + 1e-10f) - logf(pb + 1e-10f)));
}

// IMPALA._train_proc (impala.py:124-184), one warp per trajectory of L steps and L+1 states:
//   delta_t = rho_t (r_t + disc_t V_{t+1} - V_t),  disc_t = (1 - done_t) gamma
//   adv_t   = delta_t + disc_{t+1} rho_{t+1} adv_{t+1},  adv_{L-1} = delta_{L-1}   (coefficients of the NEXT step)
//   tv_t    = V_t + adv_t;   pg_t = rho_t (r_t + disc_t tv_{t+1} - V_t),  tv_L = V_L (the bootstrap value)
// logits / value: the target head over the L+1 states of each trajectory; behav / amat / reward / done: the L steps.
// Lanes own consecutive time chunks; the affine maps adv_in -> a adv_in + b are scanned as in gae_kernel.
__global__ void impala_keras_vtrace_kernel(const float* __restrict__ logits, const float* __restrict__ value,
                                           const float* __restrict__ behav, const float* __restrict__ amat,
                                           const float* __restrict__ reward, const uint8_t* __restrict__ done, int n_traj,
                                           int L, int A, float gamma, float* __restrict__ pg_adv, float* __restrict__ tv) {
  pdl_wait(); pdl_trigger();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_traj) return;
  const long long sb = (long long)warp * (L + 1), tb = (long long)warp * L;   // first state row / first step row
  auto rho = [&](int t) { return keras_rho(logits + (sb + t) * A, behav + (tb + t) * A, amat + (tb + t) * A, A); };
  auto disc = [&](int t) { return done[tb + t] ? 0.f : gamma; };
  const int chunk = (L + 31) / 32, t0 = lane * chunk, t1 = min(L, t0 + chunk);
  // coefficient of adv_{t1} in adv_{t1-1}: disc_{t1} rho_{t1}, or 0 at the end of the trajectory
  const float c_edge = (t0 < t1 && t1 < L) ? disc(t1) * rho(t1) : 0.f;
  float a = 1.f, b = 0.f, c = c_edge;
  for (int t = t1 - 1; t >= t0; --t) {
    const float r = rho(t), d = disc(t);
    const float delta = r * (reward[tb + t] + d * value[sb + t + 1] - value[sb + t]);
    b = delta + c * b;
    a = c * a;
    c = d * r;
  }
  float fa = a, fb = b;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float oa = __shfl_down_sync(0xffffffffu, fa, o), ob = __shfl_down_sync(0xffffffffu, fb, o);
    if (lane + o < 32) { fb = fa * ob + fb; fa = fa * oa; }
  }
  float incoming = __shfl_down_sync(0xffffffffu, fb, 1);   // adv_{t1}
  if (lane == 31 || t1 >= L) incoming = 0.f;
  float adv_next = incoming, tv_next = value[sb + t1] + incoming;   // t1 == L: tv_L = V_L
  c = c_edge;
  for (int t = t1 - 1; t >= t0; --t) {
    const float r = rho(t), d = disc(t), V = value[sb + t], rw = reward[tb + t];
    const float adv = r * (rw + d * value[sb + t + 1] - V) + c * adv_next;
    const float tvt = V + adv;
    pg_adv[tb + t] = r * (rw + d * tv_next - V);
    tv[tb + t] = tvt;
    adv_next = adv; tv_next = tvt; c = d * r;
  }
}

// state row of training row i (the bootstrap state of every trajectory is skipped): i + i / L
__global__ void impala_keras_rows_kernel(const int32_t* __restrict__ order, int n, int L, int32_t* __restrict__ obs_idx) {
  pdl_wait(); pdl_trigger();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) { const int i = order[k]; obs_idx[k] = i + i / L; }
}

// Keras loss of ImpalaMlp / ImpalaCnn on softmax(logits) and the value head, minibatch rows b (data rows idx[b]):
//   l_b = mean_i [adv (-y_i log(p_i + 1e-10)) - ent (-p_i log(p_i + 1e-10))] + vw (v - tv)^2
// (impala_loss with loss weight 1, 'mse' with loss weight vw = 0.5).  The minibatch loss is mean_b l_b; the gradient
// goes through log(p + 1e-10) and the softmax Jacobian: dz_j = p_j (g_j - sum_i p_i g_i) / B with g_i = dl/dp_i.
// *loss_out += loss_scale * sum_b l_b.  One block: rows are summed in a fixed order, so the loss is reproducible.
constexpr int KERAS_LOSS_THREADS = 256;
__global__ void __launch_bounds__(KERAS_LOSS_THREADS)
impala_keras_loss_kernel(const float* __restrict__ logits, const float* __restrict__ v, const int32_t* __restrict__ idx,
                         const float* __restrict__ y, const float* __restrict__ adv, const float* __restrict__ tv, int B, int A,
                         float ent, float vw, float loss_scale, float* __restrict__ dlogits, float* __restrict__ dv,
                         float* __restrict__ loss_out) {
  pdl_wait(); pdl_trigger();
  __shared__ float red[KERAS_LOSS_THREADS / 32];
  const float inv_b = 1.f / B, inv_a = 1.f / A;
  float lsum = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int r = idx ? idx[b] : b;
    const float* l = logits + (long long)b * A;
    const float* yr = y + (long long)r * A;
    float mx, lz;
    softmax_stats(l, A, mx, lz);
    const float ad = adv[r];
    float f = 0.f, pg = 0.f;
    for (int i = 0; i < A; i++) {
      const float p = expf(l[i] - mx - lz), lp = logf(p + 1e-10f);
      f += ad * (-yr[i] * lp) - ent * (-p * lp);
      pg += p * (-ad * yr[i] / (p + 1e-10f) + ent * (lp + p / (p + 1e-10f)));
    }
    for (int i = 0; i < A; i++) {
      const float p = expf(l[i] - mx - lz), lp = logf(p + 1e-10f);
      const float g = -ad * yr[i] / (p + 1e-10f) + ent * (lp + p / (p + 1e-10f));
      dlogits[(long long)b * A + i] = p * (g - pg) * inv_a * inv_b;
    }
    const float dd = v[b] - tv[r];
    dv[b] = 2.f * vw * dd * inv_b;
    lsum += f * inv_a + vw * dd * dd;
  }
  lsum = warp_sum(lsum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += red[w];
    *loss_out += loss_scale * s;
  }
}

// Keras train_on_batch(states, y) with loss='mse': mean over B*A of (q-y)^2
__global__ void mse_loss_kernel(const float* __restrict__ q, const float* __restrict__ y, long long n,
                                float inv_count, float* __restrict__ dq, float* __restrict__ loss_out) {
  pdl_wait(); pdl_trigger();
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float lsum = 0.f;
  if (i < n) {
    float d = q[i] - y[i];
    dq[i] = 2.f * d * inv_count;
    lsum = d * d * inv_count;
  }
  block_atomic_add(lsum, loss_out);
}

// ------------------------------------------------------------------------------------------
// MuZero (xt/model/muzero/muzero_model.py, muzero_utils.py): categorical value / reward supports and the unrolled step
// ------------------------------------------------------------------------------------------
constexpr int MZ_MAX_SUPPORT = 1024;   // widest support (and action count) the warp-per-row kernels take
constexpr int MZ_THREADS = 256;        // 8 rows per block
// h(x) = sign(x) (sqrt(|x| + 1) - 1) + 0.001 x and its closed-form inverse (muzero_utils.py:38-47), in float64 as numpy
__device__ inline double mz_h(double x) { return (x > 0 ? 1.0 : (x < 0 ? -1.0 : 0.0)) * (sqrt(fabs(x) + 1.0) - 1.0) + 0.001 * x; }
__device__ inline double mz_h_inv(double x) {
  const double s = x > 0 ? 1.0 : (x < 0 ? -1.0 : 0.0);
  const double r = (sqrt(1.0 + 4.0 * 0.001 * (fabs(x) + 1.0 + 0.001)) - 1.0) / (2.0 * 0.001);
  return s * (r * r - 1.0);
}
// warp-wide softmax statistics of one row: max and log of the sum of exp(l - max)
__device__ inline void warp_softmax_stats(const float* l, int S, int lane, float& mx, float& lz) {
  mx = -INFINITY;
  for (int j = lane; j < S; j += 32) mx = fmaxf(mx, l[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float z = 0.f;
  for (int j = lane; j < S; j += 32) z += expf(l[j] - mx);
  lz = logf(warp_sum(z));
}

// conver_value (muzero_model.py:200-216): out row r = i * B + b holds the two-hot projection of x[b * T + i]:
// v = h(clip(x, min, max) - min), 1 - frac(v) at floor(v) and frac(v) at floor(v) + 1 (dropped past the support).
__global__ void mz_support_project_kernel(const float* __restrict__ x, int rows, int B, int T, int S, float vmin, float vmax,
                                          float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const int i = r / B, b = r - i * B;
  const double v = mz_h(fmin(fmax((double)x[(long long)b * T + i], (double)vmin), (double)vmax) - (double)vmin);
  const double fl = floor(v);
  const int idx = (int)fl;
  const float rest = (float)(v - fl);
  float* o = out + (long long)r * S;
  for (int j = lane; j < S; j += 32) o[j] = j == idx ? 1.f - rest : (j == idx + 1 ? rest : 0.f);
}

// value_transform (muzero_model.py:218-226) of softmax(logits[r]): clip(h_inv(sum_j p_j j) + min, min, max)
__global__ void mz_support_value_kernel(const float* __restrict__ logits, int rows, int S, float vmin, float vmax,
                                        float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* l = logits + (long long)r * S;
  float mx, lz;
  warp_softmax_stats(l, S, lane, mx, lz);
  double e = 0.0;
  for (int j = lane; j < S; j += 32) e += (double)expf(l[j] - mx - lz) * j;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
  if (lane == 0) out[r] = (float)fmin(fmax(mz_h_inv(e) + (double)vmin, (double)vmin), (double)vmax);
}

// cross_entropy (muzero_utils.py:31-34) of p = softmax(logits[r]) against target row t(r), t(r) = r when T == 0, else
// (r % B) * T + r / B (targets stored sample-major [B, T, S], rows step-major):
//   l_r = inv_bs * sum_j -t_j log(p_j + 1e-10),   inv_bs = 1 / (B S): the batch mean of the mean over the support
// dlogits[r] = gradient of g_r l_r through log(p + 1e-10) and the softmax Jacobian, g_r = 1 for r < full_rows and
// g_rest after (the 1/K gradient scale of the unrolled terms); the value is not scaled.  part[block] = the sum of its
// rows' l_r, warp by warp in order: with mz_ordered_sum_kernel the loss has no atomics and a fixed summation order.
__global__ void __launch_bounds__(MZ_THREADS)
mz_support_ce_kernel(const float* __restrict__ logits, int rows, int S, const float* __restrict__ tgt, int B, int T, int full_rows,
                     float g_rest, float inv_bs, float* __restrict__ dlogits, float* __restrict__ part) {
  pdl_wait(); pdl_trigger();
  __shared__ float red[MZ_THREADS / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * (MZ_THREADS / 32) + warp;
  float lrow = 0.f;
  if (r < rows) {
    const float* l = logits + (long long)r * S;
    const long long tr = T ? (long long)(r % B) * T + r / B : r;
    const float* t = tgt + tr * S;
    float mx, lz;
    warp_softmax_stats(l, S, lane, mx, lz);
    const float c = (r < full_rows ? 1.f : g_rest) * inv_bs;
    float f = 0.f, pg = 0.f;
    for (int j = lane; j < S; j += 32) {
      const float p = expf(l[j] - mx - lz);
      f += -t[j] * logf(p + 1e-10f);
      pg += p * (-c * t[j] / (p + 1e-10f));
    }
    f = warp_sum(f); pg = warp_sum(pg);
    for (int j = lane; j < S; j += 32) {
      const float p = expf(l[j] - mx - lz);
      dlogits[(long long)r * S + j] = p * (-c * t[j] / (p + 1e-10f) - pg);
    }
    lrow = f * inv_bs;
  }
  if (lane == 0) red[warp] = lrow;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < MZ_THREADS / 32; w++) s += red[w];
    part[blockIdx.x] = s;
  }
}

// *out = offset + sum of part[0..n) in a fixed order (one block)
__global__ void mz_ordered_sum_kernel(const float* __restrict__ part, int n, float offset, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  __shared__ float red[MZ_THREADS];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += MZ_THREADS) s += part[i];
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = offset;
    for (int w = 0; w < MZ_THREADS; w++) t += red[w];
    *out = t;
  }
}

// the dynamics input concat(hidden, one_hot(action)) (muzero_model.py:120-123, 57-61): x[b] = [h[b, 0..H), e_a],
// a = action[b * a_ld + a_col]
__global__ void mz_concat_onehot_kernel(const float* __restrict__ h, int B, int H, const int32_t* __restrict__ action, int a_ld,
                                        int a_col, int A, float* __restrict__ x) {
  pdl_wait(); pdl_trigger();
  const long long n = (long long)B * (H + A);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / (H + A)), j = (int)(i - (long long)b * (H + A));
    x[i] = j < H ? h[(long long)b * H + j] : (j - H == action[(long long)b * a_ld + a_col] ? 1.f : 0.f);
  }
}

// gradient wrt the pre-activation of a hidden state h [B, H] with activation `act`: the prediction network's input
// gradient g plus c times the hidden part of the next dynamics step's input gradient dx [B, ld] (none: dx == NULL)
__global__ void mz_hidden_grad_kernel(const float* __restrict__ g, const float* __restrict__ dx, int ld, float c,
                                      const float* __restrict__ h, int act, int B, int H, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  const long long n = (long long)B * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / H, j = i - b * H;
    const float d = g[i] + (dx ? c * dx[b * ld + j] : 0.f);
    out[i] = d * act_grad_from_out(act, h[i]);
  }
}

// dst += src (the gradient of one dynamics application into the shared gradient buffer, step by step in order)
__global__ void mz_accumulate_kernel(float* __restrict__ dst, const float* __restrict__ src, long long n) {
  pdl_wait(); pdl_trigger();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] += src[i];
}

// ------------------------------------------------------------------------------------------
// MuZero tree search (xt/agent/muzero/mcts.py, util.py): N trees advanced in lock step, one warp per tree
// ------------------------------------------------------------------------------------------
// Node 0 is the root; simulation s (1-based) expands node s.  Every expanded node has A child edges (prior, visit count,
// value sum, expanded child node or -1); the root's own statistics live apart.  The statistics are float64, as NumPy 1.x
// evaluated the reference's float32 priors times Python floats, and every product is rounded before it is added
// (__dmul_rn / __dadd_rn: no contraction into fma, so the sums are the ones the reference's Python evaluates).
struct MctsTrees {
  int E, NN, A, H;         // trees allocated, nodes per tree (1 + max simulations), actions, hidden width
  float* hid;              // [NN][E][H] hidden state of every expanded node (node-major: one simulation's rows are contiguous)
  double* reward;          // [E][NN] node reward
  double* prior;           // [E][NN][A] edge prior
  double* vsum;            // [E][NN][A] edge value sum
  int* visits;             // [E][NN][A] edge visit count
  int* child;              // [E][NN][A] expanded child node, -1 while unexpanded
  double* root_vsum;       // [E]
  int* root_visits;        // [E]
  double* minmax;          // [E][2] MinMaxStats(None): minimum, maximum
  int* path_node;          // [E][NN] search path: parent node and action of every step
  int* path_act;           // [E][NN]
  int* depth;              // [E] steps on the current path
};
constexpr int MCTS_THREADS = 128;   // 4 trees per block

__device__ inline void mcts_minmax_update(double* mm, double v) {   // Python's min / max keep the first of equals
  if (v < mm[0]) mm[0] = v;
  if (v > mm[1]) mm[1] = v;
}

// root of tree e from the initial inference's policy: priors prior * (1 - frac) + noise * frac when noise is given
__global__ void __launch_bounds__(MCTS_THREADS)
mcts_root_kernel(MctsTrees t, int N, const float* __restrict__ policy, const double* __restrict__ noise, double frac) {
  pdl_wait(); pdl_trigger();
  const int e = blockIdx.x * (MCTS_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (e >= N) return;
  const int A = t.A;
  const long long base = (long long)e * t.NN * A;
  for (int a = lane; a < A; a += 32) {
    double p = (double)policy[(long long)e * A + a];
    if (noise) p = __dadd_rn(__dmul_rn(p, 1.0 - frac), __dmul_rn(noise[(long long)e * A + a], frac));
    t.prior[base + a] = p;
    t.vsum[base + a] = 0.0;
    t.visits[base + a] = 0;
    t.child[base + a] = -1;
  }
  if (lane == 0) {
    t.reward[(long long)e * t.NN] = 0.0;
    t.root_vsum[e] = 0.0;
    t.root_visits[e] = 0;
    t.minmax[2 * e] = INFINITY;
    t.minmax[2 * e + 1] = -INFINITY;
  }
}

// One descent per tree (Mcts.run_mcts / select_child / ucb_score): from the root, while the chosen child is expanded,
// pick the child of the largest (ucb, action) -- ties go to the higher action, as max() over the reference's tuples --
//   ucb = (log((N_p + pb_c_base + 1) / pb_c_base) + pb_c_init) * (sqrt(N_p) / (N_c + 1)) * prior
//         + (N_c > 0 ? normalize(value_sum / N_c) : 0)
// Records the path, and writes the dynamics input concat(hidden of the leaf's parent, one_hot(action)) as row e of x
// [N, H + A] (the layout mz_concat_onehot_kernel writes).
__global__ void __launch_bounds__(MCTS_THREADS)
mcts_select_kernel(MctsTrees t, int N, double pb_c_base, double pb_c_init, float* __restrict__ x) {
  pdl_wait(); pdl_trigger();
  const int e = blockIdx.x * (MCTS_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (e >= N) return;
  const int A = t.A, NN = t.NN;
  const long long base = (long long)e * NN * A;
  const double mn = t.minmax[2 * e], mx = t.minmax[2 * e + 1];
  int node = 0, np = t.root_visits[e], d = 0, act;
  while (true) {
    const double pb = __dadd_rn(log(__dadd_rn(__dadd_rn((double)np, pb_c_base), 1.0) / pb_c_base), pb_c_init);
    const double sq = sqrt((double)np);
    double best = -INFINITY;
    int besta = -1;
    for (int a = lane; a < A; a += 32) {
      const long long i = base + (long long)node * A + a;
      const int nc = t.visits[i];
      double s = __dmul_rn(__dmul_rn(pb, sq / (double)(nc + 1)), t.prior[i]);
      if (nc > 0) {
        const double v = t.vsum[i] / (double)nc;
        s = __dadd_rn(s, mx > mn ? (v - mn) / (mx - mn) : v);
      }
      if (s > best || (s == best && a > besta)) { best = s; besta = a; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double s2 = __shfl_xor_sync(0xffffffffu, best, o);
      const int a2 = __shfl_xor_sync(0xffffffffu, besta, o);
      if (s2 > best || (s2 == best && a2 > besta)) { best = s2; besta = a2; }
    }
    act = besta < 0 ? 0 : besta;   // only when every score is NaN
    if (lane == 0) { t.path_node[(long long)e * NN + d] = node; t.path_act[(long long)e * NN + d] = act; }
    d++;
    const long long i = base + (long long)node * A + act;
    const int c = t.child[i];
    if (c < 0) break;
    np = t.visits[i];
    node = c;
  }
  if (lane == 0) t.depth[e] = d;
  const int H = t.H;
  const float* h = t.hid + ((long long)node * t.E + e) * H;
  float* xr = x + (long long)e * (H + A);
  for (int j = lane; j < H; j += 32) xr[j] = h[j];
  for (int j = lane; j < A; j += 32) xr[H + j] = j == act ? 1.f : 0.f;
}

// Expansion of node s (init_node) from the recurrent inference's reward and policy, then Mcts.backpropagate from the
// leaf to the root: value_sum += v, visit_count += 1, minmax.update(value()), v = reward + discount * v.  The node's
// hidden row was written into t.hid by the inference.
__global__ void __launch_bounds__(MCTS_THREADS)
mcts_expand_backup_kernel(MctsTrees t, int N, int s, const float* __restrict__ reward, const float* __restrict__ value,
                          const float* __restrict__ policy, double discount) {
  pdl_wait(); pdl_trigger();
  const int e = blockIdx.x * (MCTS_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (e >= N) return;
  const int A = t.A, NN = t.NN;
  const long long base = (long long)e * NN * A, nb = base + (long long)s * A;
  for (int a = lane; a < A; a += 32) {
    t.prior[nb + a] = (double)policy[(long long)e * A + a];
    t.vsum[nb + a] = 0.0;
    t.visits[nb + a] = 0;
    t.child[nb + a] = -1;
  }
  if (lane != 0) return;
  const int d = t.depth[e];
  const int* pn = t.path_node + (long long)e * NN;
  const int* pa = t.path_act + (long long)e * NN;
  t.child[base + (long long)pn[d - 1] * A + pa[d - 1]] = s;
  t.reward[(long long)e * NN + s] = (double)reward[e];
  double* mm = t.minmax + 2 * e;
  double v = (double)value[e];
  for (int k = d - 1; k >= 0; k--) {
    const long long i = base + (long long)pn[k] * A + pa[k];
    const double sum = __dadd_rn(t.vsum[i], v);
    const int n = t.visits[i] + 1;
    t.vsum[i] = sum;
    t.visits[i] = n;
    mcts_minmax_update(mm, sum / (double)n);
    v = __dadd_rn(t.reward[(long long)e * NN + t.child[i]], __dmul_rn(discount, v));
  }
  const double sum = __dadd_rn(t.root_vsum[e], v);
  const int n = t.root_visits[e] + 1;
  t.root_vsum[e] = sum;
  t.root_visits[e] = n;
  mcts_minmax_update(mm, sum / (double)n);
}

// get_info: root child visit counts [N, A] and root value value_sum / visit_count [N]
__global__ void __launch_bounds__(MCTS_THREADS)
mcts_result_kernel(MctsTrees t, int N, int32_t* __restrict__ counts, double* __restrict__ root_value) {
  pdl_wait(); pdl_trigger();
  const int e = blockIdx.x * (MCTS_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (e >= N) return;
  const int A = t.A;
  for (int a = lane; a < A; a += 32) counts[(long long)e * A + a] = t.visits[(long long)e * t.NN * A + a];
  if (lane == 0) root_value[e] = t.root_vsum[e] / (double)t.root_visits[e];
}

}  // namespace xtb
