// agent_act.cuh -- acting for many environments of one QMIX / SCC agent network in one call (xtb_qmix_act, xtb_scc_act):
// the agent inputs of QMixAlg.build_inputs for one step with per-environment episode resets, and the masked epsilon-greedy
// choice of EpsilonGreedyActionSelector.select_action (xt/algorithm/qmix/qmix_alg.py).  fc1 -> GRU -> fc2 run between
// the two kernels on the N n agent rows (row r = e n + a: environment e, agent a), with every environment's hidden state
// in the caller's [N, n, H] buffer.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "launch.cuh"
#include "philox.cuh"

namespace xtb {

constexpr int AA_THREADS = 256;

// Row r of the inputs x [N n, W], W = o (+ A with last_on) (+ n with id_on): obs[r] (o floats), then the one-hot of
// last_action[r] (zeros when environment e is reset or the action is < 0), then the one-hot of a.  A reset environment
// also gets zero hidden rows and last actions -1 (no previous action).  With `counter` (the Philox draws of the choice),
// counter[e] advances by one for every environment.
__global__ void __launch_bounds__(AA_THREADS)
agent_act_inputs_kernel(const float* __restrict__ obs, const int32_t* __restrict__ reset, int32_t* __restrict__ last_action,
                        float* __restrict__ hidden, unsigned long long* __restrict__ counter, float* __restrict__ x, int N, int n, int o,
                        int A, int H, int last_on, int id_on) {
  pdl_wait(); pdl_trigger();
  const int W = o + (last_on ? A : 0) + (id_on ? n : 0);
  const long long rows = (long long)N * n, stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long i = tid; i < rows * W; i += stride) {
    const long long r = i / W;
    const int c = (int)(i - r * W), a = (int)(r % n);
    float v;
    if (c < o) {
      v = obs[r * o + c];
    } else if (last_on && c < o + A) {
      v = !reset[r / n] && last_action[r] == c - o ? 1.f : 0.f;
    } else {
      v = c - o - (last_on ? A : 0) == a ? 1.f : 0.f;
    }
    x[i] = v;
  }
  for (long long i = tid; i < rows * H; i += stride)
    if (reset[i / ((long long)n * H)]) hidden[i] = 0.f;
  for (long long r = tid; r < rows; r += stride)
    if (reset[r / n]) last_action[r] = -1;
  if (counter)
    for (long long e = tid; e < N; e += stride) counter[e] += 1;
}

// A uniform double in [0, 1) from 53 bits of two Philox words, as numpy's random_sample builds one from two 32-bit draws
__device__ __forceinline__ double aa_u53(uint32_t a, uint32_t b) {
  return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0);
}

// One thread per agent row r = e n + a: q [N n, A] (fc2's output), avail [N n, A] action weights, eps [N].
//   greedy = the first maximum of q with the actions of weight < 1e-6 at -inf (np.argmax: a NaN is the maximum);
//   random = searchsorted(cdf, u1, side="right") with cdf the sequential float64 cumsum of avail / sum(avail), divided by
//            its last element (np.random.choice(A, p=...));
//   action = random if u0 < eps[e] else greedy, written to actions[r] and last_action[r].
// (u0, u1) = (uniforms[e, 0, a], uniforms[e, 1, a]) when uniforms is set, else 53-bit uniforms from the words (0, 1) and
// (2, 3) of Philox4x32-10 on counter (a, e, counter[e]) with key seed.  A row without a positive weight gets an action in
// [0, A) that means nothing (the callers reject such rows).
__global__ void __launch_bounds__(AA_THREADS)
agent_act_select_kernel(const float* __restrict__ q, const int32_t* __restrict__ avail, const double* __restrict__ eps,
                        const double* __restrict__ uniforms, unsigned long long seed, const unsigned long long* __restrict__ counter,
                        int32_t* __restrict__ actions, int32_t* __restrict__ last_action, int N, int n, int A) {
  pdl_wait(); pdl_trigger();
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= (long long)N * n) return;
  const int e = (int)(r / n), a = (int)(r % n);
  const float* qr = q + r * A;
  const int32_t* av = avail + r * A;
  float best = 0.f;
  int greedy = -1;
  long long total = 0;
  for (int j = 0; j < A; j++) {
    const float v = av[j] > 0 ? qr[j] : -INFINITY;
    if (greedy < 0 || v > best || (v != v && best == best)) { best = v; greedy = j; }
    total += av[j];
  }
  double u0, u1;
  if (uniforms) {
    u0 = uniforms[(long long)e * 2 * n + a];
    u1 = uniforms[(long long)e * 2 * n + n + a];
  } else {
    const unsigned long long k = counter[e];
    uint32_t c[4] = {(uint32_t)a, (uint32_t)e, (uint32_t)(k & 0xffffffffu), (uint32_t)(k >> 32)};
    philox4x32_10(c, (uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32));
    u0 = aa_u53(c[0], c[1]);
    u1 = aa_u53(c[2], c[3]);
  }
  const double s = (double)total;
  double last = 0.0;
  for (int j = 0; j < A; j++) last = __dadd_rn(last, __ddiv_rn((double)av[j], s));
  double cum = 0.0;
  int pick = 0;
  for (int j = 0; j < A; j++) {
    cum = __dadd_rn(cum, __ddiv_rn((double)av[j], s));
    if (__ddiv_rn(cum, last) <= u1) pick++;
  }
  const int act = u0 < eps[e] ? min(pick, A - 1) : greedy;
  actions[r] = act;
  last_action[r] = act;
}

}  // namespace xtb
