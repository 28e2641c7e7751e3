// episode_replay.cuh -- QMIX's and SCC's episode replay in HBM (xtb_episode_replay_* in xtb200.h): the ring of the
// reference's ReplayBufferNP (xt/algorithm/qmix/episode_buffer_np.py) and the training batch QMixAlg.train assembles from
// the drawn episodes (qmix_alg.py: build_inputs, the mask, max_t_filled), written straight into the model's batch buffers.
//
// Slot s of the ring is one contiguous episode row of T = episode_limit + 1 steps at ring + s row_bytes, its fields in
// this order, each starting 16-byte aligned (epr_layout):
//   state f32 [T, S] | obs f32 [T, n, o] | actions i32 [T, n] | actions_onehot f32 [T, n, A] | avail_actions i32 [T, n, A] |
//   reward f32 [T] | terminated u8 [T] | filled i64 [T]
// so that storing an episode is one host-to-device copy of a row packed on the host.  Every value the batch needs is a
// copy or one rounding of a stored value, the same rounding the host path's float32 staging applies.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/xtb200.h"
#include "launch.cuh"

namespace xtb {

// The device side of an xtb_episode_replay: the ring and the row layout (byte offsets within a row)
struct EprDev {
  uint8_t* ring;                      // [capacity, row_bytes]
  long long row_bytes;
  long long o_state, o_obs, o_act, o_onehot, o_avail, o_reward, o_term, o_filled;
  int T, n, o, S, A;
  int last_action, agent_id, width;   // build_inputs' switches; width = o (+ A) (+ n)
};

// the 16-byte aligned field offsets of a row, in the order above -> row bytes
inline long long epr_layout(EprDev& d) {
  const long long T = d.T, n = d.n;
  const long long sizes[8] = {T * d.S * 4, T * n * d.o * 4, T * n * 4, T * n * d.A * 4, T * n * d.A * 4, T * 4, T, T * 8};
  long long* offs[8] = {&d.o_state, &d.o_obs, &d.o_act, &d.o_onehot, &d.o_avail, &d.o_reward, &d.o_term, &d.o_filled};
  long long o = 0;
  for (int i = 0; i < 8; i++) { *offs[i] = o; o += (sizes[i] + 15) / 16 * 16; }
  d.row_bytes = o;
  return o;
}

constexpr int kEprThreads = 128;

// max_t_filled() of the drawn episodes: the largest per-episode sum of `filled`, into seq_len[0 .. B n) (the GRU sequence
// lengths train() hands the model) and *max_out.  One CTA: a warp sums one episode at a time.
__global__ void __launch_bounds__(256) epr_seq_len_kernel(EprDev d, const int32_t* __restrict__ ids, int B, int32_t* __restrict__ seq_len,
                                                          int32_t* __restrict__ max_out) {
  __shared__ long long best;
  if (threadIdx.x == 0) best = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  for (int b = warp; b < B; b += warps) {
    const int id = ids[b];
    long long s = 0;
    if (id >= 0) {
      const long long* f = reinterpret_cast<const long long*>(d.ring + (long long)id * d.row_bytes + d.o_filled);
      for (int t = lane; t < d.T; t += 32) s += f[t];
    }
    for (int k = 16; k; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    if (lane == 0) atomicMax(&best, s);
  }
  __syncthreads();
  const int m = (int)best;
  if (seq_len)
    for (int i = threadIdx.x; i < B * d.n; i += blockDim.x) seq_len[i] = m;
  if (max_out && threadIdx.x == 0) *max_out = m;
}

// Step t of drawn episode b (grid T x B): the agent inputs [obs | previous action's one-hot (zeros at t = 0) | agent-id
// one-hot], avail as float and, when requested, the raw obs; for t < L the action, state, next state, reward, terminated
// and mask = filled[t] (times 1 - terminated[t - 1] for t > 0), in float32 as the host computes it.  NULL outputs are
// skipped.
__global__ void __launch_bounds__(kEprThreads) epr_gather_kernel(EprDev d, const int32_t* __restrict__ ids, xtb_episode_batch out) {
  const int t = blockIdx.x, b = blockIdx.y, T = d.T, L = T - 1, n = d.n, o = d.o, A = d.A, W = d.width;
  const int id = ids[b];
  if (id < 0) return;
  const uint8_t* row = d.ring + (long long)id * d.row_bytes;
  const float* obs = reinterpret_cast<const float*>(row + d.o_obs) + (long long)t * n * o;
  const float* prev = reinterpret_cast<const float*>(row + d.o_onehot) + (long long)(t - 1) * n * A;
  const int32_t* avail = reinterpret_cast<const int32_t*>(row + d.o_avail) + (long long)t * n * A;
  const long long bt = (long long)b * T + t;
  if (out.obs) {
    float* dst = out.obs + bt * n * W;
    for (int i = threadIdx.x; i < n * W; i += blockDim.x) {
      const int a = i / W;
      int c = i - a * W;
      float v;
      if (c < o) {
        v = obs[a * o + c];
      } else {
        c -= o;
        if (d.last_action && c < A) v = t ? prev[a * A + c] : 0.f;
        else v = (c - (d.last_action ? A : 0)) == a ? 1.f : 0.f;
      }
      dst[i] = v;
    }
  }
  if (out.avail)
    for (int i = threadIdx.x; i < n * A; i += blockDim.x) out.avail[bt * n * A + i] = (float)avail[i];
  if (out.raw_obs)
    for (int i = threadIdx.x; i < n * o; i += blockDim.x) out.raw_obs[bt * n * o + i] = obs[i];
  if (t >= L) return;
  const long long bl = (long long)b * L + t;
  const float* state = reinterpret_cast<const float*>(row + d.o_state) + (long long)t * d.S;
  if (out.actions) {
    const int32_t* act = reinterpret_cast<const int32_t*>(row + d.o_act) + (long long)t * n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) out.actions[bl * n + i] = act[i];
  }
  if (out.state)
    for (int i = threadIdx.x; i < d.S; i += blockDim.x) out.state[bl * d.S + i] = state[i];
  if (out.next_state)
    for (int i = threadIdx.x; i < d.S; i += blockDim.x) out.next_state[bl * d.S + i] = state[d.S + i];
  if (threadIdx.x == 0) {
    const uint8_t* term = row + d.o_term;
    const float tm = (float)term[t];
    if (out.reward) out.reward[bl] = reinterpret_cast<const float*>(row + d.o_reward)[t];
    if (out.terminated) out.terminated[bl] = tm;
    if (out.mask) {
      float m = (float)reinterpret_cast<const long long*>(row + d.o_filled)[t];
      if (t > 0) m = __fmul_rn(m, __fsub_rn(1.f, (float)term[t - 1]));
      out.mask[bl] = m;
    }
  }
}

}  // namespace xtb
