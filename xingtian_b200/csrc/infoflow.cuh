// infoflow.cuh -- the InfoFlow recommender DQN (xt/model/dqn/dqn_rec_model.py, xt/algorithm/dqn/dqn_infoflw_alg.py):
// the frozen-embedding gather of the GRU inputs, the assembly of the head's input rows (one per candidate item of a
// next state, or one per transition), the segmented max / TD target and the mse loss.  The two GRUs run on QMIX's
// kernels (qmix.cuh) in the Keras GRU v1 form; the dense head runs on the layer engine.
//
// Ids are int32 (Keras Embedding's cast) in [0, vocab), checked on the host.  A head input row of width
// D = user_dim E + 2U + item_dim E (U = item_dim E) is [Flatten(emb(user)) | h_click | h_noclick | Flatten(emb(item))].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "gemm_f32.cuh"
#include "launch.cuh"

namespace xtb {

constexpr int IF_THREADS = 256;     // row kernels: one warp per row, 8 rows per block
constexpr int IF_HIST = 5;          // n_history_click = n_history_no_click = 5

// out[i] = table[ids[i / E] * E + i % E] for i < n: Flatten / Reshape of an Embedding lookup.  Both histories of B
// transitions at once ([B][5 item_dim] ids each -> GRU step inputs [B][5][U], row b * 5 + t).
__global__ void __launch_bounds__(IF_THREADS)
infoflow_gather_kernel(const int32_t* __restrict__ ids0, const int32_t* __restrict__ ids1, const float* __restrict__ table, long long n,
                       int E, float* __restrict__ out0, float* __restrict__ out1) {
  pdl_wait(); pdl_trigger();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < 2 * n; i += (long long)gridDim.x * blockDim.x) {
    const bool second = i >= n;
    const long long k = second ? i - n : i;
    const int32_t id = (second ? ids1 : ids0)[k / E];
    (second ? out1 : out0)[k] = table[(long long)id * E + k % E];
  }
}

// Head input rows x [cap, D]: row c < off[B] belongs to the transition b with off[b] <= c < off[b + 1] and is
// [emb(user[b]) | hc[b] | hn[b] | emb(item ids of row c)], hc / hn [B, U] the GRUs' last outputs; rows in
// [off[B], cap) are zeroed (padding, never read).  Candidate rows of the target pass: off = the candidate offsets and
// item = the candidates' ids; rows of the training pass: off = 0, 1, ..., B and item = the transitions' items.
__global__ void __launch_bounds__(IF_THREADS)
infoflow_rows_kernel(const int32_t* __restrict__ user, const int32_t* __restrict__ item, const int32_t* __restrict__ off,
                     const float* __restrict__ hc, const float* __restrict__ hn, const float* __restrict__ table, int B, int cap,
                     int user_dim, int item_dim, int E, float* __restrict__ x) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int U = item_dim * E, Du = user_dim * E, D = Du + 2 * U + U;
  const int total = off[B];
  for (int c = blockIdx.x * (IF_THREADS / 32) + (threadIdx.x >> 5); c < cap; c += gridDim.x * (IF_THREADS / 32)) {
    float* xr = x + (long long)c * D;
    if (c >= total) {
      for (int j = lane; j < D; j += 32) xr[j] = 0.f;
      continue;
    }
    int lo = 0, hi = B;            // the last b with off[b] <= c
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (off[mid] <= c) lo = mid; else hi = mid; }
    const int32_t* ub = user + (long long)lo * user_dim;
    const int32_t* ic = item + (long long)c * item_dim;
    for (int j = lane; j < Du; j += 32) xr[j] = table[(long long)ub[j / E] * E + j % E];
    for (int j = lane; j < U; j += 32) {
      xr[Du + j] = hc[(long long)lo * U + j];
      xr[Du + U + j] = hn[(long long)lo * U + j];
      xr[Du + 2 * U + j] = table[(long long)ic[j / E] * E + j % E];
    }
  }
}

// dqn_infoflw_alg.py:143-153 for every transition b (one warp each): target[b] = reward[b] when done[b], else
// max(q[off[b] .. off[b+1])) * gamma + reward[b] in float64 (NumPy's float32 scalar times a Python float), rounded to
// float32 as Keras casts the targets.  A NaN among the candidates is the max, as np.argmax picks the first NaN.
__global__ void __launch_bounds__(IF_THREADS)
infoflow_td_kernel(const float* __restrict__ q, const int32_t* __restrict__ off, const double* __restrict__ reward,
                   const int32_t* __restrict__ done, int B, double gamma, float* __restrict__ target) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (IF_THREADS / 32) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int c0 = off[b], c1 = off[b + 1];
  float m = -INFINITY;
  bool nan = false;
  for (int c = c0 + lane; c < c1; c += 32) { const float v = q[c]; nan |= v != v; m = fmaxf(m, v); }
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  nan = __any_sync(0xffffffffu, nan);
  if (lane == 0) target[b] = done[b] ? (float)reward[b] : (float)((double)(nan ? NAN : m) * gamma + reward[b]);
}

// Keras loss="mse" on the [B, 1] q_value output y (activation act) against target t, one block: loss = mean (y - t)^2
// (ordered sum), dy = 2 (y - t) / B wrt the output, times act'(y) when `pre` (linear, relu, tanh: the gradient wrt the
// pre-activation; the engine's act backward takes the activations past tanh from the output gradient).  The engine's
// mse_loss_kernel has neither the activation nor a fixed summation order.
__global__ void __launch_bounds__(IF_THREADS)
infoflow_mse_kernel(const float* __restrict__ y, const float* __restrict__ t, int B, int act, int pre, float* __restrict__ dy,
                    float* __restrict__ loss) {
  __shared__ float red[IF_THREADS];
  pdl_wait(); pdl_trigger();
  const float inv = 1.f / (float)B;
  float s = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float d = y[i] - t[i];
    const float g = 2.f * d * inv;
    dy[i] = pre ? g * act_grad_from_out(act, y[i]) : g;
    s += d * d;
  }
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int w = 0; w < IF_THREADS; w++) a += red[w];
    *loss = a * inv;
  }
}

}  // namespace xtb
