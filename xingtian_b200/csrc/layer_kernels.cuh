// layer_kernels.cuh -- the layer engine's element-wise CUDA-core kernels: the activations past tanh (see gemm_f32.cuh)
// and the dueling combine layer.
#pragma once
#include <cuda_runtime.h>

#include "gemm_f32.cuh"

namespace xtb {

// y[i] = act(pre[i]) over n floats (pre may be y itself)
__global__ void act_fwd_kernel(const float* pre, long long n, int act, float* y) {
  pdl_wait(); pdl_trigger();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = act_apply_ext(act, pre[i]);
}
// g *= act'(u) over rows x N (u: z or y, act_grad_ext): the gradient wrt the output becomes the gradient wrt the
// pre-activation.  Also the layer's bias gradient, without atomics: block b takes a fixed run of rows, its row lanes
// add in a fixed order, and part[b][N] is left for the ordered reduction (bp::grad_reduce_kernel).
constexpr int ACT_BWD_BLOCKS = 132, ACT_BWD_THREADS = 256;
__global__ void __launch_bounds__(ACT_BWD_THREADS) act_bwd_kernel(float* __restrict__ g, const float* __restrict__ u, int rows,
                                                                  int N, int act, float* __restrict__ part) {
  pdl_wait(); pdl_trigger();
  __shared__ float red[ACT_BWD_THREADS];
  const int rpb = (rows + gridDim.x - 1) / gridDim.x, r0 = blockIdx.x * rpb, r1 = min(rows, r0 + rpb);
  const int W = min(N, ACT_BWD_THREADS), R = ACT_BWD_THREADS / W;      // columns per pass, row lanes
  const int rr = threadIdx.x / W;
  for (int c0 = 0; c0 < N; c0 += W) {
    const int c = c0 + threadIdx.x % W;
    float s = 0.f;
    if (rr < R && c < N)
      for (int r = r0 + rr; r < r1; r += R) {
        const long long e = (long long)r * N + c;
        const float v = g[e] * act_grad_ext(act, u[e]);
        g[e] = v;
        s += v;
      }
    red[threadIdx.x] = s;
    __syncthreads();
    if (rr == 0 && c < N) {
      float t = red[threadIdx.x];
      for (int k = 1; k < R; k++) t += red[k * W + threadIdx.x];
      part[(long long)blockIdx.x * N + c] = t;
    }
    __syncthreads();
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

}  // namespace xtb
