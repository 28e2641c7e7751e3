// optim.cuh -- fused clip + Adam over one flat fp32 parameter bucket (HBM bound, 28 B/param).
//   tf.train.AdamOptimizer + tf.clip_by_global_norm : xt/model/ppo/ppo.py:97-102,
//                                                     xt/model/impala/impala_cnn_opt.py:198-217
//   keras Adam(clipnorm)                            : xt/model/dqn/dqn_cnn.py:60
// Two launches per step: sqnorm (per-segment sum of squares, one atomic per block; the last block to finish computes
// the clip scales, lr_t and the beta powers and re-zeroes the accumulators), adam (elementwise update that also
// refreshes the batch-planar weight blobs of the tensor-core layers, bp_gemm.cuh).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "bp_gemm.cuh"
#include "launch.cuh"

namespace xtb {

constexpr int OPT_CHUNK = 1024;   // elements per block: one float4 per thread and array, ~830 blocks for PpoCnn so that every
                                  // load of the step is in flight at once (a 4096-element block left 1.4 blocks per SM: latency bound)
constexpr int OPT_THREADS = 256;

struct AdamState {          // lives in device memory
  float beta1_pow, beta2_pow, lr_t, grad_norm;
  unsigned int iterations;  // steps taken (Keras `iterations`, read by the `decay` schedule)
};
struct AdamHyper {          // lives in device memory too: a captured CUDA graph must see xtb_adam_set_lr / _set_decay
  float lr, beta1, beta2, eps, clip;
  float decay;              // Keras OptimizerV2 `decay`: lr / (1 + decay * iterations); 0 = constant lr
};

__device__ __forceinline__ void adam_prep(AdamState* st, const AdamHyper* hyp, double* norm_sq, float* seg_scale, int n_seg,
                                          int clip_mode, float grad_scale) {
  const float clip = hyp->clip, beta1 = hyp->beta1, beta2 = hyp->beta2;
  float lr = hyp->lr;
  if (hyp->decay != 0.f) lr = lr / (1.f + hyp->decay * (float)st->iterations);   // iterations counted before the step
  st->iterations += 1;
  double tot = 0.0;
  for (int s = 0; s < n_seg; s++) tot += norm_sq[s];
  float gs = fabsf(grad_scale);
  float gnorm = (float)sqrt(tot) * gs;
  st->grad_norm = gnorm;
  if (clip_mode == 1) {
    float sc = clip / fmaxf(gnorm, clip);
    for (int s = 0; s < n_seg; s++) seg_scale[s] = sc * grad_scale;
  } else if (clip_mode == 2) {
    for (int s = 0; s < n_seg; s++) {
      float n = (float)sqrt(norm_sq[s]) * gs;
      seg_scale[s] = (n > clip ? clip / n : 1.f) * grad_scale;
    }
  } else {
    for (int s = 0; s < n_seg; s++) seg_scale[s] = grad_scale;
  }
  for (int s = 0; s < n_seg; s++) norm_sq[s] = 0.0;
  float b1p = st->beta1_pow * beta1, b2p = st->beta2_pow * beta2;
  st->beta1_pow = b1p; st->beta2_pow = b2p;
  st->lr_t = lr * sqrtf(1.f - b2p) / (1.f - b1p);
}

// `ticket`: zero-initialised counter; the block that draws the last ticket sees every block's contribution.
// One block sums SQN_GROUP consecutive chunks (the optimiser's chunks are small so that adam_kernel keeps every load in
// flight; here fewer, longer blocks keep the number of same-address fp64 atomics low).
constexpr int SQN_GROUP = 4;
__global__ void __launch_bounds__(OPT_THREADS)
sqnorm_kernel(const float* __restrict__ g, const int* __restrict__ blk_seg,
              const long long* __restrict__ blk_beg, const int* __restrict__ blk_len, int n_blk,
              double* __restrict__ norm_sq, unsigned int* __restrict__ ticket, AdamState* st, const AdamHyper* __restrict__ hyp,
              float* seg_scale, int n_seg, int clip_mode, float grad_scale) {
  pdl_wait(); pdl_trigger();
  __shared__ float red[OPT_THREADS / 32];
  auto flush = [&](float s, int seg) {          // block-wide sum of s into norm_sq[seg]; uniform call sites only
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
      float t = threadIdx.x < OPT_THREADS / 32 ? red[threadIdx.x] : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (threadIdx.x == 0) atomicAdd(norm_sq + seg, (double)t);
    }
    __syncthreads();
  };
  const int e0 = blockIdx.x * SQN_GROUP, e1 = min(e0 + SQN_GROUP, n_blk);
  float s = 0.f;
  int cur = blk_seg[e0];
  for (int e = e0; e < e1; e++) {
    if (blk_seg[e] != cur) { flush(s, cur); s = 0.f; cur = blk_seg[e]; }
    const float* p = g + blk_beg[e];
    const int n = blk_len[e];
    if ((blk_beg[e] & 3) == 0) {
      const int nv = n & ~3;
      for (int i = threadIdx.x * 4; i < nv; i += OPT_THREADS * 4) {
        const float4 v = *reinterpret_cast<const float4*>(p + i);
        s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
      }
      for (int i = nv + threadIdx.x; i < n; i += OPT_THREADS) { float v = p[i]; s = fmaf(v, v, s); }
    } else {
      for (int i = threadIdx.x; i < n; i += OPT_THREADS) { float v = p[i]; s = fmaf(v, v, s); }
    }
  }
  flush(s, cur);
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
      __threadfence();
      *ticket = 0;
      adam_prep(st, hyp, norm_sq, seg_scale, n_seg, clip_mode, grad_scale);
    }
  }
}

__global__ void __launch_bounds__(OPT_THREADS)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
            float* __restrict__ v, const int* __restrict__ blk_seg,
            const long long* __restrict__ blk_beg, const int* __restrict__ blk_len,
            const float* __restrict__ seg_scale, const AdamState* __restrict__ st, const AdamHyper* __restrict__ hyp,
            const bp::BlobSeg* __restrict__ bsegs, int n_bsegs, __nv_bfloat16* __restrict__ w_hi, long long w_lo_off) {
  pdl_wait(); pdl_trigger();
  const float beta1 = hyp->beta1, beta2 = hyp->beta2, eps = hyp->eps;
  long long beg = blk_beg[blockIdx.x];
  int n = blk_len[blockIdx.x];
  float sc = seg_scale[blk_seg[blockIdx.x]];
  float lr_t = st->lr_t;
  const bool vec = ((beg & 3) == 0);      // 16-byte aligned chunk: 4 parameters per thread per iteration
  int nv = vec ? (n & ~3) : 0;
  for (int i = threadIdx.x * 4; i < nv; i += OPT_THREADS * 4) {
    long long j = beg + i;
    float4 g4 = *reinterpret_cast<const float4*>(g + j);
    float4 m4 = *reinterpret_cast<const float4*>(m + j);
    float4 v4 = *reinterpret_cast<const float4*>(v + j);
    float4 p4 = *reinterpret_cast<const float4*>(p + j);
    float gg[4] = {g4.x * sc, g4.y * sc, g4.z * sc, g4.w * sc};
    float mm[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w}, pp[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
    for (int q = 0; q < 4; q++) {
      mm[q] = beta1 * mm[q] + (1.f - beta1) * gg[q];
      vv[q] = beta2 * vv[q] + (1.f - beta2) * gg[q] * gg[q];
      pp[q] -= lr_t * mm[q] / (sqrtf(vv[q]) + eps);
    }
    *reinterpret_cast<float4*>(m + j) = make_float4(mm[0], mm[1], mm[2], mm[3]);
    *reinterpret_cast<float4*>(v + j) = make_float4(vv[0], vv[1], vv[2], vv[3]);
    *reinterpret_cast<float4*>(p + j) = make_float4(pp[0], pp[1], pp[2], pp[3]);
    if (w_hi) bp::blob_store4(bsegs, n_bsegs, w_hi, w_lo_off, j, pp);   // weight blobs of the tensor-core layers
  }
  for (int i = nv + threadIdx.x; i < n; i += OPT_THREADS) {
    long long j = beg + i;
    float gg = g[j] * sc;
    float mm = beta1 * m[j] + (1.f - beta1) * gg;
    float vv = beta2 * v[j] + (1.f - beta2) * gg * gg;
    m[j] = mm; v[j] = vv;
    float pn = p[j] - lr_t * mm / (sqrtf(vv) + eps);
    p[j] = pn;
    if (w_hi) bp::blob_store1(bsegs, n_bsegs, w_hi, w_lo_off, j, pn);
  }
}

// tf.train.RMSPropOptimizer(lr, decay, epsilon, centered=True), momentum 0 (xt/model/impala/impala_cnn_opt.py:205-206):
//   mg = rho mg + (1 - rho) g;  ms = rho ms + (1 - rho) g^2;  theta -= lr g / sqrt(ms - mg^2 + eps)
// (TF initialises ms to ONES, mg to zeros).  Same chunking, clip scales and weight-blob refresh as adam_kernel.
__global__ void __launch_bounds__(OPT_THREADS)
rmsprop_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ ms, float* __restrict__ mg,
               const int* __restrict__ blk_seg, const long long* __restrict__ blk_beg, const int* __restrict__ blk_len,
               const float* __restrict__ seg_scale, const AdamHyper* __restrict__ hyp, float rho, float rms_eps,
               const bp::BlobSeg* __restrict__ bsegs, int n_bsegs, __nv_bfloat16* __restrict__ w_hi, long long w_lo_off) {
  pdl_wait(); pdl_trigger();
  const long long beg = blk_beg[blockIdx.x];
  const int n = blk_len[blockIdx.x];
  const float sc = seg_scale[blk_seg[blockIdx.x]], lr = hyp->lr;
  const bool vec = ((beg & 3) == 0);
  const int nv = vec ? (n & ~3) : 0;
  for (int i = threadIdx.x * 4; i < nv; i += OPT_THREADS * 4) {
    const long long j = beg + i;
    const float4 g4 = *reinterpret_cast<const float4*>(g + j);
    const float4 s4 = *reinterpret_cast<const float4*>(ms + j);
    const float4 a4 = *reinterpret_cast<const float4*>(mg + j);
    const float4 p4 = *reinterpret_cast<const float4*>(p + j);
    float gg[4] = {g4.x * sc, g4.y * sc, g4.z * sc, g4.w * sc};
    float ss[4] = {s4.x, s4.y, s4.z, s4.w}, aa[4] = {a4.x, a4.y, a4.z, a4.w}, pp[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
    for (int q = 0; q < 4; q++) {
      aa[q] = rho * aa[q] + (1.f - rho) * gg[q];
      ss[q] = rho * ss[q] + (1.f - rho) * gg[q] * gg[q];
      pp[q] -= lr * gg[q] / sqrtf(ss[q] - aa[q] * aa[q] + rms_eps);
    }
    *reinterpret_cast<float4*>(ms + j) = make_float4(ss[0], ss[1], ss[2], ss[3]);
    *reinterpret_cast<float4*>(mg + j) = make_float4(aa[0], aa[1], aa[2], aa[3]);
    *reinterpret_cast<float4*>(p + j) = make_float4(pp[0], pp[1], pp[2], pp[3]);
    if (w_hi) bp::blob_store4(bsegs, n_bsegs, w_hi, w_lo_off, j, pp);
  }
  for (int i = nv + threadIdx.x; i < n; i += OPT_THREADS) {
    const long long j = beg + i;
    const float gg = g[j] * sc;
    const float aa = rho * mg[j] + (1.f - rho) * gg;
    const float ss = rho * ms[j] + (1.f - rho) * gg * gg;
    mg[j] = aa; ms[j] = ss;
    const float pn = p[j] - lr * gg / sqrtf(ss - aa * aa + rms_eps);
    p[j] = pn;
    if (w_hi) bp::blob_store1(bsegs, n_bsegs, w_hi, w_lo_off, j, pn);
  }
}

}  // namespace xtb
