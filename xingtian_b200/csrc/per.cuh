// per.cuh -- prioritized experience replay (Schaul et al., proportional variant) over the slots of a device replay ring:
// the sum / min trees, their insert and update, and the stratified draw with importance weights (xtb_per_* in xtb200.h,
// the rules of xt/algorithm/prioritized_replay_buffer_muzero.py applied to ring slots).
//
// Both trees are float64 in heap order over `leaves` = capacity rounded up to a power of two: node 1 is the root, node
// i has the children 2i and 2i + 1, and leaf j (ring slot j) is node leaves + j.  An empty leaf is 0 in the sum tree and
// +inf in the min tree.  Every internal node is written only as op(left, right) of its final children, level by level
// from the leaves up, so the trees are bitwise a function of their leaves whatever order inserts and updates came in.
// The kernels run as one CTA: a batch is at most a few thousand scattered leaves, and __syncthreads() orders the levels.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/xtb200.h"
#include "launch.cuh"

namespace xtb {

// Device-resident state: every value that changes from step to step lives here, so one captured graph serves every step.
struct PerState {
  double max_priority;          // largest raw priority (|delta| + eps) an update wrote; starts at 1, never lowered
  unsigned long long offset;    // Philox offset of the next device draw
  int32_t count;                // stored slots: leaves [0, count) hold priorities
  int32_t status;               // XTB_PER_* bits (xtb200.h); sticky
};

struct PerTree {
  double* sum;        // [2 leaves] heap order (node 0 unused)
  double* mn;         // [2 leaves]
  int32_t* last;      // [leaves] update scratch: the last batch position that writes each leaf; -1 between calls
  PerState* st;
  int leaves, depth;  // leaves = 2^depth
};

constexpr int kPerThreads = 1024;
constexpr int kPerTop = 2048;   // nodes [1, kPerTop) of the sum tree are staged in shared memory for the descent

// p ** alpha, exact for alpha 1 (CUDA's pow may miss x ** 1 by an ulp) and alpha 0
__device__ __forceinline__ double per_pow(double p, double alpha) { return alpha == 1.0 ? p : pow(p, alpha); }

__device__ __forceinline__ void per_pull(const PerTree& t, int node) {
  t.sum[node] = t.sum[2 * node] + t.sum[2 * node + 1];
  t.mn[node] = fmin(t.mn[2 * node], t.mn[2 * node + 1]);
}

// Slots [first, first + n) were (over)written: each gets max_priority ** alpha; count grows to cover them.
__global__ void __launch_bounds__(kPerThreads) per_insert_kernel(PerTree t, int first, int n, double alpha) {
  pdl_wait(); pdl_trigger();
  const double p = per_pow(t.st->max_priority, alpha);
  for (int i = threadIdx.x; i < n; i += blockDim.x) { t.sum[t.leaves + first + i] = p; t.mn[t.leaves + first + i] = p; }
  __syncthreads();
  if (threadIdx.x == 0 && first + n > t.st->count) t.st->count = first + n;
  int lo = t.leaves + first, hi = t.leaves + first + n - 1;
  for (int l = 0; l < t.depth; l++) {
    lo >>= 1; hi >>= 1;
    for (int node = lo + threadIdx.x; node <= hi; node += blockDim.x) per_pull(t, node);
    __syncthreads();
  }
}

// The reference's sequential update loop over k, with entries whose priority is not finite skipped (they set
// XTB_PER_NONFINITE) and indices outside [0, count) skipped (XTB_PER_BAD_INDEX): leaf idx[k] = (td_abs[k] + eps) ** alpha
// from the last k naming it, and max_priority = max(max_priority, td_abs[k] + eps) over every k.
__device__ __forceinline__ bool per_priority(const float* td_abs, int k, double alpha, double eps, double& d, double& p) {
  d = (double)td_abs[k] + eps;
  p = per_pow(d, alpha);
  return isfinite(d) && isfinite(p);
}
__global__ void __launch_bounds__(kPerThreads) per_update_kernel(PerTree t, const int32_t* __restrict__ idx,
                                                                 const float* __restrict__ td_abs, int n, double alpha, double eps) {
  pdl_wait(); pdl_trigger();
  __shared__ double s_max[kPerThreads / 32];
  __shared__ int s_status;
  if (threadIdx.x == 0) s_status = 0;
  const int count = t.st->count;
  double d, p;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int j = idx[k];
    if (j >= 0 && j < count && per_priority(td_abs, k, alpha, eps, d, p)) atomicMax(&t.last[j], k);
  }
  __syncthreads();
  double mx = 0.0;
  int bad = 0;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int j = idx[k];
    if (j < 0 || j >= count) { bad |= XTB_PER_BAD_INDEX; continue; }
    if (!per_priority(td_abs, k, alpha, eps, d, p)) { bad |= XTB_PER_NONFINITE; continue; }
    mx = fmax(mx, d);
    if (t.last[j] == k) { t.sum[t.leaves + j] = p; t.mn[t.leaves + j] = p; }
  }
  for (int o = 16; o; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
  if (bad) atomicOr(&s_status, bad);
  __syncthreads();
  for (int k = threadIdx.x; k < n; k += blockDim.x) {     // every reader of `last` has passed the barrier
    const int j = idx[k];
    if (j >= 0 && j < count) t.last[j] = -1;
  }
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) mx = fmax(mx, s_max[w]);
    if (mx > t.st->max_priority) t.st->max_priority = mx;
    if (s_status) t.st->status |= s_status;
  }
  for (int l = 1; l <= t.depth; l++) {
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
      const int j = idx[k];
      if (j >= 0 && j < count) per_pull(t, (t.leaves + j) >> l);   // a shared parent is written with the same value
    }
    __syncthreads();
  }
}

// B stratified draws: mass_k = (u_k + k) total / B, descend to the first leaf whose running sum exceeds mass_k, clamp to
// count - 1; w_k = ((leaf / total) count) ** -beta / (p_min count) ** -beta with p_min = max(min / total, 1e-5), all in
// float64.  u_k = u_in[k] when set, else 53 bits of Philox4x32-10 on counter (k, 0, offset) and key seed, in [0, 1); the
// device offset then advances by one.  An empty tree writes idx 0, w 0 and sets XTB_PER_EMPTY.
__global__ void __launch_bounds__(kPerThreads) per_sample_kernel(PerTree t, int B, double beta, const double* __restrict__ u_in,
                                                                 uint64_t seed, int32_t* __restrict__ idx, float* __restrict__ w) {
  pdl_wait(); pdl_trigger();
  __shared__ double s_top[kPerTop];
  const int count = t.st->count;
  const unsigned long long off = t.st->offset;
  const double total = t.sum[1], p_min = fmax(t.mn[1] / total, 1e-5);
  const int ntop = min(2 * t.leaves, kPerTop);
  for (int i = threadIdx.x; i < ntop; i += blockDim.x) s_top[i] = t.sum[i];
  __syncthreads();
  const bool empty = !(count > 0 && total > 0.0);
  if (threadIdx.x == 0) {
    if (!u_in) t.st->offset = off + 1;
    if (empty) t.st->status |= XTB_PER_EMPTY;
  }
  const double max_w = pow(p_min * count, -beta);
  for (int k = threadIdx.x; k < B; k += blockDim.x) {
    if (empty) { idx[k] = 0; w[k] = 0.f; continue; }
    double u;
    if (u_in) {
      u = u_in[k];
    } else {
      uint32_t c[4] = {(uint32_t)k, 0u, (uint32_t)(off & 0xffffffffu), (uint32_t)(off >> 32)};
      philox4x32_10(c, (uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32));
      u = ((double)(c[0] >> 5) * 67108864.0 + (double)(c[1] >> 6)) * (1.0 / 9007199254740992.0);
    }
    double mass = (u + k) * total / B;
    int node = 1;
    while (node < t.leaves) {
      const double left = 2 * node < kPerTop ? s_top[2 * node] : t.sum[2 * node];
      if (left > mass) node = 2 * node;
      else { mass -= left; node = 2 * node + 1; }
    }
    const int j = min(node - t.leaves, count - 1);
    idx[k] = j;
    w[k] = (float)(pow(t.sum[t.leaves + j] / total * count, -beta) / max_w);
  }
}

}  // namespace xtb
