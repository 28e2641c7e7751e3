// muzero_replay.cuh -- MuZero's trajectory replay in HBM (xtb_muzero_replay_* in xtb200.h): the two-level prioritized
// draw of the Muzero learner (xt/algorithm/muzero/muzero.py over prioritized_replay_buffer_muzero.py), the gather of
// the drawn minibatch and the priority updates, with the host learner's rules and float64 arithmetic.
//
// Level 1 is a float64 sum tree over the trajectory ring (leaf s = slot s, heap order, node 1 the root).  Level 2 is one
// float64 sum tree per stored trajectory over its positions: a trajectory of L steps at pool offset `off` keeps its
// tree of 2 cap nodes (cap = L rounded up to a power of two) at forest + 4 off, inside the forest range its own pool
// range owns (2 cap < 4 L), so trees need no planning of their own and may be far larger than shared memory.  As in
// per.cuh, every internal node is written only as left + right of its final children.
//
// The host's segment-tree queries are restated exactly:
//   reduce(0, n - 1) (exclusive end, split at node midpoints) = mzr_prefix(tree, leaves, n - 2): the recursion adds the
//     whole left children on the way down to the highest node whose range ends at leaf n - 2, innermost sum first;
//   find_prefixsum_idx(mass) = mzr_descend: the first leaf whose running sum exceeds mass, with the host's subtractions.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/xtb200.h"
#include "launch.cuh"

namespace xtb {

struct MzrState {
  int32_t count;    // stored slots (the host ring's len(storage)); evicted slots keep their place
  int32_t status;   // XTB_MZR_* bits: set by the last draw, or-ed by the updates after it
};

// The device side of an xtb_muzero_replay: the pool, the slot table and both tree levels
struct MzrDev {
  uint8_t* obs;                      // [pool, row_bytes] observations as the representation net reads them
  int32_t* action;                   // [pool]
  double* tv;                        // [pool] target values (the priorities need float64)
  float* reward;                     // [pool]
  float* child;                      // [pool, A] child visits
  double* traj;                      // [2 tleaves] level-1 sum tree
  double* forest;                    // [4 pool] level-2 trees
  xtb_muzero_replay_slot* slot;      // [capacity]
  MzrState* st;
  double* wt;                        // [max_batch] update scratch: the trajectory weight after batch entry i
  long long row_bytes;
  int tleaves, K, A;
};

constexpr int kMzrThreads = 1024;

__device__ __forceinline__ int mzr_cap(int len) { int c = 1; while (c < len) c *= 2; return c; }
__device__ __forceinline__ double* mzr_tree(const MzrDev& d, const xtb_muzero_replay_slot& s) { return d.forest + 4 * s.off; }

// SegmentTree.reduce(0, hi + 1) of the host: the leaves 0 .. hi summed in the order of its midpoint recursion; 0 when
// hi < 0 (the host's recursion does not terminate there)
__device__ __forceinline__ double mzr_prefix(const double* t, int leaves, int hi) {
  if (hi < 0) return 0.0;
  int n = leaves + hi;
  while ((n & 1) && n > 1) n >>= 1;   // the highest node whose range ends at leaf hi
  double acc = t[n];
  for (; n > 1; n >>= 1)
    if (n & 1) acc = t[n - 1] + acc;  // a right child: its left sibling is whole inside the range
  return acc;
}

__device__ __forceinline__ int mzr_descend(const double* t, int leaves, double mass) {
  int i = 1;
  while (i < leaves) {
    const double l = t[2 * i];
    if (l > mass) i = 2 * i;
    else { mass -= l; i = 2 * i + 1; }
  }
  return i - leaves;
}

// The host's mass `u * step + k * step`: both products rounded before the sum, as Python evaluates it (a plain
// expression would let nvcc contract one product and the add into an FMA, which skips a rounding)
__device__ __forceinline__ double mzr_mass(double u, double step, int k) {
  return __dadd_rn(__dmul_rn(u, step), __dmul_rn((double)k, step));
}

// leaf i of a tree was written: its ancestors, innermost first
__device__ __forceinline__ void mzr_pull_path(double* t, int leaves, int leaf) {
  for (int n = (leaves + leaf) >> 1; n >= 1; n >>= 1) t[n] = t[2 * n] + t[2 * n + 1];
}

// Add: slot `s` now holds the trajectory at pool [off, off + len) (its steps already copied there); slots
// [e0, e0 + ne) mod capacity were evicted.  Builds the position tree (leaf i < len - K: |value_i - tv_i| in float64, the
// rest 0), writes the trajectory's weight root / (len - K) at leaf s and 0 at the evicted leaves, and pulls the touched
// paths of the trajectory tree level by level.  value: vf (the model's float32 values, widened) or vd.
__global__ void __launch_bounds__(kMzrThreads) mzr_add_kernel(MzrDev d, int s, long long off, int len, int e0, int ne, int capacity,
                                                             const float* __restrict__ vf, const double* __restrict__ vd) {
  pdl_wait(); pdl_trigger();
  const int cap = mzr_cap(len), n_pos = len - d.K;
  double* t = d.forest + 4 * off;
  for (int i = threadIdx.x; i < cap; i += blockDim.x) {
    double p = 0.0;
    if (i < n_pos) p = fabs((vf ? (double)vf[i] : vd[i]) - d.tv[off + i]);
    t[cap + i] = p;
  }
  __syncthreads();
  for (int lo = cap >> 1; lo >= 1; lo >>= 1) {
    for (int n = lo + threadIdx.x; n < 2 * lo; n += blockDim.x) t[n] = t[2 * n] + t[2 * n + 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    d.slot[s] = xtb_muzero_replay_slot{off, len, 1};
    d.traj[d.tleaves + s] = t[1] / (double)n_pos;
    if (s + 1 > d.st->count) d.st->count = s + 1;
  }
  for (int k = threadIdx.x; k < ne; k += blockDim.x) {
    const int j = (e0 + k) % capacity;
    d.slot[j].live = 0;
    d.traj[d.tleaves + j] = 0.0;
  }
  __syncthreads();
  for (int l = 1; (d.tleaves >> l) >= 1; l++) {
    for (int k = threadIdx.x; k <= ne; k += blockDim.x) {
      const int j = k < ne ? (e0 + k) % capacity : s;
      const int n = (d.tleaves + j) >> l;
      d.traj[n] = d.traj[2 * n] + d.traj[2 * n + 1];   // a shared parent is written with the same value
    }
    __syncthreads();
  }
}

// The draw of Muzero.train: trajectory k takes mass u[k] step + k step (step = reduce(0, count - 1) / B) in the
// trajectory tree; a descent that ends on a slot without a live trajectory (evicted, or past count through rounding)
// takes the nearest live slot below it, wrapping from slot 0 to count - 1, and sets XTB_MZR_REMAPPED.  Its position takes
// mass u[B + k] total + 0 total (total = reduce(0, n_pos - 1) of its tree), clamped to n_pos - 1.
__global__ void __launch_bounds__(kMzrThreads) mzr_draw_kernel(MzrDev d, int B, const double* __restrict__ u, int32_t* __restrict__ slot_out,
                                                              int32_t* __restrict__ pos_out) {
  pdl_wait(); pdl_trigger();
  __shared__ int s_remap;
  if (threadIdx.x == 0) s_remap = 0;
  __syncthreads();
  const int count = d.st->count;
  const double step = mzr_prefix(d.traj, d.tleaves, count - 2) / B;
  for (int k = threadIdx.x; k < B; k += blockDim.x) {
    int j = mzr_descend(d.traj, d.tleaves, mzr_mass(u[k], step, k));
    if (j >= count || !d.slot[j].live) {
      int r = -1;
      for (int q = 1; q <= count && r < 0; q++) {
        const int c = ((j < count ? j : count) - q + 2 * count) % count;
        if (d.slot[c].live) r = c;
      }
      j = r < 0 ? 0 : r;
      s_remap = 1;
    }
    const xtb_muzero_replay_slot sl = d.slot[j];
    const int n_pos = sl.len - d.K, cap = mzr_cap(sl.len);
    const double* t = mzr_tree(d, sl);
    const double tot = mzr_prefix(t, cap, n_pos - 2);
    const int p = mzr_descend(t, cap, mzr_mass(u[B + k], tot, 0));
    slot_out[k] = j;
    pos_out[k] = min(p, n_pos - 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) d.st->status = s_remap ? XTB_MZR_REMAPPED : 0;
}

// The minibatch of the drawn (slot, position) pairs: observation row pos, actions pos .. pos + K - 1 and the targets
// pos .. pos + K (the value target rounded to float32, as the host's upload does).  One CTA per sample.
__global__ void __launch_bounds__(256) mzr_gather_kernel(MzrDev d, const int32_t* __restrict__ slot, const int32_t* __restrict__ pos,
                                                         uint8_t* __restrict__ obs, int32_t* __restrict__ action, float* __restrict__ tv,
                                                         float* __restrict__ tr, float* __restrict__ tp) {
  pdl_wait(); pdl_trigger();
  const int k = blockIdx.x, K = d.K, A = d.A;
  const long long r0 = d.slot[slot[k]].off + pos[k];
  const uint8_t* src = d.obs + r0 * d.row_bytes;
  uint8_t* dst = obs + (long long)k * d.row_bytes;
  if (d.row_bytes % 16 == 0 && ((uintptr_t)src | (uintptr_t)dst) % 16 == 0) {
    for (long long i = threadIdx.x; i < d.row_bytes / 16; i += blockDim.x)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  } else {
    for (long long i = threadIdx.x; i < d.row_bytes; i += blockDim.x) dst[i] = src[i];
  }
  for (int i = threadIdx.x; i < K; i += blockDim.x) action[(long long)k * K + i] = d.action[r0 + i];
  for (int i = threadIdx.x; i <= K; i += blockDim.x) {
    tv[(long long)k * (K + 1) + i] = (float)d.tv[r0 + i];
    tr[(long long)k * (K + 1) + i] = d.reward[r0 + i];
  }
  for (int i = threadIdx.x; i < (K + 1) * A; i += blockDim.x) tp[(long long)k * (K + 1) * A + i] = d.child[r0 * A + i];
}

// The priority updates of Muzero.train, in batch order i: new_pri_i = max(|value_i - tv[pos_i]|, 1e-5) (NaN stays
// NaN) goes to position leaf pos_i of trajectory slot_i, then trajectory leaf i (the batch position) takes slot_i's
// weight at that moment, unless slot i holds no live trajectory.  The sequence stops before the first entry whose
// priority is not > 0 (XTB_MZR_BAD_PRIORITY), as the host's ValueError does.  The first entry of each drawn slot
// applies all of that slot's entries in order (their weights go to d.wt); then the batch-position leaves are written
// (they are distinct) and the trajectory tree pulled level by level.
__global__ void __launch_bounds__(kMzrThreads) mzr_update_kernel(MzrDev d, int B, const int32_t* __restrict__ slot,
                                                                const int32_t* __restrict__ pos, const float* __restrict__ vf,
                                                                const double* __restrict__ vd) {
  pdl_wait(); pdl_trigger();
  __shared__ int s_stop;
  if (threadIdx.x == 0) s_stop = B;
  __syncthreads();
  __shared__ int s_bad;
  if (threadIdx.x == 0) s_bad = 0;
  auto pri = [&](int i) {
    const xtb_muzero_replay_slot& sl = d.slot[slot[i]];
    const double v = vf ? (double)vf[i] : vd[i];
    const double a = fabs(v - d.tv[sl.off + pos[i]]);
    return a != a ? a : fmax(a, 1e-5);
  };
  const int count = d.st->count;
  __syncthreads();
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const int s = slot[i];
    // an entry that names no live trajectory or a position outside it, or whose batch position i is not a stored slot
    // (the host's update_priorities raises there), stops the sequence as a bad priority does
    const bool ok = i < count && s >= 0 && s < count && d.slot[s].live && pos[i] >= 0 && pos[i] < d.slot[s].len - d.K;
    if (!ok) atomicOr(&s_bad, XTB_MZR_BAD_INDEX);
    else if (!(pri(i) > 0.0)) atomicOr(&s_bad, XTB_MZR_BAD_PRIORITY);
    if (!ok || !(pri(i) > 0.0)) atomicMin(&s_stop, i);
  }
  __syncthreads();
  const int stop = s_stop;
  for (int i = threadIdx.x; i < stop; i += blockDim.x) {
    const int s = slot[i];
    bool first = true;
    for (int j = 0; j < i && first; j++) first = slot[j] != s;
    if (!first) continue;
    const xtb_muzero_replay_slot sl = d.slot[s];
    const int cap = mzr_cap(sl.len);
    const double n_pos = (double)(sl.len - d.K);
    double* t = mzr_tree(d, sl);
    for (int j = i; j < stop; j++) {
      if (slot[j] != s) continue;
      t[cap + pos[j]] = pri(j);
      mzr_pull_path(t, cap, pos[j]);
      d.wt[j] = t[1] / n_pos;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < stop; i += blockDim.x)
    if (d.slot[i].live) d.traj[d.tleaves + i] = d.wt[i];
  __syncthreads();
  for (int l = 1; (d.tleaves >> l) >= 1; l++) {
    for (int i = threadIdx.x; i < stop; i += blockDim.x)
      if (d.slot[i].live) { const int n = (d.tleaves + i) >> l; d.traj[n] = d.traj[2 * n] + d.traj[2 * n + 1]; }
    __syncthreads();
  }
  if (threadIdx.x == 0 && s_bad) d.st->status |= s_bad;
}

}  // namespace xtb
