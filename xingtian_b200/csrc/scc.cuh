// scc.cuh -- SCC kernels (xt/model/scc/scc_tf.py): the critic inputs, the fused critic-head / TD / credit / actor-loss
// step, and the head's weight gradients.  The agent network is QMIX's (qmix.cuh); the critic's hidden layers run on the
// layer engine.
//
// Critic layout.  A critic state row r = b L + t holds n_agents slices of D = o + A floats (raw observation, one-hot
// action).  With the multi-channel critic, agent a of group j is channel a: group j's net reads its agents' slices as rows
// r n_j + (a - a0_j) of a group-major buffer (group j starting at row B L a0_j), and
//   V = b_v + sum_a u_a,  u_a = h_a . w_a   (concat: w_a = kernel rows a U .. a U + U - 1; add: w_a = the whole kernel).
// The single-channel critic is one channel over the whole n D row (h_0 . w + b_v).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "launch.cuh"
#include "qmix.cuh"

namespace xtb {

constexpr int SCC_MAX_GROUPS = 8;
constexpr int SCC_MAX_UNITS = 512;    // critic width U (dense_unit_number) the kernels take
constexpr int SCC_THREADS = 256;      // fused step: one warp per critic row, 8 rows per block
constexpr int SCC_HG_ROWS = 64;       // head-gradient kernel: rows per partial sum

// The hidden outputs [rows, U] of one critic evaluation, by channel.
struct SccH {
  const float* h[SCC_MAX_GROUPS];     // group j's rows (multi-channel) / the rows (single-channel: one group of one channel)
  int a0[SCC_MAX_GROUPS + 1];         // first channel of each group; a0[ng] = channel count
  int ng;
};

// channel c of row r
__device__ __forceinline__ const float* scc_row(const SccH& H, int r, int c, int U) {
  int j = 0;
  while (j + 1 < H.ng && c >= H.a0[j + 1]) j++;
  const int nj = H.a0[j + 1] - H.a0[j];
  return H.h[j] + ((long long)r * nj + (c - H.a0[j])) * U;
}

// u_c = h_c(r) . w_c summed over the warp (every lane gets it)
__device__ __forceinline__ float scc_dot(const float* h, const float* w, int U, int lane) {
  float s = 0.f;
  for (int k = lane; k < U; k += 32) s = fmaf(h[k], w[k], s);
  return qwarp_sum(s);
}

// Critic inputs of the step.  s[b, t] = concat_a [raw[b, t, a, :o], one_hot(act[b, t, a], A)] for t < L, and every
// evaluation reads s'[b, t] = s[b, min(t + 1, L - 1)] (scc_tf.py:544-546 shifts through an alias of s).  Writes
//   xs: the full rows (multi-channel: group-major channel rows [B L n, D]; single: [B L, n D]);
//   xm: the rows of the credit evaluations.  Multi-channel: channel rows laid out as xs with the channel's own slice
//       zeroed (n <= 2) or its action part zeroed (n > 2).  Single-channel, V variants of [B L, n D]: n <= 2, variant i
//       has agent i's slice zeroed; n > 2, variants 2 (i mc + j) and 2 (i mc + j) + 1 have the action parts of the
//       agents in subsets[i mc + j] zeroed, the second also agent i's.
__global__ void __launch_bounds__(256)
scc_inputs_kernel(const float* __restrict__ raw, const int32_t* __restrict__ act, const uint32_t* __restrict__ subsets,
                  float* __restrict__ xs, float* __restrict__ xm, int B, int L, int n, int o, int A, int multi, int mc,
                  SccH groups) {
  pdl_wait(); pdl_trigger();
  const int D = o + A, T = L + 1;
  const long long total = (long long)B * L * n * D;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % D);
    const long long ra = e / D;
    const int a = (int)(ra % n);
    const int r = (int)(ra / n);
    const int b = r / L, t = min(r % L + 1, L - 1);
    const float v = c < o ? raw[(((long long)b * T + t) * n + a) * o + c] : (act[((long long)b * L + t) * n + a] == c - o ? 1.f : 0.f);
    const bool is_act = c >= o;
    if (multi) {
      int j = 0;
      while (j + 1 < groups.ng && a >= groups.a0[j + 1]) j++;
      const int nj = groups.a0[j + 1] - groups.a0[j];
      const long long row = (long long)B * L * groups.a0[j] + (long long)r * nj + (a - groups.a0[j]);
      xs[row * D + c] = v;
      xm[row * D + c] = (n <= 2 || is_act) ? 0.f : v;
    } else {
      const long long off = (long long)r * n * D + (long long)a * D + c;
      xs[off] = v;
      const long long vs = (long long)B * L * n * D;
      if (n <= 2) {
        for (int i = 0; i < n; i++) xm[i * vs + off] = i == a ? 0.f : v;
      } else {
        for (int i = 0; i < n; i++)
          for (int j = 0; j < mc; j++) {
            const bool in_s = (subsets[i * mc + j] >> a) & 1u;
            const long long v0 = 2LL * (i * mc + j);
            xm[v0 * vs + off] = is_act && in_s ? 0.f : v;
            xm[(v0 + 1) * vs + off] = is_act && (in_s || a == i) ? 0.f : v;
          }
      }
    }
  }
}

// Critic states [rows, n D] given by the caller -> the group-major channel rows of the multi-channel critic (no shift).
__global__ void __launch_bounds__(256)
scc_split_kernel(const float* __restrict__ s, float* __restrict__ xs, int rows, int n, int D, SccH groups) {
  pdl_wait(); pdl_trigger();
  const long long total = (long long)rows * n * D;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % D);
    const int a = (int)((e / D) % n);
    const int r = (int)(e / ((long long)n * D));
    int j = 0;
    while (j + 1 < groups.ng && a >= groups.a0[j + 1]) j++;
    const int nj = groups.a0[j + 1] - groups.a0[j];
    xs[((long long)rows * groups.a0[j] + (long long)r * nj + (a - groups.a0[j])) * D + c] = s[e];
  }
}

// V of every row: b_v + sum_c h_c . w_c (one warp per row)
__global__ void __launch_bounds__(SCC_THREADS)
scc_value_kernel(SccH eh, const float* __restrict__ head, int rows, int U, int concat, float* __restrict__ v_out) {
  pdl_wait(); pdl_trigger();
  const int lane = threadIdx.x & 31, r = blockIdx.x * (SCC_THREADS / 32) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int C = eh.a0[eh.ng], K = concat ? C * U : U;
  float v = 0.f;
  for (int c = 0; c < C; c++) v += scc_dot(scc_row(eh, r, c, U), head + (concat ? c * U : 0), U, lane);
  if (lane == 0) v_out[r] = v + head[K];
}

struct SccStep {
  SccH eh, th, mh;       // eval / target evaluations of the full rows, eval evaluation of the credit rows (variant 0)
  long long mh_stride;   // single-channel: floats between credit variants
  SccH dz;               // d loss / d (second layer pre-activation), laid out as eh (written through)
};

// The learner step of SCCModel.train (scc_tf.py:398-417, 535-564, 657-707) for every critic row r = b L + t (one warp):
//   V = V_eval(s'), Vt = V_target(s'), td = V - (reward + gamma (1 - terminated) Vt), mixer loss = sum (mask td)^2 / sum mask;
//   credit_i: multi-channel u_i(s') - u_i(credit row of i) (exactly the reference's V difference, which only channel i's
//   term separates); single-channel V(s') - V(variant i) (n <= 2) or the mean over j of V(variant 2(i mc + j)) -
//   V(variant 2(i mc + j) + 1);
//   actor loss = sum (mask Q_i - mask credit_i)^2 / (n sum mask), Q_i = qe[b, t, i, act].
// Writes dv[r] = d mixer loss / d V, the second-layer pre-activation gradients dz (relu' from the output), d actor loss /
// d Q into dq (zeroed by the caller) and part[2 block + {0, 1}] the block's sums of both squares, warp by warp in order.
__global__ void __launch_bounds__(SCC_THREADS)
scc_step_kernel(SccStep p, const float* __restrict__ head, const float* __restrict__ thead, const float* __restrict__ qe,
                const int32_t* __restrict__ act, const float* __restrict__ reward, const float* __restrict__ term,
                const float* __restrict__ mask, const float* __restrict__ msum, int B, int L, int n, int A, int U, int concat,
                int multi, int mc, float gamma, float* __restrict__ dv, float* __restrict__ dq, float* __restrict__ part) {
  __shared__ float red[2][SCC_THREADS / 32];
  pdl_wait(); pdl_trigger();
  const int BL = B * L, T = L + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * (SCC_THREADS / 32) + warp;
  float sq_m = 0.f, sq_a = 0.f;
  if (r < BL) {
    const int C = multi ? n : 1, K = concat ? C * U : U;
    float v = 0.f, vt = 0.f;
    for (int c = 0; c < C; c++) {
      const int wo = concat ? c * U : 0;
      v += scc_dot(scc_row(p.eh, r, c, U), head + wo, U, lane);
      vt += scc_dot(scc_row(p.th, r, c, U), thead + wo, U, lane);
    }
    v += head[K];
    vt += thead[K];
    const float m = mask[r];
    const float mtd = (v - (reward[r] + gamma * (1.f - term[r]) * vt)) * m;
    sq_m = mtd * mtd;
    const float g = 2.f * mtd * m * msum[1];
    if (lane == 0) dv[r] = g;
    // d loss / d (second layer pre-activation) of every channel
    for (int c = 0; c < C; c++) {
      const float* h = scc_row(p.eh, r, c, U);
      float* dz = const_cast<float*>(scc_row(p.dz, r, c, U));
      const float* w = head + (concat ? c * U : 0);
      for (int k = lane; k < U; k += 32) dz[k] = h[k] > 0.f ? g * w[k] : 0.f;
    }
    // credits, then the actor loss and d loss / d Q
    const float inv_alive = 1.f / ((float)n * msum[0]);
    const long long cur = ((long long)(r / L) * T + r % L) * n;
    for (int i = 0; i < n; i++) {
      float credit;
      if (multi) {
        const float* w = head + (concat ? i * U : 0);
        credit = scc_dot(scc_row(p.eh, r, i, U), w, U, lane) - scc_dot(scc_row(p.mh, r, i, U), w, U, lane);
      } else if (n <= 2) {
        credit = v - (scc_dot(p.mh.h[0] + i * p.mh_stride + (long long)r * U, head, U, lane) + head[K]);
      } else {
        float s = 0.f;
        for (int j = 0; j < mc; j++) {
          const long long v0 = 2LL * (i * mc + j);
          const float with_i = scc_dot(p.mh.h[0] + v0 * p.mh_stride + (long long)r * U, head, U, lane) + head[K];
          const float without_i = scc_dot(p.mh.h[0] + (v0 + 1) * p.mh_stride + (long long)r * U, head, U, lane) + head[K];
          s += with_i - without_i;
        }
        credit = s / (float)mc;
      }
      const int ac = act[(long long)r * n + i];
      const float d = m * qe[(cur + i) * A + ac] - m * credit;
      sq_a += d * d;
      if (lane == 0) dq[(cur + i) * A + ac] = 2.f * d * m * inv_alive;
    }
  }
  if (lane == 0) { red[0][warp] = sq_m; red[1][warp] = sq_a; }
  __syncthreads();
  if (threadIdx.x < 2) {
    float s = 0.f;
    for (int w = 0; w < SCC_THREADS / 32; w++) s += red[threadIdx.x][w];
    part[2 * blockIdx.x + threadIdx.x] = s;
  }
}

// Partial sums of the head's gradients over SCC_HG_ROWS rows: element e < K of the kernel (concat: channel e / U, unit
// e % U; add: unit e of every channel; single: unit e), e = K the bias.  hpart[chunk][K + 1].
__global__ void __launch_bounds__(128)
scc_head_grad_kernel(SccH eh, const float* __restrict__ dv, int rows, int U, int concat, float* __restrict__ hpart) {
  pdl_wait(); pdl_trigger();
  const int C = eh.a0[eh.ng], K = concat ? C * U : U;
  const int e = blockIdx.y * blockDim.x + threadIdx.x;
  if (e > K) return;
  const int r0 = blockIdx.x * SCC_HG_ROWS, r1 = min(rows, r0 + SCC_HG_ROWS);
  float s = 0.f;
  for (int r = r0; r < r1; r++) {
    const float g = dv[r];
    if (e == K) { s += g; continue; }
    if (concat) {
      s = fmaf(g, scc_row(eh, r, e / U, U)[e % U], s);
    } else {
      float hs = 0.f;
      for (int c = 0; c < C; c++) hs += scc_row(eh, r, c, U)[e];
      s = fmaf(g, hs, s);
    }
  }
  hpart[(long long)blockIdx.x * (K + 1) + e] = s;
}

// grad[e] = sum of the chunks' partials in chunk order; thread K + 1 of the grid writes both losses:
// out[0] = mixer loss, out[1] = actor loss (their partial sums in block order).
__global__ void __launch_bounds__(128)
scc_reduce_kernel(const float* __restrict__ hpart, int n_chunk, int K, float* __restrict__ grad, const float* __restrict__ part,
                  int n_part, const float* __restrict__ msum, int n, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e <= K) {
    float s = 0.f;
    for (int c = 0; c < n_chunk; c++) s += hpart[(long long)c * (K + 1) + e];
    grad[e] = s;
  } else if (e == K + 1) {
    float sm = 0.f, sa = 0.f;
    for (int i = 0; i < n_part; i++) { sm += part[2 * i]; sa += part[2 * i + 1]; }
    out[0] = sm / msum[0];
    out[1] = sa / ((float)n * msum[0]);
  }
}

}  // namespace xtb
