// qmix.cuh -- QMIX kernels (xt/model/qmix/qmix_tf.py): the GRU recurrence of the agent network over whole episodes, its
// reverse-time backward, and the fused hypernetwork-mixer / TD-loss step.  The dense layers around them (fc1, fc2, the
// hypernetworks) run on the layer engine.
//
// Agent rows are stored [B][T][n_agents] (T = L + 1 steps per episode, the layout fc1 and fc2 run on); GRU sequence
// s = b * n_agents + a reads row (b * T + t) * n_agents + a at step t, which is the reference's transpose to (episode,
// agent) sequences and back without moving data.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "launch.cuh"

namespace xtb {

constexpr int QG_THREADS = 256;       // GRU kernels: one CTA per group of QG sequences
constexpr int QM_THREADS = 256;       // mixer kernel: one warp per (episode, step) row, 8 rows per block
constexpr int QM_MAX_AGENTS = 32;     // lane a keeps agent a's chosen / target Q
constexpr int QM_MAX_EMBED = 128;     // lane j keeps embed units j, j + 32, ...

// Shared memory of the GRU kernels (floats): the h rows of the gates kernel [H][2H + 1] and of the candidate kernel
// [H][H + 1] (rows padded by one float, so the backward's column reads are bank-conflict free), then 5 vectors of H per
// sequence of the group.
__host__ __device__ inline long long qgru_smem_floats(int H, int G) {
  return (long long)H * (2 * H + 1) + (long long)H * (H + 1) + 5LL * G * H;
}

__device__ inline float qsigmoid(float x) { return 1.f / (1.f + expf(-x)); }
// Keras hard_sigmoid (TF 1.15 backend): clip(0.2 x + 0.5, 0, 1), each operation rounded as TF rounds it
__device__ inline float qhard_sigmoid(float x) { return fminf(fmaxf(__fadd_rn(__fmul_rn(0.2f, x), 0.5f), 0.f), 1.f); }
__device__ inline float qhard_sigmoid_grad(float v) { return v > 0.f && v < 1.f ? 0.2f : 0.f; }

// Where a GRU's recurrent weights sit and which gate activation it uses.  The gate block is [H][2H] at wg (row stride
// ldg), the reset gate in columns [r_col, r_col + H) and the update gate in the other H; the candidate block is
// [H][H] at wc (row stride ldc).  The gate pre-activations xg / dag and the [r|u] activations share the gate block's
// column order.
//   TF GRUCell (QMIX, SCC): gates [r|u] (r_col 0) in rows H.. of gates/kernel [2H, 2H], candidate rows H.. of
//   candidate/kernel [2H, H], sigmoid.
//   Keras GRU v1: recurrent_kernel [H, 3H] = [z | r | h] read in place (ldg = ldc = 3H, r_col H), hard_sigmoid.
struct GruRec {
  const float* wg; const float* wc; int ldg, ldc, r_col, hard;
};

__device__ inline void qgru_load_weights(const GruRec& w, int H, float* wg, float* wc) {
  const int P2 = 2 * H + 1, P1 = H + 1;
  for (int e = threadIdx.x; e < H * 2 * H; e += blockDim.x) { int k = e / (2 * H), j = e % (2 * H); wg[k * P2 + j] = w.wg[(long long)k * w.ldg + j]; }
  for (int e = threadIdx.x; e < H * H; e += blockDim.x) { int k = e / H, j = e % H; wc[k * P1 + j] = w.wc[(long long)k * w.ldc + j]; }
}

// A GRU over whole sequences: TF 1.15's GRUCell inside tf.nn.dynamic_rnn, or Keras's GRU v1 (reset_after=False),
// whose recurrence is the same with another gate activation and weight layout (GruRec).  xg [rows, 2H] holds the input
// projections x W_g + b_g of every step in the gate block's column order, xc [rows, H] holds x W_c + b_c (one GEMM
// each).  Per step t < len(s):
//   [r|u] = act(xg + h W_g),  c = tanh(xc + (r * h) W_c),  h' = u h + (1 - u) c
// hout [rows, H] gets h' (zero for t >= len(s): dynamic_rnn's outputs past the sequence length); with `store`, xg is
// overwritten by [r|u], xc by c and rh [rows, H] gets r * h (the backward pass's activations).  h0 [S, H] is the
// initial state (NULL: zeros) and hT [S, H] (may alias h0, or NULL) the state after len(s) steps.
__global__ void __launch_bounds__(QG_THREADS)
qmix_gru_fwd_kernel(GruRec W, float* xg, float* xc, const float* h0, float* hT,
                    float* __restrict__ hout, float* __restrict__ rh, const int32_t* __restrict__ seq_len, int S, int T, int n, int H,
                    int G, int store) {
  extern __shared__ float sm[];
  float* wg = sm;
  float* wc = wg + H * (2 * H + 1);
  float* hs = wc + H * (H + 1);
  float* rs = hs + G * H;
  float* us = rs + G * H;
  __shared__ int lens[64];
  pdl_wait(); pdl_trigger();
  const int s0 = blockIdx.x * G, ng = min(G, S - s0);
  qgru_load_weights(W, H, wg, wc);
  const int r_col = W.r_col;
  int tmax = 0;
  for (int g = 0; g < ng; g++) tmax = max(tmax, min(max(seq_len[s0 + g], 0), T));
  if (threadIdx.x < ng) lens[threadIdx.x] = min(max(seq_len[s0 + threadIdx.x], 0), T);
  for (int e = threadIdx.x; e < ng * H; e += blockDim.x) hs[e] = h0 ? h0[(long long)(s0 + e / H) * H + e % H] : 0.f;
  __syncthreads();
  auto row_of = [&](int g, int t) { const int s = s0 + g; return ((long long)(s / n) * T + t) * n + s % n; };
  const int P2 = 2 * H + 1, P1 = H + 1;
  for (int t = 0; t < tmax; t++) {
    for (int o = threadIdx.x; o < ng * 2 * H; o += blockDim.x) {
      const int g = o / (2 * H), j = o % (2 * H);
      if (t >= lens[g]) continue;
      const long long row = row_of(g, t);
      const float* h = hs + g * H;
      float acc = xg[row * 2 * H + j];
      for (int k = 0; k < H; k++) acc = fmaf(h[k], wg[k * P2 + j], acc);
      const float v = W.hard ? qhard_sigmoid(acc) : qsigmoid(acc);
      if (store) xg[row * 2 * H + j] = v;
      const int jr = j - r_col;
      if (jr >= 0 && jr < H) rs[g * H + jr] = v * h[jr]; else us[g * H + j - (H - r_col)] = v;
    }
    __syncthreads();
    for (int o = threadIdx.x; o < ng * H; o += blockDim.x) {
      const int g = o / H, j = o % H;
      if (t >= lens[g]) continue;
      const long long row = row_of(g, t);
      const float* r = rs + g * H;
      float acc = xc[row * H + j];
      for (int k = 0; k < H; k++) acc = fmaf(r[k], wc[k * P1 + j], acc);
      const float c = tanhf(acc), u = us[g * H + j];
      const float hn = u * hs[g * H + j] + (1.f - u) * c;
      if (store) { xc[row * H + j] = c; rh[row * H + j] = r[j]; }
      hs[g * H + j] = hn;
      hout[row * H + j] = hn;
    }
    __syncthreads();
  }
  for (int g = 0; g < ng; g++)
    for (int e = threadIdx.x; e < (T - lens[g]) * H; e += blockDim.x) hout[row_of(g, lens[g] + e / H) * H + e % H] = 0.f;
  if (hT)
    for (int e = threadIdx.x; e < ng * H; e += blockDim.x) hT[(long long)(s0 + e / H) * H + e % H] = hs[e];
}

// Backward of qmix_gru_fwd_kernel (store = 1, h0 = zeros) in reverse time, carrying dh.  dy [rows, H] is d loss / d hout.
// Writes the gradients wrt the pre-activations of the gates, dag [rows, 2H] (the gate block's column order), and of the
// candidate, dac [rows, H] (zero rows for t >= len(s)); the weight gradients and d loss / d x follow as GEMMs over all
// rows.  The gate derivative is taken from the activation: v (1 - v) for sigmoid; 0.2 inside hard_sigmoid's clip and 0
// where it saturated (TF's clip_by_value gradient, except at a pre-activation within an fp32 rounding of +-2.5).
__global__ void __launch_bounds__(QG_THREADS)
qmix_gru_bwd_kernel(GruRec W, const float* __restrict__ ru, const float* __restrict__ cc,
                    const float* __restrict__ hout, const float* __restrict__ dy, float* __restrict__ dag, float* __restrict__ dac,
                    const int32_t* __restrict__ seq_len, int S, int T, int n, int H, int G) {
  extern __shared__ float sm[];
  float* wg = sm;
  float* wc = wg + H * (2 * H + 1);
  float* dh = wc + H * (H + 1);     // [G][H]  carried d loss / d h
  float* dn = dh + G * H;           // [G][H]  d loss / d h_prev, being summed
  float* ds = dn + G * H;           // [G][3H] [gate block (da_r, da_u) | da_c] of the current step
  __shared__ int lens[64];
  pdl_wait(); pdl_trigger();
  const int s0 = blockIdx.x * G, ng = min(G, S - s0);
  qgru_load_weights(W, H, wg, wc);
  const int r_col = W.r_col, u_col = H - r_col, hard = W.hard;
  int tmax = 0;
  for (int g = 0; g < ng; g++) tmax = max(tmax, min(max(seq_len[s0 + g], 0), T));
  if (threadIdx.x < ng) lens[threadIdx.x] = min(max(seq_len[s0 + threadIdx.x], 0), T);
  for (int e = threadIdx.x; e < ng * H; e += blockDim.x) dh[e] = 0.f;
  __syncthreads();
  auto row_of = [&](int g, int t) { const int s = s0 + g; return ((long long)(s / n) * T + t) * n + s % n; };
  for (int g = 0; g < ng; g++)
    for (int e = threadIdx.x; e < (T - lens[g]) * 3 * H; e += blockDim.x) {
      const long long row = row_of(g, lens[g] + e / (3 * H));
      const int j = e % (3 * H);
      if (j < 2 * H) dag[row * 2 * H + j] = 0.f; else dac[row * H + j - 2 * H] = 0.f;
    }
  const int P2 = 2 * H + 1, P1 = H + 1;
  for (int t = tmax - 1; t >= 0; t--) {
    for (int o = threadIdx.x; o < ng * H; o += blockDim.x) {
      const int g = o / H, j = o % H;
      if (t >= lens[g]) continue;
      const long long row = row_of(g, t);
      const float hp = t > 0 ? hout[(row - n) * H + j] : 0.f;
      const float d = dy[row * H + j] + dh[o];
      const float u = ru[row * 2 * H + u_col + j], c = cc[row * H + j];
      const float da_u = hard ? d * (hp - c) * qhard_sigmoid_grad(u) : d * (hp - c) * u * (1.f - u);
      const float da_c = d * (1.f - u) * (1.f - c * c);
      ds[g * 3 * H + u_col + j] = da_u;
      ds[g * 3 * H + 2 * H + j] = da_c;
      dag[row * 2 * H + u_col + j] = da_u;
      dac[row * H + j] = da_c;
      dn[o] = d * u;
    }
    __syncthreads();
    for (int o = threadIdx.x; o < ng * H; o += blockDim.x) {
      const int g = o / H, k = o % H;
      if (t >= lens[g]) continue;
      const long long row = row_of(g, t);
      const float* dc = ds + g * 3 * H + 2 * H;
      float drh = 0.f;
      for (int j = 0; j < H; j++) drh = fmaf(dc[j], wc[k * P1 + j], drh);
      const float hp = t > 0 ? hout[(row - n) * H + k] : 0.f;
      const float r = ru[row * 2 * H + r_col + k];
      const float da_r = hard ? drh * hp * qhard_sigmoid_grad(r) : drh * hp * r * (1.f - r);
      ds[g * 3 * H + r_col + k] = da_r;
      dag[row * 2 * H + r_col + k] = da_r;
      dn[o] += drh * r;
    }
    __syncthreads();
    for (int o = threadIdx.x; o < ng * H; o += blockDim.x) {
      const int g = o / H, k = o % H;
      if (t >= lens[g]) continue;
      const float* da = ds + g * 3 * H;
      float acc = dn[o];
      for (int j = 0; j < 2 * H; j++) acc = fmaf(da[j], wg[k * P2 + j], acc);
      dh[o] = acc;
    }
    __syncthreads();
  }
}

// GEMM A-loader of the GRU weight gradients (gemm_f32_kernel, K = agent rows): A'(m, row) = feature m of the row's
// input [x | h | 1]: x = fc1's output, h = hsrc[row] (shift 0) or the previous step's output of the same sequence
// (shift 1: hsrc[row - n], zero at t = 0); feature 2H is the ones row, whose product is the bias gradient.  The output
// [2H + 1, N] is the kernel [2H, N] followed by the bias [N], the variables' layout.
struct AGruFeat {
  static constexpr bool K_CONTIG = false;
  const float* x; const float* h; int H, n, T, shift;
  __device__ void prep_m(int, int, int, RowInfo*) const {}
  __device__ void prep_k(int k0, int Kend, int BK, RowInfo* rk) const {
    for (int i = threadIdx.x; i < BK; i += blockDim.x) {
      const int row = k0 + i;
      RowInfo r; r.valid = row < Kend; r.base = row; r.iy0 = 0;
      r.ix0 = shift ? (r.valid && (row / n) % T > 0 ? row - n : -1) : row;
      rk[i] = r;
    }
  }
  __device__ float load(int, int m, int kk, int, const RowInfo*, const RowInfo* rk) const {
    const RowInfo r = rk[kk];
    if (!r.valid) return 0.f;
    if (m < H) return x[(long long)r.base * H + m];
    if (m < 2 * H) return r.ix0 < 0 ? 0.f : h[(long long)r.ix0 * H + m - H];
    return 1.f;
  }
};

__device__ inline float qwarp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ inline float qsign(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }
// msum[0] = sum of mask[0..n), in a fixed order (one block), msum[1] = 1 / msum[0]
__global__ void __launch_bounds__(QM_THREADS)
qmix_mask_sum_kernel(const float* __restrict__ mask, int n, float* __restrict__ msum) {
  __shared__ float red[QM_THREADS];
  pdl_wait(); pdl_trigger();
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += mask[i];
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < QM_THREADS; w++) t += red[w]; msum[0] = t; msum[1] = 1.f / t; }
}

// _build_mix_net2 on one row r: y = elu(q . |w1| + b1) . |wf| + v.  Lane a holds q_a (a < n); lane j keeps the hidden
// units j + 32 i in hid[i].
struct QMixRow {
  float hid[QM_MAX_EMBED / 32];
  float y;
};
__device__ __forceinline__ QMixRow qmix_mix_row(float qa, const float* w1, const float* b1, const float* wf, float v, int n, int E, int lane) {
  QMixRow o;
  float part = 0.f;
#pragma unroll
  for (int i = 0; i < QM_MAX_EMBED / 32; i++) {
    const int j = lane + 32 * i;
    float pre = 0.f;
#pragma unroll 1
    for (int a = 0; a < n; a++) {
      const float q = __shfl_sync(0xffffffffu, qa, a);
      if (j < E) pre = fmaf(q, fabsf(w1[a * E + j]), pre);
    }
    if (j < E) {
      pre += b1[j];
      const float h = pre > 0.f ? pre : expm1f(pre);
      o.hid[i] = h;
      part = fmaf(h, fabsf(wf[j]), part);
    } else {
      o.hid[i] = 0.f;
    }
  }
  o.y = qwarp_sum(part) + v;
  return o;
}

// The TD step of QMixModel.build_train_graph (qmix_tf.py:401-481) for every (episode b, step t < L) row r = b L + t:
// chosen-action Q of every agent from qe (the eval agent's [B, T, n, A] output), the target value of step t+1 (double Q:
// the target Q at the argmax of the eval Q, both with unavailable actions at -999999 and ties to the lowest index as
// tf.argmax; else the masked max of the target Q), both mixers on the hypernet outputs (eval: w1 [rows, n E], b1, wf
// [rows, E], v [rows]; target: the *t arrays), td = q_tot - (reward + gamma (1 - terminated) target_q_tot) and
// loss = sum (mask td)^2 / sum mask.  Writes d loss / d (hypernet outputs) into dw1 / db1 / dwf / dv and d loss /
// d (chosen Q) into dq (zeroed by the caller, same layout as qe); part[block] = the block's sum of (mask td)^2, warp
// by warp in order.  msum: sum mask and its reciprocal (qmix_mask_sum_kernel).
__global__ void __launch_bounds__(QM_THREADS)
qmix_mix_td_kernel(const float* __restrict__ qe, const float* __restrict__ qt, const float* __restrict__ avail, const int32_t* __restrict__ act,
                   const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ wf, const float* __restrict__ v,
                   const float* __restrict__ w1t, const float* __restrict__ b1t, const float* __restrict__ wft, const float* __restrict__ vt,
                   const float* __restrict__ reward, const float* __restrict__ term, const float* __restrict__ mask,
                   const float* __restrict__ msum, int B, int L, int n,
                   int A, int E, float gamma, int double_q, float* __restrict__ dq, float* __restrict__ dw1, float* __restrict__ db1,
                   float* __restrict__ dwf, float* __restrict__ dv, float* __restrict__ part) {
  __shared__ float red[QM_THREADS];
  pdl_wait(); pdl_trigger();
  const int rows = B * L, T = L + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * (QM_THREADS / 32) + warp;
  float sq = 0.f;
  if (r < rows) {
    const int b = r / L, t = r % L;
    const long long cur = ((long long)b * T + t) * n, nxt = cur + n;
    float qa = 0.f, tqa = 0.f;
    int aa = 0;
    for (int a = 0; a < n; a++) {
      const int ac = act[(long long)r * n + a];
      const float* av = avail + (nxt + a) * A;
      const float* tq = qt + (nxt + a) * A;
      const float* eq = qe + (nxt + a) * A;
      float best = -INFINITY; int bi = A;
      for (int j = lane; j < A; j += 32) {
        const float x = av[j] == 0.f ? -999999.f : (double_q ? eq[j] : tq[j]);
        if (x > best) { best = x; bi = j; }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      const float tv = double_q ? (av[bi] == 0.f ? -999999.f : tq[bi]) : best;
      if (lane == a) { qa = qe[(cur + a) * A + ac]; tqa = tv; aa = ac; }
    }
    const QMixRow me = qmix_mix_row(qa, w1 + (long long)r * n * E, b1 + (long long)r * E, wf + (long long)r * E, v[r], n, E, lane);
    const QMixRow mt = qmix_mix_row(tqa, w1t + (long long)r * n * E, b1t + (long long)r * E, wft + (long long)r * E, vt[r], n, E, lane);
    const float m = mask[r];
    const float td = me.y - (reward[r] + gamma * (1.f - term[r]) * mt.y);
    const float mtd = td * m;
    sq = mtd * mtd;
    const float g = 2.f * mtd * m * msum[1];      // d loss / d q_tot (msum[1] = 1 / sum mask)
    if (lane == 0) dv[r] = g;
    float dqa = 0.f;
#pragma unroll
    for (int i = 0; i < QM_MAX_EMBED / 32; i++) {
      const int j = lane + 32 * i;
      const bool in = j < E;
      const float wfj = in ? wf[(long long)r * E + j] : 0.f, h = me.hid[i];
      const float dpre = g * fabsf(wfj) * (h > 0.f ? 1.f : h + 1.f);   // elu' from its output, as EluGrad
      if (in) { dwf[(long long)r * E + j] = g * h * qsign(wfj); db1[(long long)r * E + j] = dpre; }
#pragma unroll 1
      for (int a = 0; a < n; a++) {
        const float q = __shfl_sync(0xffffffffu, qa, a);
        if (in) dw1[((long long)r * n + a) * E + j] = dpre * q * qsign(w1[((long long)r * n + a) * E + j]);
      }
    }
    for (int a = 0; a < n; a++) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < QM_MAX_EMBED / 32; i++) {
        const int j = lane + 32 * i;
        if (j < E) {
          const float wfj = wf[(long long)r * E + j], h = me.hid[i];
          s = fmaf(g * fabsf(wfj) * (h > 0.f ? 1.f : h + 1.f), fabsf(w1[((long long)r * n + a) * E + j]), s);
        }
      }
      s = qwarp_sum(s);
      if (lane == a) dqa = s;
    }
    if (lane < n) dq[(cur + lane) * A + aa] = dqa;
  }
  if (lane == 0) red[warp] = sq;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < QM_THREADS / 32; w++) s += red[w];
    part[blockIdx.x] = s;
  }
}

// loss = (sum of the blocks' partial sums, in block order) / sum mask
__global__ void qmix_loss_kernel(const float* __restrict__ part, int n_part, const float* __restrict__ msum, float* __restrict__ out) {
  pdl_wait(); pdl_trigger();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < n_part; i++) s += part[i];
    *out = s / *msum;
  }
}

}  // namespace xtb
