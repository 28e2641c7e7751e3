// gemm_f32.cuh -- fp32 CUDA-core implicit-GEMM family (bring-up / reference path).
//
// One tiled kernel  C[m,n] = epi( sum_k A(m,k) * B(k,n) )  whose A/B operands are produced by
// loader functors (im2col gather with fused uint8 decode + minibatch gather, transposed-conv
// gather, transposed im2col for weight gradients, plain / transposed dense) and whose result is
// consumed by an epilogue functor (bias+activation, activation-gradient mask, split-K atomic
// accumulation).  The wgmma kernels in bp_gemm.cuh implement the same contracts on the
// tensor cores; this file is the numerically straightforward fp32 version they are checked
// against on the device, and the fallback for shapes the tensor-core path does not cover.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/xtb200.h"
#include "launch.cuh"

namespace xtb {

// keep the bf16 hi/lo planes of a tensor current (hi == NULL: tensor has no tensor-core consumer)
__device__ __forceinline__ void f32_store_plane(__nv_bfloat16* hi, long long lo_off, long long e, float x) {
  if (!hi) return;
  __nv_bfloat16 h = __float2bfloat16_rn(x);
  hi[e] = h;
  hi[lo_off + e] = __float2bfloat16_rn(x - __bfloat162float(h));
}

// exact floor(m/d) for 0 <= m < 2^24, 1 <= d < 2^16:  (m * (floor(2^40/d)+1)) >> 40   (the error term m*e/(d*2^40),
// e <= d, stays below 1/d while m*d < 2^40)
__host__ __device__ inline unsigned long long fastdiv_magic(int d) { return ((1ULL << 40) / (unsigned long long)d) + 1ULL; }
__device__ __forceinline__ int fastdiv(int m, unsigned long long magic) {
  return (int)(((unsigned long long)(unsigned)m * magic) >> 40);
}

struct ConvGeom {
  unsigned long long mP, mOW, mHW, mW;   // fastdiv magics of P, OW, H*W, W
  int H, W, C;        // input
  int OH, OW, Cout;   // output
  int KH, KW, S;      // kernel, stride
  int padT, padL;     // TF SAME: pad before; VALID: 0
  int K;              // KH*KW*C
  int P;              // OH*OW
};

// packed (ky,kx) pair
__host__ __device__ inline int pack_yx(int y, int x) { return (y << 16) | (x & 0xffff); }

struct RowInfo {  // per output-position info shared by conv loaders
  int base;       // element offset of the patch origin (may point before the image when padded)
  int iy0, ix0;   // top-left input coordinate of the patch
  int valid;      // row < M
};

__device__ inline float act_apply(int act, float x) {
  if (act == 1) return x > 0.f ? x : 0.f;
  if (act == 2) return tanhf(x);
  return x;
}
// derivative of the activation expressed with the activation OUTPUT y
__device__ inline float act_grad_from_out(int act, float y) {
  if (act == 1) return y > 0.f ? 1.f : 0.f;
  if (act == 2) return 1.f - y * y;
  return 1.f;
}

// ------------------------------------------------------------------------------------------
// The activations past tanh (enum xtb_act, include/xtb200.h).  The GEMM epilogues above and in bp_gemm.cuh apply only
// relu / tanh / linear: code for the others in their unrolled bodies slowed every network (instruction fetch, register
// pressure).  A layer with one of these runs its GEMM linear into fp32 and act_fwd_kernel applies the activation; the
// data gradients into its tensor are taken wrt its output y, and act_bwd_kernel turns their sum into the gradient wrt
// the pre-activation before the layer's own backward.
// ------------------------------------------------------------------------------------------
constexpr float kLeakyAlpha = 0.2f;
constexpr float kSeluScale = 1.0507009873554805f, kSeluAlpha = 1.6732632423543772f;
constexpr float kGeluC = 0.7978845608028654f, kGeluA = 0.044715f;   // sqrt(2/pi)

__host__ __device__ inline bool act_is_ext(int act) { return act > XTB_ACT_TANH; }
// the activations whose derivative is taken from the retained pre-activation z: y does not determine it (swish, gelu)
// or determines it badly near saturation (softsign)
__host__ __device__ inline bool act_keeps_z(int act) {
  return act == XTB_ACT_SOFTSIGN || act == XTB_ACT_SWISH || act == XTB_ACT_GELU;
}

__device__ inline float act_apply_ext(int act, float x) {
  switch (act) {
    case XTB_ACT_SIGMOID: return 1.f / (1.f + expf(-x));
    case XTB_ACT_SOFTSIGN: return x / (1.f + fabsf(x));
    case XTB_ACT_SOFTPLUS: return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));
    case XTB_ACT_LEAKY_RELU: return x > 0.f ? x : kLeakyAlpha * x;
    case XTB_ACT_ELU: return x > 0.f ? x : expm1f(x);
    case XTB_ACT_SELU: return kSeluScale * (x > 0.f ? x : kSeluAlpha * expm1f(x));
    case XTB_ACT_SWISH: return x / (1.f + expf(-x));
    case XTB_ACT_GELU: return 0.5f * x * (1.f + tanhf(kGeluC * (x + kGeluA * x * x * x)));
    default: return x;
  }
}
// derivative from u = the pre-activation z where act_keeps_z(act), the output y otherwise
__device__ inline float act_grad_ext(int act, float u) {
  switch (act) {
    case XTB_ACT_SIGMOID: return u * (1.f - u);
    case XTB_ACT_SOFTSIGN: { const float d = 1.f + fabsf(u); return 1.f / (d * d); }
    case XTB_ACT_SOFTPLUS: return -expm1f(-u);
    case XTB_ACT_LEAKY_RELU: return u > 0.f ? 1.f : kLeakyAlpha;
    case XTB_ACT_ELU: return u > 0.f ? 1.f : u + 1.f;
    case XTB_ACT_SELU: return u > 0.f ? kSeluScale : u + kSeluScale * kSeluAlpha;
    case XTB_ACT_SWISH: { const float s = 1.f / (1.f + expf(-u)); return s * (1.f + u * (1.f - s)); }
    case XTB_ACT_GELU: {
      const float t = tanhf(kGeluC * (u + kGeluA * u * u * u));
      return 0.5f * (1.f + t) + 0.5f * u * (1.f - t * t) * kGeluC * (1.f + 3.f * kGeluA * u * u);
    }
    default: return 1.f;
  }
}

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

// ------------------------------------------------------------------------------------------
// A loaders.  Interface:
//   static constexpr bool K_CONTIG      : thread mapping hint (k fastest in memory?)
//   __device__ void prep_m(int m0,int M,int BM, RowInfo* rm)   once per CTA
//   __device__ void prep_k(int k0,int Kend,int BK, RowInfo* rk) once per k-tile
//   __device__ float load(int mm,int m,int kk,int k, const RowInfo* rm, const RowInfo* rk)
// ------------------------------------------------------------------------------------------

__device__ inline void conv_row_info(const ConvGeom& g, const int32_t* idx, int m, int M, RowInfo& r) {
  r.valid = m < M;
  if (!r.valid) { r.base = 0; r.iy0 = 0; r.ix0 = 0; return; }
  int b = m / g.P;
  int p = m - b * g.P;
  int oy = p / g.OW;
  int ox = p - oy * g.OW;
  int sb = idx ? idx[b] : b;
  r.iy0 = oy * g.S - g.padT;
  r.ix0 = ox * g.S - g.padL;
  r.base = ((sb * g.H + r.iy0) * g.W + r.ix0) * g.C;
}

// forward conv: A(m,k) = x[b, oy*S-padT+ky, ox*S-padL+kx, ci]
template <typename T, bool PAD>
struct AIm2col {
  static constexpr bool K_CONTIG = true;
  const T* x; const int32_t* idx; ConvGeom g; const int* koff; const int* kyx;
  __device__ void prep_m(int m0, int M, int BM, RowInfo* rm) const {
    for (int i = threadIdx.x; i < BM; i += blockDim.x) conv_row_info(g, idx, m0 + i, M, rm[i]);
  }
  __device__ void prep_k(int, int, int, RowInfo*) const {}
  __device__ float load(int mm, int, int, int k, const RowInfo* rm, const RowInfo*) const {
    const RowInfo r = rm[mm];
    if (!r.valid) return 0.f;
    if (PAD) {
      int yx = kyx[k];
      int iy = r.iy0 + (yx >> 16), ix = r.ix0 + (yx & 0xffff);
      if ((unsigned)iy >= (unsigned)g.H || (unsigned)ix >= (unsigned)g.W) return 0.f;
    }
    return (float)x[(long long)r.base + koff[k]];
  }
};

// weight gradient of a conv: A'(m'=kw, k'=m) = im2col(m, kw); row kw==K is the all-ones bias row
template <typename T, bool PAD>
struct AIm2colT {
  static constexpr bool K_CONTIG = false;
  const T* x; const int32_t* idx; ConvGeom g; const int* koff; const int* kyx; int Mrows;  // Mrows = B*P
  __device__ void prep_m(int, int, int, RowInfo*) const {}
  __device__ void prep_k(int k0, int Kend, int BK, RowInfo* rk) const {
    for (int i = threadIdx.x; i < BK; i += blockDim.x) conv_row_info(g, idx, k0 + i, Kend, rk[i]);
  }
  __device__ float load(int, int m, int kk, int, const RowInfo*, const RowInfo* rk) const {
    const RowInfo r = rk[kk];
    if (!r.valid) return 0.f;
    if (m == g.K) return 1.f;
    if (PAD) {
      int yx = kyx[m];
      int iy = r.iy0 + (yx >> 16), ix = r.ix0 + (yx & 0xffff);
      if ((unsigned)iy >= (unsigned)g.H || (unsigned)ix >= (unsigned)g.W) return 0.f;
    }
    return (float)x[(long long)r.base + koff[m]];
  }
};

// data gradient of a conv (gather form of the transposed conv):
// rows m=(b,iy,ix) of dX, k=(ky,kx,co): A(m,k) = dY[b,(iy+padT-ky)/S,(ix+padL-kx)/S,co] when valid
struct ADgrad {
  static constexpr bool K_CONTIG = true;
  const float* dy; ConvGeom g; const int* dkyx; const int* dco; int sshift;
  __device__ void prep_m(int m0, int M, int BM, RowInfo* rm) const {
    int HW = g.H * g.W;
    for (int i = threadIdx.x; i < BM; i += blockDim.x) {
      int m = m0 + i; RowInfo r; r.valid = m < M;
      if (r.valid) {
        int b = m / HW; int p = m - b * HW; int iy = p / g.W; int ix = p - iy * g.W;
        r.base = b * g.P * g.Cout; r.iy0 = iy + g.padT; r.ix0 = ix + g.padL;
      } else { r.base = 0; r.iy0 = 0; r.ix0 = 0; }
      rm[i] = r;
    }
  }
  __device__ void prep_k(int, int, int, RowInfo*) const {}
  __device__ float load(int mm, int, int, int k, const RowInfo* rm, const RowInfo*) const {
    const RowInfo r = rm[mm];
    if (!r.valid) return 0.f;
    int yx = dkyx[k];
    int ty = r.iy0 - (yx >> 16), tx = r.ix0 - (yx & 0xffff);
    int mask = g.S - 1;
    if (ty < 0 || tx < 0 || (ty & mask) || (tx & mask)) return 0.f;
    int oy = ty >> sshift, ox = tx >> sshift;
    if (oy >= g.OH || ox >= g.OW) return 0.f;
    return dy[(long long)r.base + (oy * g.OW + ox) * g.Cout + dco[k]];
  }
};

// dense: A(m,k) = X[row(m)*ld + k]
template <typename T>
struct ADense {
  static constexpr bool K_CONTIG = true;
  const T* x; const int32_t* idx; int ld;
  __device__ void prep_m(int m0, int M, int BM, RowInfo* rm) const {
    for (int i = threadIdx.x; i < BM; i += blockDim.x) {
      int m = m0 + i; RowInfo r; r.valid = m < M; r.iy0 = r.ix0 = 0;
      r.base = r.valid ? (idx ? idx[m] : m) : 0;
      rm[i] = r;
    }
  }
  __device__ void prep_k(int, int, int, RowInfo*) const {}
  __device__ float load(int mm, int, int, int k, const RowInfo* rm, const RowInfo*) const {
    const RowInfo r = rm[mm];
    if (!r.valid) return 0.f;
    return (float)x[(long long)r.base * ld + k];
  }
};

// dense weight gradient: A'(m'=kw, k'=b) = X[row(b)*ld + kw]; row kw==Kw is the ones (bias) row
template <typename T>
struct ADenseT {
  static constexpr bool K_CONTIG = false;
  const T* x; const int32_t* idx; int ld; int Kw;
  __device__ void prep_m(int, int, int, RowInfo*) const {}
  __device__ void prep_k(int k0, int Kend, int BK, RowInfo* rk) const {
    for (int i = threadIdx.x; i < BK; i += blockDim.x) {
      int b = k0 + i; RowInfo r; r.valid = b < Kend; r.iy0 = r.ix0 = 0;
      r.base = r.valid ? (idx ? idx[b] : b) : 0;
      rk[i] = r;
    }
  }
  __device__ float load(int, int m, int kk, int, const RowInfo*, const RowInfo* rk) const {
    const RowInfo r = rk[kk];
    if (!r.valid) return 0.f;
    if (m == Kw) return 1.f;
    return (float)x[(long long)r.base * ld + m];
  }
};

// ------------------------------------------------------------------------------------------
// B loaders:  __device__ float load(int k, int n)   (k < K and n < N guaranteed by caller)
// ------------------------------------------------------------------------------------------
struct BRowMajor {     // B(k,n) = W[k*ld + n]
  const float* w; int ld;
  __device__ float load(int k, int n) const { return w[(long long)k * ld + n]; }
};
struct BTransposed {   // B(k,n) = W[n*ld + k]
  const float* w; int ld;
  __device__ float load(int k, int n) const { return w[(long long)n * ld + k]; }
};
struct BConvDgrad {    // B(k=(ky,kx,co), n=ci) = W[ky,kx,ci,co]
  const float* w; const int* wk; int Cout;
  __device__ float load(int k, int n) const { return w[wk[k] + n * Cout]; }
};

// ------------------------------------------------------------------------------------------
// Epilogues: __device__ void store(int m,int n,float acc)
// ------------------------------------------------------------------------------------------
struct EpiBiasAct {    // out = act(alpha*acc + bias[n])
  float* out; const float* bias; float alpha; int act; int ld; __nv_bfloat16* hi; long long lo_off;
  __device__ void store(int m, int n, float acc) const {
    long long o = (long long)m * ld + n;
    float r = act_apply(act, alpha * acc + bias[n]);
    out[o] = r;
    f32_store_plane(hi, lo_off, o, r);
  }
};
struct EpiDgrad {      // gout (+)= acc * act'(srcout)
  float* gout; const float* srcout; int act; int ld; int accumulate; __nv_bfloat16* hi; long long lo_off;
  __device__ void store(int m, int n, float acc) const {
    long long o = (long long)m * ld + n;
    float g = acc * act_grad_from_out(act, srcout[o]);
    float r = accumulate ? gout[o] + g : g;
    gout[o] = r;
    f32_store_plane(hi, lo_off, o, r);
  }
};
struct EpiAtomic {     // dW += alpha*acc  (split-K)
  float* out; float alpha; int ld;
  __device__ void store(int m, int n, float acc) const { atomicAdd(out + (long long)m * ld + n, alpha * acc); }
};

// ------------------------------------------------------------------------------------------
// The kernel.  TM x TN outputs per thread; grid = (ceil(M/BM), ceil(N/BN), ksplit)
// ------------------------------------------------------------------------------------------
template <int BM, int BN, int BK, int TM, int TN, class AL, class BL, class EP>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_f32_kernel(AL al, BL bl, EP ep, int M, int N, int K, int k_chunk) {
  pdl_wait(); pdl_trigger();
  constexpr int NT = (BM / TM) * (BN / TN);
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ RowInfo rm[AL::K_CONTIG ? BM : 1];
  __shared__ RowInfo rk[AL::K_CONTIG ? 1 : BK];

  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int kbeg = blockIdx.z * k_chunk;
  const int kend = min(K, kbeg + k_chunk);
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);

  al.prep_m(m0, M, BM, rm);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; i++)
#pragma unroll
    for (int j = 0; j < TN; j++) acc[i][j] = 0.f;
  __syncthreads();

  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    al.prep_k(k0, kend, BK, rk);
    if (!AL::K_CONTIG) __syncthreads();
#pragma unroll
    for (int e = tid; e < BM * BK; e += NT) {
      int mm, kk;
      if (AL::K_CONTIG) { kk = e % BK; mm = e / BK; } else { mm = e % BM; kk = e / BM; }
      float v = 0.f;
      if (m0 + mm < M && k0 + kk < kend) v = al.load(mm, m0 + mm, kk, k0 + kk, rm, rk);
      As[kk][mm] = v;
    }
#pragma unroll
    for (int e = tid; e < BN * BK; e += NT) {
      int nn = e % BN, kk = e / BN;
      float v = 0.f;
      if (n0 + nn < N && k0 + kk < kend) v = bl.load(k0 + kk, n0 + nn);
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; kk++) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i++) a[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; j++) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; i++) {
    int m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; j++) {
      int n = n0 + tx * TN + j;
      if (n < N) ep.store(m, n, acc[i][j]);
    }
  }
}

}  // namespace xtb
