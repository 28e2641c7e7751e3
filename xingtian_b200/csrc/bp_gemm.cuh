// bp_gemm.cuh -- wgmma GEMM family over "batch-planar" tensors for sm_90a (H100).
//
// Layout.  Every tensor on the tensor-core path (decoded frames, activations, activation gradients, weights) is
// stored as two bf16 planes hi = bf16(x), lo = bf16(x - hi) ("bf16x3": hi*hi + hi*lo + lo*hi with fp32 register
// accumulators reproduces fp32 products to ~2^-17) in the batch-planar order
//
//        element (row r, feature f)  ->  plane[ ((f >> 3) * pitch + r) * 8 + (f & 7) ]
//
// i.e. [feature chunk of 8][row][8]: for activations the row is the SAMPLE and a feature is (pixel, channel) in HWC
// order; for a weight matrix W[K, N] the row is k and the feature is n.  Consequences:
//   * the 16-byte pieces of consecutive rows are adjacent, so ANY operand tile -- the 128 samples x 64 channels of
//     one filter tap, the 64 samples x 128 features of a weight-gradient operand, a weight tile -- is a handful of
//     contiguous runs that the TMA engine moves with cp.async.bulk (no gather, no im2col copy, no tensor map), and
//     lands in shared memory directly in the wgmma no-swizzle (INTERLEAVE) canonical layout (8 rows x 16 B core
//     matrices);
//   * a convolution is a GEMM per output pixel whose M rows are the samples and whose K loop walks the filter
//     taps: stride, padding (out-of-image taps are simply skipped) and the transposed convolution of the data
//     gradient are all "which feature chunks does this stage read" -- no zero-filled operand tiles, no parity classes.
//
// Kernels (persistent, one CTA per SM, warp specialised: one bulk-copy producer warp fills a ring of shared-memory
// stages guarded by full / empty mbarriers; two consumer warpgroups issue wgmma on the stages, each owning 64 rows of
// the 128-row tile with its accumulator in registers, and run the epilogue from those registers):
//   bp_rows_kernel<0>  forward     D[b, n]  = act(alpha * sum_k A[b, k] W[k, n] + bias)        conv / dense
//   bp_rows_kernel<1>  forward, split-K partial sums (dense layers with a long K)
//   bp_rows_kernel<2>  data grad   D[b, k]  = (sum_n G[b, n] W[k, n]) * act'(X[b, k])           conv / dense
//   bp_wgrad_kernel    weight grad D[k, n]  = sum_b X[b, k] G[b, n]   (samples are the reduction axis; a conv layer's
//                      CTAs each own one accumulator (filter row ky, M tile) and a slice of the output pixels, and write
//                      per-slice partial sums that grad_reduce_kernel adds in a fixed order: no atomics)
// wgmma descriptors (no swizzle):  K-major operand  LBO = chunk-plane stride, SBO = 128 B, K step = 2 planes;
//                                  MN-major operand LBO = 128 B, SBO = chunk-plane stride, K step = 256 B.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "gemm_f32.cuh"

#ifndef XTB_BP_WAIT_HINT
#define XTB_BP_WAIT_HINT 20000u   // suspend-time hint (ns) of mbarrier.try_wait
#endif

namespace xtb {
namespace bp {

typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(XTB_BP_WAIT_HINT)
      : "memory");
  return ok;
}
// bounded wait: a protocol bug traps (kernel error) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 20)) __trap();
  }
}
// TMA bulk copy global -> shared (1-D, no tensor map); completion is counted in bytes on the mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// shared-memory load in the shared state space: a generic load could alias the global stores around it, which would
// pin it behind them.  Volatile keeps it after the mbarrier wait that makes the data visible.
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// one lane of a converged warp issues the bulk copies with warp-uniform operands
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// shared-memory matrix descriptor of wgmma, no swizzle (layout type 0, base offset 0)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// emits nothing: tells the compiler the accumulators' old values are dead before a scale-d 0 wgmma overwrites them (its
// "+f" operands would otherwise keep them live, e.g. through the epilogue that reads them last)
template <int R>
__device__ __forceinline__ void discard_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "=f"(d[i]));
}

// D[64 x n] (+)= A[64 x 16] B[16 x n], bf16 operands from shared memory, fp32 accumulators d[n / 2] in the wgmma
// register layout; TA / TB = 1: operand is MN-major ("transposed").  scale_d = 1: D += A B; scale_d = 0: D = A B, which
// starts an accumulator without register writes between wgmma instructions (those make ptxas serialize them, C7515).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]),
        "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]),
        "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n48(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, %27, %28;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]),
        "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]),
        "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n96(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, %51, %52;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]),
        "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]),
        "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]),
        "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
        "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
        "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]),
        "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]),
        "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
        "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma(float* d, uint64_t a, uint64_t b, uint32_t scale_d = 1) {
  static_assert(N == 16 || N == 32 || N == 48 || N == 64 || N == 96 || N == 128, "wgmma width");
  if constexpr (N == 16) wgmma_n16<TA, TB>(d, a, b, scale_d);
  else if constexpr (N == 32) wgmma_n32<TA, TB>(d, a, b, scale_d);
  else if constexpr (N == 48) wgmma_n48<TA, TB>(d, a, b, scale_d);
  else if constexpr (N == 64) wgmma_n64<TA, TB>(d, a, b, scale_d);
  else if constexpr (N == 96) wgmma_n96<TA, TB>(d, a, b, scale_d);
  else wgmma_n128<TA, TB>(d, a, b, scale_d);
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
// hi = bf16x2(a,b); lo = bf16x2(a - float(hi.a), b - float(hi.b)); a bf16 widened to fp32 is its bits << 16
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16(a, b);
  float ha = __uint_as_float(hi << 16), hb = __uint_as_float(hi & 0xffff0000u);
  lo = pack_bf16(a - ha, b - hb);
}
__device__ __forceinline__ void unpack2(uint32_t w, float& a, float& b) {
  a = __uint_as_float(w << 16);
  b = __uint_as_float(w & 0xffff0000u);
}
__device__ __forceinline__ void unpack8(const uint4& u, float v[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; i++) unpack2(w[i], v[2 * i], v[2 * i + 1]);
}
__device__ __forceinline__ void split8(const float v[8], uint4& hi, uint4& lo) {
  split2(v[0], v[1], hi.x, lo.x);
  split2(v[2], v[3], hi.y, lo.y);
  split2(v[4], v[5], hi.z, lo.z);
  split2(v[6], v[7], hi.w, lo.w);
}

// ------------------------------------------------------------------------------------------
// batch-planar tensor handle
// ------------------------------------------------------------------------------------------
struct BpT {
  bf16* hi;            // hi plane; NULL = absent
  long long lo_off;    // lo plane = hi + lo_off (elements)
  int pitch;           // rows per feature chunk (multiple of 16)
};
__host__ __device__ inline long long bp_index(int pitch, int row, int f) { return ((long long)(f >> 3) * pitch + row) * 8 + (f & 7); }

// Warp roles of both GEMM kernels: warps 0..7 are two consumer warpgroups (wgmma needs a warpgroup to start at a warp
// index that is a multiple of 4), warp 8 is the producer.  Consumer warpgroup g computes rows [64 g, 64 g + 64) of
// every tile; its warp w holds rows 16 w + lane / 4 (+ 8) and columns 8 i + 2 (lane % 4) (+ 1) of the accumulator.
constexpr int BP_CONSUMER_WGS = 2;
constexpr int BP_P_WARP = 4 * BP_CONSUMER_WGS;
constexpr int BP_THREADS = 32 * (BP_P_WARP + 1);
constexpr int BP_CONSUMER_WARPS = 4 * BP_CONSUMER_WGS;   // arrivals that free a ring slot (one per consumer warp)

// ------------------------------------------------------------------------------------------
// bp_rows_kernel: the M rows of a tile are 128 samples; a "unit" is what one accumulator tile produces
//   conv forward  : unit = output pixel, N = Cout           K stages walk the filter rows of that pixel
//   conv data grad: unit = input pixel,  N = Cin            K stages walk the taps that reach that pixel
//   dense         : unit = (N tile, K split)                K stages walk a range of feature chunks
// Weights ("blob"): batch-planar W^T, i.e. [n chunk][k row][8] with pitch = K rows.  Forward reads it MN-major (rows k,
// chunks along n), the data gradient K-major (rows = output feature k, chunks along the reduction n): same bytes.
//
// The stage walk of a conv unit (which feature chunks, which weight rows) is a host-built table (StageEnt per stage,
// UnitEnt per unit, built once per layer in xtb_net_create): the role loops are a table fetch, an mbarrier wait and a
// handful of adds per stage.
// ------------------------------------------------------------------------------------------
constexpr int RW_THREADS = BP_THREADS;
constexpr int RW_A_PLANE = 2048;                 // 128 rows x 16 B
constexpr int RW_STAGE_A = 2 * 8 * RW_A_PLANE;   // hi + lo, 8 chunks (64 K elements)
constexpr int RW_STAGE_B = 16384;
constexpr int RW_MAX_STAGES = 4;
constexpr int RW_EPI_BANKS = 2;                  // data-gradient epilogue operand buffers (one per accumulator bank)

// Planes the data-gradient epilogue reads besides its accumulator: the source activation for act' (relu: hi; tanh: hi
// and lo) and, when it accumulates, the output planes (hi and lo).  The producer warp prefetches them into shared memory.
__host__ __device__ inline int dgrad_epi_planes(int src_act, int accumulate) {
  return (src_act == 1 ? 1 : (src_act == 2 ? 2 : 0)) + (accumulate ? 2 : 0);
}

struct StageEnt {            // one K stage of a conv unit (8 bytes; the tables are copied to shared memory at kernel start)
  uint32_t a_chunk;          // first operand feature chunk of the stage
  uint16_t w_row;            // first weight-blob row of the stage (forward: k row; data gradient: tap * Cin)
  uint16_t nch;              // feature chunks in this stage (even, <= 8)
};
typedef uint32_t UnitEnt;    // first stage index | stage count << 24
struct StageDesc { uint32_t a_off, w_off, nch; };   // byte offsets inside a plane / blob plane

struct RowsArgs {
  BpT a; int a_split;                               // operand rows (activations / gradients); a_split: lo plane is read
  const bf16* w_hi; const bf16* w_lo; int w_pitch;  // weight blob planes
  int w_res; int w_res_chunks;                      // blob resident in shared memory (conv): chunks to load per plane
  int mode;                                         // 0 conv forward, 1 conv data gradient, 2 dense
  const StageEnt* stages; const UnitEnt* units;     // conv stage walk (global; n_stage_ents / n_units entries)
  int n_stage_ents;
  int kchunks, kc_split, n_ntiles;                  // dense: K chunks in total / per split, N tiles
  int n_units, n_btiles, B, N;                      // tiles = n_units * n_btiles; N = accumulator columns per plane
  // forward epilogue
  BpT out; float* out_f32; int ld_f32; const float* bias; float alpha; int act;
  float* part; long long part_z; int ld_part;       // split-K partial sums part[z][b][ld_part]
  // data-gradient epilogue: out = acc * act'(src) (+ out); column sums into db_part[cta][N] when non-NULL
  BpT src; int src_act; int accumulate; float* db_part;
};

// per-tile stage source: conv = run of the shared-memory table, dense = arithmetic progression.  setup() copies the
// kernel parameters it needs into registers once per role.
struct TileWalk {
  const uint2* stages_sm; const uint32_t* units_sm;
  uint32_t a_pstride, w_pitch; int mode, n_ntiles, kc_split, kchunks, N;
  const uint2* st; uint32_t a0, w0, da, dw; int ns, nch_last;
  __device__ __forceinline__ void setup(const RowsArgs& a, const uint2* s_sm, const uint32_t* u_sm) {
    stages_sm = s_sm; units_sm = u_sm;
    a_pstride = (uint32_t)a.a.pitch * 16u; w_pitch = (uint32_t)a.w_pitch;
    mode = a.mode; n_ntiles = a.n_ntiles; kc_split = a.kc_split; kchunks = a.kchunks; N = a.N;
  }
  template <int KIND>
  __device__ __forceinline__ void init(int u) {
    if (mode == 2) {
      const int nt = u % n_ntiles, z = u / n_ntiles;
      const int cbeg = z * kc_split, cend = min(kchunks, cbeg + kc_split);
      ns = (cend - cbeg + 7) >> 3;
      nch_last = cend - cbeg - 8 * (ns - 1);
      a0 = (uint32_t)cbeg * a_pstride; da = 8u * a_pstride;
      if (KIND == 2) { w0 = ((uint32_t)cbeg * w_pitch + (uint32_t)nt * N) * 16u; dw = 8u * w_pitch * 16u; }
      else { w0 = ((uint32_t)(nt * (N >> 3)) * w_pitch + (uint32_t)cbeg * 8u) * 16u; dw = 1024u; }
      st = nullptr;
    } else {
      const uint32_t ue = units_sm[u];
      st = stages_sm + (ue & 0xffffffu); ns = (int)(ue >> 24);
    }
  }
  __device__ __forceinline__ StageDesc get(int s) const {
    if (st) {
      const uint2 v = st[s];
      return StageDesc{v.x * a_pstride, (v.y & 0xffffu) * 16u, v.y >> 16};
    }
    return StageDesc{a0 + (uint32_t)s * da, w0 + (uint32_t)s * dw, (uint32_t)(s == ns - 1 ? nch_last : 8)};
  }
};

// N = accumulator columns per plane (16, 32, 48 or 64).  epi_banks: data-gradient epilogue buffers (0 when the epilogue
// reads nothing but its accumulator, else 1 or 2; see rows_smem)
template <int KIND, int N>
__global__ void __launch_bounds__(RW_THREADS, 1)
bp_rows_kernel(const __grid_constant__ RowsArgs a, int n_stages, int stage_bytes, int wres_bytes, int epi_banks) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  constexpr int NCH = N >> 3;                            // feature chunks of an accumulator tile
  // data-gradient epilogue operands behind the stage ring: per bank [plane][chunk][128 rows][16 B]
  const int epi_planes = KIND == 2 ? dgrad_epi_planes(a.src_act, a.accumulate) : 0;
  const int epi_bank_bytes = epi_planes * NCH * RW_A_PLANE;
  uint8_t* epi_sm = smem + wres_bytes + n_stages * stage_bytes;
  // stage-walk tables behind those: [stages : n_stage_ents x 8 B][units : n_units x 4 B]
  uint2* stages_sm = reinterpret_cast<uint2*>(epi_sm + epi_banks * epi_bank_bytes);
  uint32_t* units_sm = reinterpret_cast<uint32_t*>(stages_sm + a.n_stage_ents);
  __shared__ __align__(8) uint64_t bars[2 * RW_MAX_STAGES + 1 + 2 * RW_EPI_BANKS];
  __shared__ float red_sh[BP_CONSUMER_WARPS][64];
  __shared__ float bias_sh[64];

  // warp index through a shuffle: provably warp-uniform, so ptxas treats the role branches as non-divergent and does
  // not serialize the wgmma instructions behind them
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[RW_MAX_STAGES]), wbar = smem_u32(&bars[2 * RW_MAX_STAGES]);
  const uint32_t efull0 = wbar + 8, eempty0 = efull0 + 8 * RW_EPI_BANKS;
  if (tid == 0) {
    for (int s = 0; s < RW_MAX_STAGES; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, BP_CONSUMER_WARPS); }
    mbar_init(wbar, 1);
    for (int k = 0; k < RW_EPI_BANKS; k++) { mbar_init(efull0 + 8 * k, 1); mbar_init(eempty0 + 8 * k, BP_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  // Static inputs are fetched BEFORE the dependency wait, i.e. under the tail of the preceding kernel: the stage-walk
  // tables never change after bind, and the weight blob of a conv layer was written at least two kernels back (by the
  // blob refresh of the previous optimiser step; the layer's own operand producer sits in between), so it is complete
  // by the time the previous kernel has passed its own wait and released this one.
  if (a.mode != 2) {      // every thread helps, one barrier
    const uint2* gs = reinterpret_cast<const uint2*>(a.stages);
    for (int i = tid; i < a.n_stage_ents; i += RW_THREADS) stages_sm[i] = __ldg(gs + i);
    for (int i = tid; i < a.n_units; i += RW_THREADS) units_sm[i] = __ldg(a.units + i);
  }
  if (warp == BP_P_WARP && a.w_res && elect_one()) {
    const uint32_t bytes = (uint32_t)a.w_res_chunks * a.w_pitch * 16;
    mbar_expect_tx(wbar, 2 * bytes);
    bulk_g2s(smem_u32(smem), a.w_hi, bytes, wbar);
    bulk_g2s(smem_u32(smem) + bytes, a.w_lo, bytes, wbar);
  }
  pdl_wait();
  pdl_trigger();
  if (KIND == 0 && a.mode != 2 && tid < N) bias_sh[tid] = a.bias[tid];
  __syncthreads();
  const uint32_t wres = smem_u32(smem);                  // resident weights: hi plane chunks then lo plane chunks
  const uint32_t stage0 = wres + (uint32_t)wres_bytes;
  const int total = a.n_units * a.n_btiles;
  constexpr bool CAT = (KIND != 2);                      // forward: one MMA over [W_hi | W_lo], accumulator 2N columns
  const int nbt = a.n_btiles;
  // tile = blockIdx.x + i * gridDim.x  ->  (unit u, batch tile bt), advanced without divisions
  const int du = (int)gridDim.x / nbt, dbt = (int)gridDim.x - du * nbt;

  if (warp == BP_P_WARP) {
    // ================= TMA producer: converged warp, one elected lane issues the copies ==============================
    const bool a_split = a.a_split != 0, w_res = a.w_res != 0;
    const uint32_t a_pstride = (uint32_t)a.a.pitch * 16u, w_pstride = (uint32_t)a.w_pitch * 16u;
    const char* a_hi = reinterpret_cast<const char*>(a.a.hi);
    const char* a_lo = a_hi + a.a.lo_off * 2;
    const char* w_hi = reinterpret_cast<const char*>(a.w_hi);
    const char* w_lo = reinterpret_cast<const char*>(a.w_lo);
    constexpr int n_bh_fwd = N >> 3;
    int stage = 0; uint32_t phase = 0;
    int u = (int)blockIdx.x / nbt, bt = (int)blockIdx.x - u * nbt;
    const int Bsz = a.B;
    TileWalk tw; tw.setup(a, stages_sm, units_sm);
    // data-gradient epilogue operands: source planes (act'), then output planes (accumulate)
    const int src_act = a.src_act, accumulate = a.accumulate;
    const char* s_hi = reinterpret_cast<const char*>(a.src.hi);
    const char* s_lo = s_hi + a.src.lo_off * 2;
    const char* o_hi = reinterpret_cast<const char*>(a.out.hi);
    const char* o_lo = o_hi + a.out.lo_off * 2;
    const uint32_t s_ps = (uint32_t)a.src.pitch * 16u, o_ps = (uint32_t)a.out.pitch * 16u;
    int ebank = 0; uint32_t ephase = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const int b0 = bt * 128, nr = min(128, Bsz - b0);
      const uint32_t a_bytes = (uint32_t)nr * 16u, row_off = (uint32_t)b0 * 16u;
      tw.init<KIND>(u);
      for (int s = 0; s < tw.ns; s++) {
        const StageDesc d = tw.get(s);
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const int nch = (int)d.nch;
        const int n_bh = w_res ? 0 : (KIND == 2 ? nch : n_bh_fwd);
        const uint32_t b_bytes = (KIND == 2) ? (uint32_t)N * 16u : (uint32_t)nch * 128u;
        const uint32_t fb = full0 + 8 * stage;
        if (elect_one()) {
          mbar_expect_tx(fb, a_bytes * (a_split ? 2 * nch : nch) + b_bytes * 2 * n_bh);
          const uint32_t sA = stage0 + (uint32_t)stage * stage_bytes, sB = sA + RW_STAGE_A;
          const char* ah = a_hi + d.a_off + row_off;
          for (int c = 0; c < nch; c++) bulk_g2s(sA + c * RW_A_PLANE, ah + (uint32_t)c * a_pstride, a_bytes, fb);
          if (a_split) {
            const char* al = a_lo + d.a_off + row_off;
            for (int c = 0; c < nch; c++) bulk_g2s(sA + 8 * RW_A_PLANE + c * RW_A_PLANE, al + (uint32_t)c * a_pstride, a_bytes, fb);
          }
          if (!w_res) {
            const char* wh = w_hi + d.w_off; const char* wl = w_lo + d.w_off;
            if (KIND == 2) {
              for (int c = 0; c < n_bh; c++) {
                bulk_g2s(sB + c * (N * 16), wh + (uint32_t)c * w_pstride, b_bytes, fb);
                bulk_g2s(sB + 8192 + c * (N * 16), wl + (uint32_t)c * w_pstride, b_bytes, fb);
              }
            } else {
              for (int c = 0; c < n_bh; c++) {
                bulk_g2s(sB + c * 1024, wh + (uint32_t)c * w_pstride, b_bytes, fb);
                bulk_g2s(sB + (n_bh_fwd + c) * 1024, wl + (uint32_t)c * w_pstride, b_bytes, fb);
              }
            }
          }
        }
        __syncwarp();
        if (++stage == n_stages) { stage = 0; phase ^= 1; }
      }
      // The tile's epilogue operands, issued behind its K stages: the epilogue runs only after the first stage of the
      // next tile, so the copies have a tile's MMAs to land, and the ring is never held up by the bank still in use by
      // the epilogue before.  Rows [b0, b0 + nr) of the unit's NCH output chunks, per plane.
      if (KIND == 2 && epi_planes) {
        mbar_wait(eempty0 + 8 * ebank, ephase ^ 1);
        if (elect_one()) {
          const uint32_t fb = efull0 + 8 * ebank;
          mbar_expect_tx(fb, a_bytes * (uint32_t)(NCH * epi_planes));
          const uint32_t oc0 = (uint32_t)((tw.mode == 2 ? u % tw.n_ntiles : u) * NCH);
          uint32_t dst = smem_u32(epi_sm) + (uint32_t)(ebank * epi_bank_bytes);
          auto plane = [&](const char* base, uint32_t ps) {
            const char* src = base + oc0 * ps + row_off;
            for (int c = 0; c < NCH; c++, dst += RW_A_PLANE) bulk_g2s(dst, src + (uint32_t)c * ps, a_bytes, fb);
          };
          if (src_act == 1 || src_act == 2) plane(s_hi, s_ps);
          if (src_act == 2) plane(s_lo, s_ps);
          if (accumulate) { plane(o_hi, o_ps); plane(o_lo, o_ps); }
        }
        __syncwarp();
        if (++ebank == epi_banks) { ebank = 0; ephase ^= 1; }
      }
      u += du; bt += dbt;
      if (bt >= nbt) { bt -= nbt; u++; }
    }
  } else if (warp < BP_P_WARP) {
    // ================= consumers: wgmma on the ring stages, epilogue from the accumulator registers =================
    constexpr int ACC = CAT ? 2 * N : N;                 // accumulator columns
    float dbacc[N / 4];                                  // data gradient: column sums of this thread's columns
#pragma unroll
    for (int j = 0; j < N / 4; j++) dbacc[j] = 0.f;
    const int wg = warp >> 2, q = lane & 3;
    const int row_in_tile = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const bool a_split = a.a_split != 0, w_res = a.w_res != 0;
    // kernel parameters used per tile live in registers: the barrier waits are asm volatile with a memory clobber, after
    // which the compiler would re-read the constant bank
    const int act = a.act, mode = a.mode, Bsz = a.B, n_nt = a.n_ntiles, ld_f32 = a.ld_f32, src_act = a.src_act, accumulate = a.accumulate;
    const int ld_part = a.ld_part;
    const float alpha = a.alpha;
    bf16* const out_hi = a.out.hi; const long long out_lo = a.out.lo_off;
    float* const out_f32 = a.out_f32; const float* const bias_g = a.bias;
    float* const part = a.part; const long long part_z = a.part_z;
    const long long out_pstride = (long long)a.out.pitch * 8;      // elements between feature chunks
    const int b_pad = (Bsz + 15) & ~15;
    // data-gradient epilogue operands in shared memory: this thread's word of (plane p, chunk i, tile row r) lies at
    // epi_thr + bank * epi_bank_bytes + (p * NCH + i) * RW_A_PLANE + 16 * (r - row_in_tile); the output planes follow
    // the source planes
    const uint32_t epi_thr = smem_u32(epi_sm) + (uint32_t)(row_in_tile * 16 + 4 * q);
    const int epi_out_plane = epi_planes - (accumulate ? 2 : 0);
    int ebank = 0; uint32_t ephase = 0;
    // descriptor constant parts; the low 14 bits hold (shared address >> 4) and are advanced by plain adds
    const uint64_t adesc = make_desc(0, RW_A_PLANE, 128);
    const uint64_t bdesc = (KIND == 2) ? make_desc(0, (uint32_t)N * 16, 128) : make_desc(0, 128, 1024);
    const uint32_t a_row_add = (uint32_t)(wg * 64 * 16) >> 4;      // this warpgroup's 64 rows
    const uint32_t a_lo_add = (8 * RW_A_PLANE) >> 4, a_step = (2 * RW_A_PLANE) >> 4;
    const uint32_t w_pstride = (uint32_t)a.w_pitch * 16u;
    // resident weights: forward MN-major (LBO 128, SBO = pitch rows), data gradient K-major (LBO = pitch rows, SBO 128)
    const uint64_t wdesc = (KIND == 2) ? make_desc(0, w_pstride, 128) : make_desc(0, 128, w_pstride);
    const uint32_t w_lo_add = ((uint32_t)a.w_res_chunks * w_pstride) >> 4;
    const uint32_t b_step = (KIND == 2) ? (w_res ? (2 * w_pstride) >> 4 : (2u * N * 16u) >> 4) : (256 >> 4);
    const uint32_t b_lo_add = w_res ? w_lo_add : (8192 >> 4);
    const uint64_t b_const = w_res ? wdesc : bdesc;
    if (w_res) mbar_wait(wbar, 0);
    int stage = 0; uint32_t phase = 0;
    int held = -1;                                       // ring slot whose wgmma group may still be reading
    // this warpgroup's 64 rows of batch tile bt all lie at or beyond B: no MMAs and no epilogue for that tile
    auto idle = [&](int bt) { return bt * 128 + wg * 64 >= Bsz; };

    // One K stage into accumulator bank acc; the first stage of a tile starts the bank with scale-d 0.  Every value that
    // steers a branch or a trip count between wgmma_fence and wgmma_wait must be provably warp-uniform (kernel
    // parameters, shuffle results and what derives from them): ptxas otherwise serializes the wgmma instructions (C7520),
    // one MMA in flight at a time.  An idle warpgroup still waits on the full barrier and frees the slot, so the producer
    // protocol does not change.
    auto mma_stage = [&](float* acc, const StageDesc& d, bool first, bool skip) {
      mbar_wait(full0 + 8 * stage, phase);
      const uint32_t sA = stage0 + (uint32_t)stage * stage_bytes;
      uint32_t a_lo32 = (sA >> 4) + a_row_add;
      uint32_t b_lo32 = w_res ? (wres + d.w_off) >> 4 : (sA + RW_STAGE_A) >> 4;
      const int ksteps = __shfl_sync(0xffffffffu, skip ? 0 : (int)d.nch >> 1, 0);
      uint32_t sd = first ? 0u : 1u;
      wgmma_fence();
      // the a_split test stays outside the issue loops: a branch between wgmma instructions makes ptxas serialize them
      if (a_split) {
        for (int j = 0; j < ksteps; j++) {
          const uint64_t ah = adesc | a_lo32, bh = b_const | b_lo32, al = adesc | (a_lo32 + a_lo_add);
          if (KIND != 2) {
            wgmma<2 * N, 0, 1>(acc, ah, bh, sd);                                   // A_hi x [W_hi | W_lo]
            wgmma<N, 0, 1>(acc, al, bh);                                           // A_lo x W_hi
          } else {
            wgmma<N, 0, 0>(acc, ah, bh, sd);
            wgmma<N, 0, 0>(acc, ah, b_const | (b_lo32 + b_lo_add));
            wgmma<N, 0, 0>(acc, al, bh);
          }
          a_lo32 += a_step; b_lo32 += b_step; sd = 1u;
        }
      } else {
        for (int j = 0; j < ksteps; j++) {
          const uint64_t ah = adesc | a_lo32, bh = b_const | b_lo32;
          if (KIND != 2) {
            wgmma<2 * N, 0, 1>(acc, ah, bh, sd);
          } else {
            wgmma<N, 0, 0>(acc, ah, bh, sd);
            wgmma<N, 0, 0>(acc, ah, b_const | (b_lo32 + b_lo_add));
          }
          a_lo32 += a_step; b_lo32 += b_step; sd = 1u;
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                                   // all earlier groups are complete: free the slot they read
      if (held >= 0 && lane == 0) mbar_arrive(empty0 + 8 * held);
      held = stage;
      if (++stage == n_stages) { stage = 0; phase ^= 1; }
    };

    int tile = blockIdx.x;
    int u = (int)blockIdx.x / nbt, bt = (int)blockIdx.x - u * nbt;
    TileWalk tw; tw.setup(a, stages_sm, units_sm);
    // issue the first stage of tile (u, bt) into bank acc; false if the unit has no stages
    auto start_tile = [&](float* acc) {
      tw.init<KIND>(u);
      tw.ns = __shfl_sync(0xffffffffu, tw.ns, 0);
      if (tw.ns == 0) return false;
      discard_regs<ACC / 2>(acc);
      mma_stage(acc, tw.get(0), true, idle(bt));
      return true;
    };

    // epilogue of tile (cu, cbt) from bank cur: bias / activation / ReLU mask, batch-planar and fp32 stores.  The data
    // gradient reads act' and the accumulated planes from the epilogue buffer at shared address eb (this thread's word)
    auto epilogue = [&](const float* cur, int cu, int cbt, bool empty, uint32_t eb) {
      const int btile0 = cbt * 128;
      int oc0, z = 0;                          // first output chunk of the unit
      if (mode == 2) { const int nt = cu % n_nt; z = cu / n_nt; oc0 = nt * NCH; }
      else oc0 = cu * NCH;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int b = btile0 + row_in_tile + 8 * h;
#pragma unroll
        for (int i = 0; i < NCH; i++) {
          const int c = 8 * i + 2 * q;           // column inside the tile
          float v0 = cur[4 * i + 2 * h], v1 = cur[4 * i + 2 * h + 1];
          if (CAT) { v0 += cur[4 * (i + NCH) + 2 * h]; v1 += cur[4 * (i + NCH) + 2 * h + 1]; }
          if (empty) { v0 = 0.f; v1 = 0.f; }
          if (KIND == 0) {
            if (b < Bsz) {
              const int f = oc0 * 8 + c;
              float bb0, bb1;
              if (mode == 2) { const float2 t2 = __ldg(reinterpret_cast<const float2*>(bias_g + f)); bb0 = t2.x; bb1 = t2.y; }
              else { bb0 = bias_sh[c]; bb1 = bias_sh[c + 1]; }
              if (act == 2) { v0 = tanhf(alpha * v0 + bb0); v1 = tanhf(alpha * v1 + bb1); }
              else {            // relu / linear without a branch per element
                const float lo = act == 1 ? 0.f : -INFINITY;
                v0 = fmaxf(fmaf(alpha, v0, bb0), lo); v1 = fmaxf(fmaf(alpha, v1, bb1), lo);
              }
              if (out_hi) {
                bf16* p = out_hi + (long long)(oc0 + i) * out_pstride + (long long)b * 8 + 2 * q;
                uint32_t hi, lo;
                split2(v0, v1, hi, lo);
                *reinterpret_cast<uint32_t*>(p) = hi;
                *reinterpret_cast<uint32_t*>(p + out_lo) = lo;
              }
              if (out_f32) *reinterpret_cast<float2*>(out_f32 + (long long)b * ld_f32 + f) = make_float2(v0, v1);
            }
          } else if (KIND == 1) {
            if (b < Bsz)
              *reinterpret_cast<float2*>(part + (long long)z * part_z + (long long)b * ld_part + oc0 * 8 + c) = make_float2(v0, v1);
          } else {
            bf16* p = out_hi + (long long)(oc0 + i) * out_pstride + (long long)b * 8 + 2 * q;
            if (b < Bsz) {
              const uint32_t e = eb + (uint32_t)(i * RW_A_PLANE + 128 * h);        // plane 0, chunk i, row b
              if (src_act == 1) {
                float s0, s1;
                unpack2(lds_u32(e), s0, s1);
                v0 = s0 > 0.f ? v0 : 0.f; v1 = s1 > 0.f ? v1 : 0.f;
              } else if (src_act == 2) {
                float s0, s1, t0, t1;
                unpack2(lds_u32(e), s0, s1);
                unpack2(lds_u32(e + NCH * RW_A_PLANE), t0, t1);
                const float y0 = s0 + t0, y1 = s1 + t1;
                v0 *= 1.f - y0 * y0; v1 *= 1.f - y1 * y1;
              }
              dbacc[2 * i] += v0; dbacc[2 * i + 1] += v1;
              if (accumulate) {
                const uint32_t eo = e + (uint32_t)(epi_out_plane * NCH * RW_A_PLANE);
                float s0, s1, t0, t1;
                unpack2(lds_u32(eo), s0, s1);
                unpack2(lds_u32(eo + NCH * RW_A_PLANE), t0, t1);
                v0 += s0 + t0; v1 += s1 + t1;
              }
              uint32_t hi, lo;
              split2(v0, v1, hi, lo);
              *reinterpret_cast<uint32_t*>(p) = hi;
              *reinterpret_cast<uint32_t*>(p + out_lo) = lo;
            } else if (b < b_pad && !accumulate) {
              // gradient rows up to the next multiple of 16 are read by the weight-gradient K loop: keep them zero
              *reinterpret_cast<uint32_t*>(p) = 0u;
              *reinterpret_cast<uint32_t*>(p + out_lo) = 0u;
            }
          }
        }
      }
    };

    // Tile loop, software-pipelined over two accumulator banks: the remaining stages of the current tile go into cur,
    // then the first stage of the next tile into nxt, and the current tile's epilogue runs while that group is on the
    // tensor pipe (its operands are in shared memory).  The wgmma_wait<1> of that first stage completes cur's groups.
    // Registers cannot be indexed at run time, so the loop is unrolled by two: even tiles in acc0, odd tiles in acc1.
    // The forward at N = 64 (2 x 64 accumulators per bank) does not fit both banks and the epilogue in the 168 registers
    // per thread of a 288-thread CTA: it starts the next tile after the epilogue instead, one bank live at a time.
    constexpr bool OVERLAP = !(KIND == 0 && N == 64);
    auto finish_tile = [&](float* cur, float* nxt) {
      for (int s = 1; s < tw.ns; s++) mma_stage(cur, tw.get(s), false, idle(bt));
      // a unit without stages (a data-gradient pixel that no filter tap reaches) stores zeros: its bank was never
      // written, and zeroing it here would put register writes between wgmma instructions
      const bool empty = tw.ns == 0;
      const int cu = u, cbt = bt;
      tile += gridDim.x; u += du; bt += dbt;
      if (bt >= nbt) { bt -= nbt; u++; }
      if (!(OVERLAP && tile < total && start_tile(nxt))) {
        wgmma_wait<0>();
        if (held >= 0 && lane == 0) mbar_arrive(empty0 + 8 * held);
        held = -1;
      }
      fence_regs<ACC / 2>(cur);
      // every consumer warp waits for the tile's epilogue operands, idle ones included (the producer copies them for
      // every tile): a wait loop inside the idle branch, with the next tile's wgmma group in flight, makes ptxas
      // serialize the kernel's wgmma instructions (C7518)
      if (KIND == 2 && epi_planes) mbar_wait(efull0 + 8 * ebank, ephase);
      if (!idle(cbt)) epilogue(cur, cu, cbt, empty, epi_thr + (uint32_t)(ebank * epi_bank_bytes));
      if (KIND == 2 && epi_planes) {       // every consumer warp frees the bank
        __syncwarp();
        if (lane == 0) mbar_arrive(eempty0 + 8 * ebank);
        if (++ebank == epi_banks) { ebank = 0; ephase ^= 1; }
      }
      if (!OVERLAP && tile < total) start_tile(nxt);
    };
    float acc0[ACC / 2], acc1[ACC / 2];
    if (tile < total) start_tile(acc0);
    while (tile < total) {
      finish_tile(acc0, acc1);
      if (tile >= total) break;
      finish_tile(acc1, acc0);
    }
    if (KIND == 2 && a.db_part) {
      // column sums of this CTA: the 8 row lanes of a column -> one row per consumer warp -> fixed-order sum over warps
#pragma unroll
      for (int j = 0; j < N / 4; j++) {
        float s = dbacc[j];
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        s += __shfl_xor_sync(0xffffffffu, s, 8);
        s += __shfl_xor_sync(0xffffffffu, s, 16);
        if (lane < 4) red_sh[warp][8 * (j >> 1) + 2 * lane + (j & 1)] = s;
      }
      asm volatile("bar.sync 1, %0;" ::"n"(32 * BP_CONSUMER_WARPS) : "memory");
      if (tid < N) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < BP_CONSUMER_WARPS; w++) t += red_sh[w][tid];
        a.db_part[(long long)blockIdx.x * N + tid] = t;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// bp_wgrad_kernel: dW[k, n] = sum_b X[b, k] G[b, n].  Both operands are MN-major (their shared-memory rows are the
// reduction axis = samples), one K chunk = 64 samples.  M = 128 features of X = 16 consecutive feature chunks:
//   conv  : the KW*C features of one filter row at one output pixel are contiguous ("run"); accumulator r =
//           (filter row ky, M tile mt) holds dW rows (ky, kx, ci).  The grid is R x S CTAs: CTA (r, s) adds accumulator r
//           over the (output pixel, 64 samples) chunks s, s + S, ... and writes its partial sums part[s][r][128][N];
//           chunks that fall outside the image (SAME padding) are read from a zero buffer.  The (pixel, accumulator) ->
//           operand mapping is a host-built table (WgEnt).
//   dense : accumulator = (M tile r of the input features, N tile); the CTA reduces over all samples and stores dW.
// ------------------------------------------------------------------------------------------
constexpr int WG_KB = 64;                        // samples per K chunk
constexpr int WG_PLANE = WG_KB * 16;             // 1024
constexpr int WG_STAGE_A = 2 * 16 * WG_PLANE;    // hi + lo, 16 chunks
constexpr int WG_STAGE_B = 2 * 8 * WG_PLANE;     // hi + lo, up to 8 chunks (N <= 64)
constexpr int WG_STAGE = WG_STAGE_A + WG_STAGE_B;
constexpr int WG_STAGES = 4;
constexpr int WG_THREADS = BP_THREADS;

struct WgEnt {               // conv: one (output pixel, accumulator) pair (8 bytes, copied to shared memory)
  int32_t x_chunk;           // first X feature chunk of the M tile (may be negative at a padded border)
  uint16_t okmask;           // bit c: chunk c of the tile lies inside the image and inside the filter row
  uint16_t valid;            // the filter row exists for this pixel
};

struct WgradArgs {
  BpT x; int x_split; BpT g; const bf16* zeros;
  int mode;                                      // 0 conv, 1 dense
  const WgEnt* tab;                              // conv: [n_opix][R]
  int R;                                         // conv: accumulators (the grid is R x slices)
  int N, B, n_bsub, n_opix;
  int x_chunks, r_tiles, n_ntiles;               // dense: feature chunks of X, M tiles, N tiles
  float* part;                                   // conv: partial sums [slice][R][128][N]
  float* dw; int ldw; int k_rows;                // dense: dW[k_rows][ldw]
};

// stage source of one (K chunk, accumulator) pair
struct WgWalk {
  __device__ __forceinline__ static WgEnt get(const WgradArgs& a, const uint2* tab_sm, int opix, int r, int rt) {
    if (a.mode == 0) {
      const uint2 v = tab_sm[opix * a.R + r];
      return WgEnt{(int32_t)v.x, (uint16_t)(v.y & 0xffffu), (uint16_t)(v.y >> 16)};
    }
    const int c0 = rt * 16, left = a.x_chunks - c0;
    return WgEnt{c0, (uint16_t)(left >= 16 ? 0xffffu : ((1u << left) - 1u)), (uint16_t)1};
  }
};

// N = accumulator columns (16, 32, 48 or 64)
template <int N>
__global__ void __launch_bounds__(WG_THREADS, 1)
bp_wgrad_kernel(const __grid_constant__ WgradArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  __shared__ __align__(8) uint64_t bars[2 * WG_STAGES];
  uint2* tab_sm = reinterpret_cast<uint2*>(smem + WG_STAGES * WG_STAGE);     // conv: [n_opix][R] entries behind the stage ring

  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // see bp_rows_kernel
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[WG_STAGES]);
  if (tid == 0) {
    for (int s = 0; s < WG_STAGES; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, BP_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  const bool conv = a.mode == 0;
  if (conv) {             // static table: fetched under the tail of the preceding kernel
    const uint2* gt = reinterpret_cast<const uint2*>(a.tab);
    for (int i = tid; i < a.n_opix * a.R; i += WG_THREADS) tab_sm[i] = __ldg(gt + i);
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  const uint32_t stage0 = smem_u32(smem);
  // jobs of this CTA: conv = accumulator r over the chunk slice s; dense = tiles (rt, nt), each over all samples
  const int n_slices = conv ? (int)gridDim.x / a.R : 1;
  const int r_conv = conv ? (int)blockIdx.x / n_slices : 0, slice = conv ? (int)blockIdx.x - r_conv * n_slices : 0;
  const int n_tiles = conv ? 1 : a.r_tiles * a.n_ntiles;
  const int n_kc = conv ? a.n_opix * a.n_bsub : a.n_bsub;
  const int tile0 = conv ? 0 : (int)blockIdx.x, tile_step = conv ? 1 : (int)gridDim.x;
  const int kc0 = conv ? slice : 0, kc_step = conv ? n_slices : 1;

  if (warp == BP_P_WARP) {
    // ================= TMA producer: converged warp, one elected lane issues the copies ==============================
    const uint32_t pstride_x = (uint32_t)a.x.pitch * 16u, pstride_g = (uint32_t)a.g.pitch * 16u;
    const char* x_hi = reinterpret_cast<const char*>(a.x.hi);
    const char* x_lo = x_hi + a.x.lo_off * 2;
    const char* g_hi = reinterpret_cast<const char*>(a.g.hi);
    const char* g_lo = g_hi + a.g.lo_off * 2;
    const char* zeros = reinterpret_cast<const char*>(a.zeros);
    const bool x_split = a.x_split != 0;
    constexpr int n_bh = N >> 3;
    int stage = 0; uint32_t phase = 0;
    for (int tile = tile0; tile < n_tiles; tile += tile_step) {
      const int rt = tile / a.n_ntiles, nt = tile - rt * a.n_ntiles;
      for (int kc = kc0; kc < n_kc; kc += kc_step) {
        const int opix = conv ? kc / a.n_bsub : 0, bs = conv ? kc - opix * a.n_bsub : kc;
        const WgEnt e = WgWalk::get(a, tab_sm, opix, r_conv, rt);
        if (!e.valid) continue;
        const int b0 = bs * WG_KB;
        const uint32_t bytes = (uint32_t)((min(WG_KB, a.B - b0) + 15) & ~15) * 16u, row_off = (uint32_t)b0 * 16u;
        const uint32_t g_off = (uint32_t)((conv ? opix : nt) * n_bh) * pstride_g + row_off;
        const long long x_off = (long long)e.x_chunk * (long long)pstride_x + row_off;
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t fb = full0 + 8 * stage;
        if (elect_one()) {
          mbar_expect_tx(fb, bytes * ((x_split ? 32 : 16) + 2 * n_bh));
          const uint32_t sA = stage0 + (uint32_t)stage * WG_STAGE, sB = sA + WG_STAGE_A;
          const uint32_t mask = e.okmask;
#pragma unroll 4
          for (int c = 0; c < 16; c++)
            bulk_g2s(sA + c * WG_PLANE, ((mask >> c) & 1u) ? x_hi + x_off + (long long)((uint32_t)c * pstride_x) : zeros, bytes, fb);
          if (x_split) {
#pragma unroll 4
            for (int c = 0; c < 16; c++)
              bulk_g2s(sA + (16 + c) * WG_PLANE, ((mask >> c) & 1u) ? x_lo + x_off + (long long)((uint32_t)c * pstride_x) : zeros, bytes, fb);
          }
          for (int c = 0; c < n_bh; c++) {
            bulk_g2s(sB + c * WG_PLANE, g_hi + g_off + (uint32_t)c * pstride_g, bytes, fb);
            bulk_g2s(sB + (8 + c) * WG_PLANE, g_lo + g_off + (uint32_t)c * pstride_g, bytes, fb);
          }
        }
        __syncwarp();
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp < BP_P_WARP) {
    // ================= consumers: warpgroup g owns the accumulator rows (features) [64 g, 64 g + 64) =================
    float acc[N / 2];
    const int wg = warp >> 2, q = lane & 3;
    const bool x_split = a.x_split != 0;
    const uint64_t desc = make_desc(0, 128, WG_PLANE);      // MN-major operands: LBO 128 B, SBO = chunk plane
    const uint32_t x_row_add = (uint32_t)(wg * 8 * WG_PLANE) >> 4;
    int stage = 0; uint32_t phase = 0;
    for (int tile = tile0; tile < n_tiles; tile += tile_step) {
      const int rt = tile / a.n_ntiles, nt = tile - rt * a.n_ntiles;
#pragma unroll
      for (int j = 0; j < N / 2; j++) acc[j] = 0.f;
      int held = -1;
      for (int kc = kc0; kc < n_kc; kc += kc_step) {
        const int opix = conv ? kc / a.n_bsub : 0, bs = conv ? kc - opix * a.n_bsub : kc;
        // the skip and the trip count steer the wgmma issue: warp-uniform through a shuffle (see bp_rows_kernel)
        if (!__shfl_sync(0xffffffffu, (int)WgWalk::get(a, tab_sm, opix, r_conv, rt).valid, 0)) continue;
        const int ksteps = __shfl_sync(0xffffffffu, ((min(WG_KB, a.B - bs * WG_KB) + 15) & ~15) >> 4, 0);
        mbar_wait(full0 + 8 * stage, phase);
        const uint32_t sA = stage0 + (uint32_t)stage * WG_STAGE;
        uint32_t x32 = (sA >> 4) + x_row_add, g32 = (sA + WG_STAGE_A) >> 4;
        wgmma_fence();
        if (x_split) {          // outside the issue loops (see bp_rows_kernel)
          for (int j = 0; j < ksteps; j++) {
            const uint64_t xh = desc | x32, gh = desc | g32;
            wgmma<N, 1, 1>(acc, xh, gh);
            wgmma<N, 1, 1>(acc, xh, desc | (g32 + ((8 * WG_PLANE) >> 4)));
            wgmma<N, 1, 1>(acc, desc | (x32 + ((16 * WG_PLANE) >> 4)), gh);
            x32 += 256 >> 4; g32 += 256 >> 4;
          }
        } else {
          for (int j = 0; j < ksteps; j++) {
            const uint64_t xh = desc | x32;
            wgmma<N, 1, 1>(acc, xh, desc | g32);
            wgmma<N, 1, 1>(acc, xh, desc | (g32 + ((8 * WG_PLANE) >> 4)));
            x32 += 256 >> 4; g32 += 256 >> 4;
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (held >= 0 && lane == 0) mbar_arrive(empty0 + 8 * held);
        held = stage;
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs<N / 2>(acc);
      if (held >= 0 && lane == 0) mbar_arrive(empty0 + 8 * held);
      // epilogue: row m = feature within the M tile; an accumulator no chunk reached stays zero
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        float* dst;
        bool ok;
        if (conv) {
          dst = a.part + (((long long)slice * a.R + r_conv) * 128 + m) * N;
          ok = true;
        } else {
          const int k = rt * 128 + m;
          dst = a.dw + (long long)k * a.ldw + nt * N;
          ok = k < a.k_rows;
        }
        if (ok) {
#pragma unroll
          for (int i = 0; i < N / 8; i++)
            *reinterpret_cast<float2*>(dst + 8 * i + 2 * q) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Ordered reduction of per-CTA partial sums into the flat gradient bucket (assignment, not accumulation).
// ------------------------------------------------------------------------------------------
struct RedSeg {
  const float* part; int n_slabs; long long slab;   // slab stride (floats); element idx of the segment inside a slab
  int count;                                         // elements of one slab that this segment covers
  int kind;                                          // 0: conv weight partials [R][128][N]; 1: plain vector (bias)
  int N, C, KW, mts, s2d_k4;                         // conv mapping
  long long dst_off; float alpha;
  float* dst_ptr;                                    // destination base instead of the gradient bucket (kind 1), or NULL
};
// real HWIO row of row k' = ((ty*k4 + tx)*16 + dy*4 + dx)*4 + c of the (k4 x k4, stride 1, 64 channel) conv over a
// space-to-depth plane: ((4ty+dy)*4k4 + 4tx+dx)*4 + c of the (4k4 x 4k4, stride 4, 4 channel) conv
__host__ __device__ inline int s2d_real_row(int m, int k4) {
  int tap = m >> 6, ty = tap / k4, tx = tap - ty * k4;
  int dy = (m >> 4) & 3, dx = (m >> 2) & 3, c = m & 3;
  return (((4 * ty + dy) * 4 * k4 + 4 * tx + dx) << 2) + c;
}
constexpr int RED_MAX = 24;
struct RedSegs { RedSeg s[RED_MAX]; };
// One block = 128 consecutive elements of one segment: warp w sums slabs w, w + 8, ... with float4 loads (512 B per
// warp and slab), then warp 0 adds the eight partial sums in warp order -- a fixed tree, bitwise reproducible.
__global__ void __launch_bounds__(256) grad_reduce_kernel(const __grid_constant__ RedSegs segs, float* __restrict__ grads) {
  pdl_wait(); pdl_trigger();
  __shared__ float4 sh[8][32];
  const RedSeg& s = segs.s[blockIdx.y];
  if ((int)blockIdx.x * 128 >= s.count) return;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = ((int)blockIdx.x * 32 + lane) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < s.count) {
    const bool vec = ((s.count | (int)(s.slab & 3)) & 3) == 0 && (reinterpret_cast<unsigned long long>(s.part) & 15ull) == 0;
    if (vec) {
#pragma unroll 5
      for (int k = w; k < s.n_slabs; k += 8) {
        const float4 x = *reinterpret_cast<const float4*>(s.part + (long long)k * s.slab + i);
        acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
      }
    } else {
      for (int k = w; k < s.n_slabs; k += 8) {
        const float* p = s.part + (long long)k * s.slab + i;
        acc.x += p[0];
        if (i + 1 < s.count) acc.y += p[1];
        if (i + 2 < s.count) acc.z += p[2];
        if (i + 3 < s.count) acc.w += p[3];
      }
    }
  }
  sh[w][lane] = acc;
  __syncthreads();
  if (w != 0 || i >= s.count) return;
  float4 t = sh[0][lane];
#pragma unroll
  for (int q = 1; q < 8; q++) { const float4 x = sh[q][lane]; t.x += x.x; t.y += x.y; t.z += x.z; t.w += x.w; }
  const float v[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const int ie = i + e;
    if (ie >= s.count) break;
    long long dst;
    if (s.kind == 0) {
      const int n = ie % s.N, mm = (ie / s.N) & 127, r = ie / (s.N * 128);
      const int ky = r / s.mts, mt = r - ky * s.mts;
      const int feat = mt * 128 + mm;
      if (feat >= s.KW * s.C) continue;
      int row = ky * s.KW * s.C + feat;
      if (s.s2d_k4) row = s2d_real_row(row, s.s2d_k4);
      dst = s.dst_off + (long long)row * s.N + n;
    } else dst = s.dst_off + ie;
    (s.dst_ptr ? s.dst_ptr : grads)[dst] = s.alpha * v[e];
  }
}

// ------------------------------------------------------------------------------------------
// layout kernels
// ------------------------------------------------------------------------------------------
// fp32 row-major [B][F] -> batch-planar hi/lo planes; rows [B, round16(B)) are zero-filled
__global__ void bp_split_kernel(const float* __restrict__ src, int B, int F, BpT dst) {
  pdl_wait(); pdl_trigger();
  const int b_pad = (B + 15) & ~15;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int chunks = F >> 3;
  if (i >= (long long)chunks * b_pad) return;
  const int c = (int)(i / b_pad), b = (int)(i - (long long)c * b_pad);
  uint4 hi = make_uint4(0, 0, 0, 0), lo = hi;
  if (b < B) {
    const float4* p = reinterpret_cast<const float4*>(src + (long long)b * F + c * 8);
    float4 x = p[0], y = p[1];
    float v[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
    split8(v, hi, lo);
  }
  bf16* o = dst.hi + ((long long)c * dst.pitch + b) * 8;
  *reinterpret_cast<uint4*>(o) = hi;
  *reinterpret_cast<uint4*>(o + dst.lo_off) = lo;
}
// batch-planar planes -> fp32 row-major [B][F]  (x = hi + lo)
__global__ void bp_merge_kernel(BpT src, int B, int F, float* __restrict__ dst) {
  pdl_wait(); pdl_trigger();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int chunks = F >> 3;
  if (i >= (long long)chunks * B) return;
  const int c = (int)(i / B), b = (int)(i - (long long)c * B);
  const bf16* p = src.hi + ((long long)c * src.pitch + b) * 8;
  float h[8], l[8];
  unpack8(*reinterpret_cast<const uint4*>(p), h);
  unpack8(*reinterpret_cast<const uint4*>(p + src.lo_off), l);
  float4* o = reinterpret_cast<float4*>(dst + (long long)b * F + c * 8);
  o[0] = make_float4(h[0] + l[0], h[1] + l[1], h[2] + l[2], h[3] + l[3]);
  o[1] = make_float4(h[4] + l[4], h[5] + l[5], h[6] + l[6], h[7] + l[7]);
}
// column sums of a batch-planar gradient tensor (bias gradient when no data-gradient epilogue produced it):
// db[f % period] += sum_b g[b, f]; one warp per feature chunk
__global__ void bp_colsum_kernel(BpT g, int B, int F, int period, float* __restrict__ db) {
  pdl_wait(); pdl_trigger();
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= (F >> 3)) return;
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int b = lane; b < B; b += 32) {
    const bf16* p = g.hi + ((long long)c * g.pitch + b) * 8;
    float h[8], l[8];
    unpack8(*reinterpret_cast<const uint4*>(p), h);
    unpack8(*reinterpret_cast<const uint4*>(p + g.lo_off), l);
#pragma unroll
    for (int i = 0; i < 8; i++) s[i] += h[i] + l[i];
  }
#pragma unroll
  for (int i = 0; i < 8; i++) {
    float v = s[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) atomicAdd(db + (c * 8 + i) % period, v);
  }
}
// split-K partial sums part[z][b][N] -> act(sum_z + bias): fp32 row-major and/or batch-planar planes.  FIN_ZL lanes share
// one 8-feature piece: lane zl sums slabs zl, zl + FIN_ZL, ... and a fixed xor tree combines them (bitwise reproducible).
constexpr int FIN_ZL = 8;
__global__ void bp_splitk_finish_kernel(const float* __restrict__ part, int n_z, long long part_z, int B, int N,
                                        const float* __restrict__ bias, int act, float* __restrict__ out_f32, BpT out) {
  pdl_wait(); pdl_trigger();
  const int b_pad = (B + 15) & ~15;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long i = t / FIN_ZL;
  const int zl = (int)(t - i * FIN_ZL);
  const int chunks = N >> 3;
  const int c = (int)(i / b_pad), b = (int)(i - (long long)c * b_pad);
  const bool valid = i < (long long)chunks * b_pad && b < B;
  float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (valid) {
    const float* p0 = part + (long long)b * N + c * 8;
#pragma unroll 4
    for (int z = zl; z < n_z; z += FIN_ZL) {
      const float4* p = reinterpret_cast<const float4*>(p0 + (long long)z * part_z);
      float4 x = p[0], y = p[1];
      v[0] += x.x; v[1] += x.y; v[2] += x.z; v[3] += x.w; v[4] += y.x; v[5] += y.y; v[6] += y.z; v[7] += y.w;
    }
  }
#pragma unroll
  for (int o = FIN_ZL / 2; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  if (!valid || zl != 0) return;
#pragma unroll
  for (int k = 0; k < 8; k++) v[k] = act_apply(act, v[k] + bias[c * 8 + k]);
  if (out_f32) {
    float4* o = reinterpret_cast<float4*>(out_f32 + (long long)b * N + c * 8);
    o[0] = make_float4(v[0], v[1], v[2], v[3]);
    o[1] = make_float4(v[4], v[5], v[6], v[7]);
  }
  if (out.hi) {
    uint4 hi, lo;
    split8(v, hi, lo);
    bf16* o = out.hi + ((long long)c * out.pitch + b) * 8;
    *reinterpret_cast<uint4*>(o) = hi;
    *reinterpret_cast<uint4*>(o + out.lo_off) = lo;
  }
}

// Weight blobs: for every tensor-core layer the kernel matrix W[K, N] as batch-planar W^T planes
// blob[((n >> 3) * K + k') * 8 + (n & 7)], k' = space-to-depth row order for a stride-4 first layer.
struct BlobSeg { long long w_off, blob_off; int K, N, s2d_k4; };
// inverse of s2d_real_row: real HWIO row -> row of the space-to-depth ordered blob
__host__ __device__ inline int s2d_blob_row(int k, int k4) {
  const int c = k & 3, pix = k >> 2, x = pix % (4 * k4), y = pix / (4 * k4);
  return (((y >> 2) * k4 + (x >> 2)) << 6) + ((y & 3) << 4) + ((x & 3) << 2) + c;
}
// Blob planes of the parameters at flat index j .. j+cnt-1 (cnt <= 4, same weight row, n % 4 == 0 when cnt == 4):
// used by the optimiser kernel so that the blobs are refreshed by the same pass that updates the parameters.
__device__ __forceinline__ void blob_store1(const BlobSeg* __restrict__ segs, int n_segs, bf16* __restrict__ hi, long long lo_off,
                                            long long j, float p) {
  for (int q = 0; q < n_segs; q++) {
    const long long w0 = segs[q].w_off;
    const int K = segs[q].K, N = segs[q].N;
    if (j < w0 || j >= w0 + (long long)K * N) continue;
    const int rel = (int)(j - w0), k = rel / N, n = rel - k * N;
    const int kp = segs[q].s2d_k4 ? s2d_blob_row(k, segs[q].s2d_k4) : k;
    bf16* o = hi + segs[q].blob_off + ((long long)(n >> 3) * K + kp) * 8 + (n & 7);
    const bf16 h = __float2bfloat16_rn(p);
    o[0] = h; o[lo_off] = __float2bfloat16_rn(p - __bfloat162float(h));
    return;
  }
}
__device__ __forceinline__ void blob_store4(const BlobSeg* __restrict__ segs, int n_segs, bf16* __restrict__ hi, long long lo_off,
                                            long long j, const float p[4]) {
  for (int q = 0; q < n_segs; q++) {
    const long long w0 = segs[q].w_off, w1 = w0 + (long long)segs[q].K * segs[q].N;
    if (j + 3 < w0 || j >= w1) continue;
    const int K = segs[q].K, N = segs[q].N;
    const int rel = (int)(j - w0), k = rel / N, n = rel - k * N;
    if (j >= w0 && j + 3 < w1 && (n & 3) == 0) {          // the common case: four parameters of one weight row
      const int kp = segs[q].s2d_k4 ? s2d_blob_row(k, segs[q].s2d_k4) : k;
      bf16* o = hi + segs[q].blob_off + ((long long)(n >> 3) * K + kp) * 8 + (n & 7);
      uint32_t h0, l0, h1, l1;
      split2(p[0], p[1], h0, l0); split2(p[2], p[3], h1, l1);
      *reinterpret_cast<uint2*>(o) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(o + lo_off) = make_uint2(l0, l1);
    } else {
      for (int i = 0; i < 4; i++) blob_store1(segs, n_segs, hi, lo_off, j + i, p[i]);
    }
    return;
  }
}
__global__ void bp_wprep_kernel(const float* __restrict__ params, const BlobSeg* __restrict__ segs, bf16* __restrict__ hi,
                                long long lo_off) {
  pdl_wait(); pdl_trigger();
  const BlobSeg s = segs[blockIdx.y];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // one (n chunk, k') piece per thread
  const int chunks = s.N >> 3;
  if (i >= (long long)chunks * s.K) return;
  const int c = (int)(i / s.K), kp = (int)(i - (long long)c * s.K);
  const int k = s.s2d_k4 ? s2d_real_row(kp, s.s2d_k4) : kp;
  const float4* p = reinterpret_cast<const float4*>(params + s.w_off + (long long)k * s.N + c * 8);
  float4 x = p[0], y = p[1];
  float v[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
  uint4 h, l;
  split8(v, h, l);
  bf16* o = hi + s.blob_off + ((long long)c * s.K + kp) * 8;
  *reinterpret_cast<uint4*>(o) = h;
  *reinterpret_cast<uint4*>(o + lo_off) = l;
}

// uint8 frames [n][H][W][4] (+ minibatch gather) -> batch-planar space-to-depth plane (exact in bf16, hi only); with
// is_signed every byte is read as int8 (two's complement, -128..127, also exact in bf16):
// the image is embedded at (padT, padL) in a zero canvas of [4*H4][4*W4] pixels, pixel block (Y, X) = 64 features
// (dy, dx, c); a 16-byte output piece = 8 source bytes (2 pixels x 4 channels).
// One block = one image row of 32 samples.  Phase 1 reads that row of every sample with 16-byte loads (contiguous
// 336-byte runs per sample) into shared memory; phase 2 hands every piece to one warp whose lanes are the 32 samples,
// so each store instruction writes 512 contiguous bytes of the plane.
constexpr int DEC_SAMPLES = 32;
constexpr int DEC_THREADS = 256;
__global__ void __launch_bounds__(DEC_THREADS)
bp_decode_s2d_kernel(const uint8_t* __restrict__ obs, const int32_t* __restrict__ idx, int B, int H, int W, int H4, int W4,
                     int padT, int padL, int is_signed, BpT dst) {
  // One block = one image row (canvas row Y, sub-row dy) of DEC_SAMPLES samples: 4*H4 x ceil(B/32) blocks, so that the
  // inference batch (B = 32: one sample group) still spreads over 84 blocks.
  extern __shared__ __align__(16) uint8_t dec_sm[];
  pdl_wait(); pdl_trigger();
  const int Y = blockIdx.x >> 2, dy = blockIdx.x & 3, b0 = blockIdx.y * DEC_SAMPLES;
  const int row_bytes = W * 4, units = row_bytes >> 4;          // 16-byte units per image row
  const int sstride = row_bytes + 8;                            // per-sample stride: +8 B keeps 8-byte lane reads conflict-free
  const int ns = min(DEC_SAMPLES, B - b0);
  const long long img = (long long)H * row_bytes;
  const int y = 4 * Y + dy - padT;
  const bool in_img = y >= 0 && y < H;
  for (int i = threadIdx.x; i < ns * units; i += DEC_THREADS) {
    const int sidx = i / units, ux = i - sidx * units;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (in_img) {
      const long long srow = idx ? idx[b0 + sidx] : b0 + sidx;
      v = *reinterpret_cast<const uint4*>(obs + srow * img + (long long)y * row_bytes + ux * 16);
    }
    uint2* d = reinterpret_cast<uint2*>(dec_sm + sidx * sstride + ux * 16);
    d[0] = make_uint2(v.x, v.y);
    d[1] = make_uint2(v.z, v.w);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half_units = W >> 1;                                // 8-byte units (pixel pairs) per image row
  for (int q = warp; q < W4 * 2; q += DEC_THREADS / 32) {
    const int X = q >> 1, dxh = q & 1;
    const int u8 = 2 * X + dxh - (padL >> 1);                   // pixel pair inside the source row
    uint4 o = make_uint4(0, 0, 0, 0);
    if (lane < ns && u8 >= 0 && u8 < half_units) {
      const uint2 v = *reinterpret_cast<const uint2*>(dec_sm + lane * sstride + u8 * 8);
      auto byte = [is_signed](uint32_t w, int sh) {
        const uint32_t u = (w >> sh) & 0xffu;
        return is_signed ? (float)(int8_t)u : (float)u;
      };
      o.x = pack_bf16(byte(v.x, 0), byte(v.x, 8));
      o.y = pack_bf16(byte(v.x, 16), byte(v.x, 24));
      o.z = pack_bf16(byte(v.y, 0), byte(v.y, 8));
      o.w = pack_bf16(byte(v.y, 16), byte(v.y, 24));
    }
    if (lane < ns)
      *reinterpret_cast<uint4*>(dst.hi + ((long long)((Y * W4 + X) * 8 + dy * 2 + dxh) * dst.pitch + b0 + lane) * 8) = o;
  }
}

}  // namespace bp
}  // namespace xtb
