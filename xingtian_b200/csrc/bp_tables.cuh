// bp_tables.cuh -- the data the host hands the wgmma kernels of bp_gemm.cuh: the batch-planar tensor handle and the
// tables xtb_net_create builds (conv stage walks, weight-gradient walks, weight-blob segments, ordered reductions).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace xtb {
namespace bp {

typedef __nv_bfloat16 bf16;

// batch-planar tensor handle (see bp_gemm.cuh for the layout)
struct BpT {
  bf16* hi;            // hi plane; NULL = absent
  long long lo_off;    // lo plane = hi + lo_off (elements)
  int pitch;           // rows per feature chunk (multiple of 16)
};

// conv forward / data gradient: the K-stage walk of one unit (see bp_rows_kernel)
struct StageEnt {            // one K stage of a conv unit (8 bytes; the tables are copied to shared memory at kernel start)
  uint32_t a_chunk;          // first operand feature chunk of the stage
  uint16_t w_row;            // first weight-blob row of the stage (forward: k row; data gradient: tap * Cin)
  uint16_t nch;              // feature chunks in this stage (even, <= 8)
};
typedef uint32_t UnitEnt;    // first stage index | stage count << 24

struct WgEnt {               // conv: one (output pixel, accumulator) pair (8 bytes, copied to shared memory)
  int32_t x_chunk;           // first X feature chunk of the M tile (may be negative at a padded border)
  uint16_t okmask;           // bit c: chunk c of the tile lies inside the image and inside the filter row
  uint16_t valid;            // the filter row exists for this pixel
};

// ordered reduction of per-CTA partial sums into the flat gradient bucket (see grad_reduce_kernel)
struct RedSeg {
  const float* part; int n_slabs; long long slab;   // slab stride (floats); element idx of the segment inside a slab
  int count;                                         // elements of one slab that this segment covers
  int kind;                                          // 0: conv weight partials [R][128][N]; 1: plain vector (bias)
  int N, C, KW, mts, s2d_k4;                         // conv mapping
  long long dst_off; float alpha;
  float* dst_ptr;                                    // destination base instead of the gradient bucket (kind 1), or NULL
};

// Weight blobs: for every tensor-core layer the kernel matrix W[K, N] as batch-planar W^T planes
// blob[((n >> 3) * K + k') * 8 + (n & 7)], k' = space-to-depth row order for a stride-4 first layer.
struct BlobSeg { long long w_off, blob_off; int K, N, s2d_k4; };

}  // namespace bp
}  // namespace xtb
