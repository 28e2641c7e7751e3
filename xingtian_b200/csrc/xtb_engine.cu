// xtb_engine.cu -- C-ABI implementation (see include/xtb200.h).
#include "../../include/xtb200.h"

#include <cuda_runtime.h>

#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "gemm_f32.cuh"
#include "optim.cuh"
#include "rl_kernels.cuh"
#include "stager.cuh"
#include "bp_gemm.cuh"
#include "comm.cuh"
#include <cstdlib>
#include <type_traits>

using namespace xtb;

// ------------------------------------------------------------------------------------------
// errors / bookkeeping
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};

static int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CUDA_TRY(x)                                                                          \
  do {                                                                                       \
    cudaError_t e_ = (x);                                                                    \
    if (e_ != cudaSuccess)                                                                   \
      return fail(XTB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
  } while (0)
#define LAUNCH_CHECK()                                                                       \
  do {                                                                                       \
    g_launches.fetch_add(1, std::memory_order_relaxed);                                      \
    cudaError_t e_ = cudaPeekAtLastError();                                                  \
    if (e_ != cudaSuccess)                                                                   \
      return fail(XTB_ERR_CUDA, "%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e_)); \
  } while (0)

extern "C" int xtb_version(void) { return XTB_VERSION; }
extern "C" const char* xtb_last_error(void) { return g_err.c_str(); }
extern "C" long long xtb_launch_count(void) { return g_launches.load(); }

static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- data-parallel communicator ---------------------------------------------------------------
static NcclApi g_nccl;
static xtb_comm* g_comm = nullptr;          // installed communicator: gradients are all-reduced inside the training loops
extern "C" int xtb_comm_unique_id(const char* nccl_path, void* id128) {
  if (!id128) return fail(XTB_ERR_ARG, "xtb_comm_unique_id: null pointer");
  if (const char* err = g_nccl.load(nccl_path)) return fail(XTB_ERR_STATE, "cannot load NCCL: %s", err);
  NcclUniqueId id;
  int rc = g_nccl.GetUniqueId(&id);
  if (rc) return fail(XTB_ERR_CUDA, "ncclGetUniqueId: %s", g_nccl.GetErrorString(rc));
  memcpy(id128, &id, sizeof id);
  return XTB_OK;
}
extern "C" int xtb_comm_create(const char* nccl_path, const void* id128, int rank, int world, xtb_comm** out) {
  if (!id128 || !out || world < 1 || rank < 0 || rank >= world) return fail(XTB_ERR_ARG, "xtb_comm_create: bad argument");
  if (const char* err = g_nccl.load(nccl_path)) return fail(XTB_ERR_STATE, "cannot load NCCL: %s", err);
  auto* c = new xtb_comm();
  c->rank = rank; c->world = world;
  NcclUniqueId id;
  memcpy(&id, id128, sizeof id);
  int rc = g_nccl.CommInitRank(&c->comm, world, id, rank);
  if (rc) { delete c; return fail(XTB_ERR_CUDA, "ncclCommInitRank: %s", g_nccl.GetErrorString(rc)); }
  cudaError_t e = cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->join, cudaEventDisableTiming);
  if (e != cudaSuccess) { g_nccl.CommDestroy(c->comm); delete c; return fail(XTB_ERR_CUDA, "xtb_comm_create: %s", cudaGetErrorString(e)); }
  *out = c;
  return XTB_OK;
}
static void drop_graphs_of(const void* obj);
extern "C" void xtb_comm_destroy(xtb_comm* c) {
  if (!c) return;
  if (g_comm == c) g_comm = nullptr;
  // captured training graphs hold NCCL kernels of this communicator: they go first, and nothing may be in flight
  drop_graphs_of(c);
  cudaDeviceSynchronize();
  if (c->comm) g_nccl.CommDestroy(c->comm);
  if (c->side) cudaStreamDestroy(c->side);
  if (c->fork) cudaEventDestroy(c->fork);
  if (c->join) cudaEventDestroy(c->join);
  delete c;
}
extern "C" int xtb_comm_world(const xtb_comm* c) { return c ? c->world : 1; }
// NULL uninstalls.  While installed, the fused training loops scale losses/gradients by 1/(world * B_local), sum the
// gradient bucket over ranks before the optimiser step and stay inside the CUDA graph.
extern "C" int xtb_set_grad_comm(xtb_comm* c) { g_comm = c; return XTB_OK; }
// sum `count` floats in place over the ranks of `c`, on `stream`
extern "C" int xtb_comm_allreduce(xtb_comm* c, float* buf, long long count, void* stream) {
  if (!c || !buf || count < 0) return fail(XTB_ERR_ARG, "xtb_comm_allreduce: bad argument");
  if (count == 0 || c->world == 1) return XTB_OK;
  int rc = g_nccl.AllReduce(buf, buf, (size_t)count, kNcclFloat, kNcclSum, c->comm, S(stream));
  if (rc) return fail(XTB_ERR_CUDA, "ncclAllReduce: %s", g_nccl.GetErrorString(rc));
  return XTB_OK;
}
// Early bucket [off, off+count): forked onto the communicator's side stream at the current point of `stream`, so the
// exchange overlaps whatever is enqueued on `stream` afterwards; comm_join() makes `stream` wait for it.
static int comm_fork_allreduce(xtb_comm* c, float* buf, long long count, cudaStream_t st) {
  CUDA_TRY(cudaEventRecord(c->fork, st));
  CUDA_TRY(cudaStreamWaitEvent(c->side, c->fork, 0));
  int rc = g_nccl.AllReduce(buf, buf, (size_t)count, kNcclFloat, kNcclSum, c->comm, c->side);
  if (rc) return fail(XTB_ERR_CUDA, "ncclAllReduce: %s", g_nccl.GetErrorString(rc));
  CUDA_TRY(cudaEventRecord(c->join, c->side));
  return XTB_OK;
}
static int comm_join(xtb_comm* c, cudaStream_t st) {
  CUDA_TRY(cudaStreamWaitEvent(st, c->join, 0));
  return XTB_OK;
}

// ------------------------------------------------------------------------------------------
// network
// ------------------------------------------------------------------------------------------
static const int kSMs = 132;                    // H100 SXM: persistent kernels size their grids to one wave
static const int kMaxDynSmem = 232448 - 3072;   // 227 KiB per CTA minus the kernels' static shared memory (<= 3 KiB)

struct LayerPlan {
  xtb_layer_desc d;
  ConvGeom g{};          // conv only
  int in_size = 0;       // floats per sample of the source tensor
  int out_size = 0;
  int K = 0, N = 0;      // weight matrix [K,N]
  long long w_off = 0, b_off = 0;
  int src_act = 0;       // activation of the producing layer of the source tensor
  int adv_act = 0;       // dueling: activation of the producing layer of the 1-wide stream (tensor d.k)
  // device tables (conv, fp32 path)
  int* koff = nullptr; int* kyx = nullptr;            // forward / wgrad, indexed by k=(ky,kx,ci)
  int* dkyx = nullptr; int* dco = nullptr; int* wk = nullptr;  // dgrad, indexed by k=(ky,kx,co)
  int Kd = 0;            // KH*KW*Cout
  int sshift = 0;
  bool pad = false;
  // ---- tensor-core (batch-planar) plan; tc = the layer's shapes are covered
  bool tc = false;
  bool s2d = false;      // stride-4 4-channel first layer run as a (k/4 x k/4, stride 1) conv over a space-to-depth plane
  int k4 = 0;
  ConvGeom q{};          // geometry the tensor-core kernels use (space-to-depth view for s2d layers)
  long long blob_off = 0;   // element offset of this layer's weight blob (hi plane)
  bool w_res = false;       // conv: blob resident in shared memory
  int n_fwd = 0, n_dg = 0;  // accumulator columns: forward (Cout / dense N tile), data gradient (Cin / dense K tile)
  int run_chunks = 0, mts = 0, R = 0;   // conv weight gradient: chunks per filter row, M tiles per row, accumulators
  size_t part_off = 0, dbpart_off = 0;  // workspace offsets of the partial-sum areas
  size_t act_part_off = 0;              // act_is_ext layers: act_bwd_kernel's bias partial sums [ACT_BWD_BLOCKS][N]
  // host-built stage walks of the tensor-core kernels (conv layers) and their workspace offsets
  std::vector<bp::StageEnt> fwd_st, dg_st; std::vector<bp::UnitEnt> fwd_un, dg_un; std::vector<bp::WgEnt> wg_tab;
  size_t fwd_st_off = 0, fwd_un_off = 0, dg_st_off = 0, dg_un_off = 0, wg_off = 0;
};

// layer `lp` reads tensor t: through src, or as the second (1-wide) input of a dueling layer
static inline bool reads(const LayerPlan& lp, int t) { return lp.d.src == t || (lp.d.kind == XTB_DUELING && lp.d.k == t); }

// The K-stage walk of every unit of a conv layer (see bp_rows_kernel): forward = per filter row the taps inside the
// image are one contiguous feature run, cut into stages of <= 64 elements; data gradient = one stage per filter tap
// whose output position exists.  Weight gradient: per (output pixel, accumulator) the first X chunk and which of the
// 16 chunks of the M tile are real.  Returns the largest stage count of any unit (a UnitEnt holds at most 255).
static uint32_t build_conv_tables(LayerPlan& lp) {
  const ConvGeom& q = lp.q;
  const int Cout = lp.N;
  uint32_t max_count = 0;
  for (int oy = 0; oy < q.OH; oy++)
    for (int ox = 0; ox < q.OW; ox++) {
      uint32_t first = (uint32_t)lp.fwd_st.size(), count = 0;
      for (int ky = 0; ky < q.KH; ky++) {
        int iy = oy * q.S - q.padT + ky;
        if (iy < 0 || iy >= q.H) continue;
        int x0 = ox * q.S - q.padL, xl = std::max(x0, 0), xh = std::min(x0 + q.KW, q.W);
        if (xh <= xl) continue;
        int chunk = ((iy * q.W + xl) * q.C) >> 3, rem = ((xh - xl) * q.C) >> 3, wrow = (ky * q.KW + (xl - x0)) * q.C;
        while (rem > 0) {
          int nch = std::min(8, rem);
          lp.fwd_st.push_back(bp::StageEnt{(uint32_t)chunk, (uint16_t)wrow, (uint16_t)nch});
          chunk += nch; rem -= nch; wrow += nch * 8; count++;
        }
      }
      lp.fwd_un.push_back(first | (count << 24));
      max_count = std::max(max_count, count);
    }
  for (int iy = 0; iy < q.H; iy++)
    for (int ix = 0; ix < q.W; ix++) {
      uint32_t first = (uint32_t)lp.dg_st.size(), count = 0;
      for (int t = 0; t < q.KH * q.KW; t++) {
        int ky = t / q.KW, kx = t - ky * q.KW;
        int ty = iy + q.padT - ky, tx = ix + q.padL - kx;
        if (ty < 0 || tx < 0) continue;
        int oy = ty / q.S, ox = tx / q.S;
        if (oy * q.S != ty || ox * q.S != tx || oy >= q.OH || ox >= q.OW) continue;
        lp.dg_st.push_back(bp::StageEnt{(uint32_t)(((oy * q.OW + ox) * Cout) >> 3), (uint16_t)(t * q.C), (uint16_t)(Cout >> 3)});
        count++;
      }
      lp.dg_un.push_back(first | (count << 24));
      max_count = std::max(max_count, count);
    }
  for (int oy = 0; oy < q.OH; oy++)
    for (int ox = 0; ox < q.OW; ox++)
      for (int r = 0; r < lp.R; r++) {
        int ky = r / lp.mts, mt = r - ky * lp.mts;
        int iy = oy * q.S - q.padT + ky;
        bp::WgEnt e{0, 0, 0};
        if (iy >= 0 && iy < q.H) {
          int xc0 = ox * q.S - q.padL;
          long long chunk0 = ((long long)(iy * q.W + xc0) * q.C) / 8 + mt * 16;
          e.x_chunk = (int32_t)chunk0;
          for (int c = 0; c < 16; c++) {
            int cj = mt * 16 + c, px = xc0 + (cj * 8) / q.C;
            if (cj < lp.run_chunks && px >= 0 && px < q.W) e.okmask |= (uint16_t)(1u << c);
          }
          e.valid = 1;
        }
        lp.wg_tab.push_back(e);
      }
  return max_count;
}

// Which forms of a tensor's value, and of its gradient, hold the current data: bits of the fp32 row-major buffer and
// of the batch-planar planes.  Tensor 0 is the observation: its planes are the decoded-frame canvas.
enum Form : uint8_t { kNone = 0, kF32 = 1, kPlanes = 2, kBoth = 3 };
struct TensorForms { uint8_t val = kNone, grad = kNone; };

struct xtb_net {
  xtb_net_desc desc;
  int max_batch = 0, pitch = 0;
  std::vector<LayerPlan> L;
  std::vector<int> tsize;       // per tensor floats/sample (0 = obs)
  long long n_params = 0;
  size_t ws_bytes = 0;
  std::vector<size_t> out_off, gout_off;  // byte offsets in workspace per tensor (fp32 row-major)
  std::vector<size_t> obp_off, gbp_off;   // byte offsets of the batch-planar hi planes (lo plane follows at plane_elems)
  std::vector<size_t> z_off;              // byte offset of the retained pre-activation (fp32 row-major), 0 = none
  std::vector<long long> plane_elems;     // elements per plane of tensor t = tsize * pitch
  size_t obs_bp_off = 0; int obs_feats = 0;            // decoded-frame plane (space-to-depth canvas)
  int H4 = 0, W4 = 0;
  size_t blob_off = 0; long long blob_elems = 0;       // weight blobs: hi plane, lo plane follows
  size_t splitk_off = 0, zeros_off = 0, segs_off = 0, heads_part_off = 0;
  std::vector<bp::BlobSeg> blob_segs;
  bool any_tc = false;
  float* params = nullptr; float* grads = nullptr; char* ws = nullptr;
  std::vector<TensorForms> cur;           // per tensor: changed only by wrote() / invalidate() / ensure_f32 / ensure_bp
  std::vector<bp::RedSeg> pending;        // ordered reductions queued by the running backward pass
};

static int same_pad(int size, int k, int s, int* out, int* before) {
  int o = (size + s - 1) / s;
  int total = (o - 1) * s + k - size;
  if (total < 0) total = 0;
  *out = o; *before = total / 2;
  return 0;
}

// ------------------------------------------------------------------------------------------
// tensor-core path (bp_gemm.cuh).  g_tc_mode: 1 = use tensor cores where the shape is covered,
// 0 = fp32 CUDA-core kernels only (XTB_TC=0 in the environment, or xtb_set_tc_mode).
// ------------------------------------------------------------------------------------------
static int g_tc_mode = [] { const char* e = getenv("XTB_TC"); return e ? atoi(e) : 1; }();
extern "C" int xtb_set_tc_mode(int mode) { g_tc_mode = mode; return XTB_OK; }
extern "C" int xtb_get_tc_mode(void) { return g_tc_mode; }

static inline bp::BpT out_bp(const xtb_net* n, int t) { return bp::BpT{(bp::bf16*)(n->ws + n->obp_off[t]), n->plane_elems[t], n->pitch}; }
static inline bp::BpT gout_bp(const xtb_net* n, int t) { return bp::BpT{(bp::bf16*)(n->ws + n->gbp_off[t]), n->plane_elems[t], n->pitch}; }
static inline bp::BpT obs_bp(const xtb_net* n) { return bp::BpT{(bp::bf16*)(n->ws + n->obs_bp_off), 0, n->pitch}; }
static inline bp::BpT no_bp() { return bp::BpT{nullptr, 0, 0}; }
// fp32 row-major value / gradient of tensor t, [max_batch][tsize]
static inline float* out_f32(const xtb_net* n, int t) { return (float*)(n->ws + n->out_off[t]); }
static inline float* gout_f32(const xtb_net* n, int t) { return (float*)(n->ws + n->gout_off[t]); }
// retained pre-activation of tensor t, [max_batch][tsize] fp32; NULL unless its layer's activation keeps it (act_keeps_z)
static inline float* z_buf(const xtb_net* n, int t) { return n->z_off[t] ? (float*)(n->ws + n->z_off[t]) : nullptr; }
// where the GEMM of a layer with an activation past tanh (act_is_ext) writes its pre-activation: the retained buffer, or
// the fp32 output that act_fwd_kernel then overwrites in place
static inline float* pre_buf(const xtb_net* n, int t) { float* z = z_buf(n, t); return z ? z : out_f32(n, t); }

// the forms of tensor t's value (or gradient) that are current
static inline uint8_t forms(const xtb_net* n, int t, bool grad) { return grad ? n->cur[t].grad : n->cur[t].val; }
// the forms f of tensor t's value (or gradient) were just written: every other form is stale
static inline void wrote(xtb_net* n, int t, bool grad, Form f) { (grad ? n->cur[t].grad : n->cur[t].val) = f; }
// nothing of the values / of the gradients of any tensor is current
static void invalidate(xtb_net* n, bool values, bool grads) {
  for (TensorForms& c : n->cur) { if (values) c.val = kNone; if (grads) c.grad = kNone; }
}
static inline const bp::bf16* blob_hi(const xtb_net* n, const LayerPlan& lp) { return (const bp::bf16*)(n->ws + n->blob_off) + lp.blob_off; }
static inline bool use_tc(const LayerPlan& lp) { return g_tc_mode && lp.tc; }

static int pick_tile(int n) { return n % 64 == 0 ? 64 : (n % 32 == 0 ? 32 : (n % 16 == 0 ? 16 : 0)); }

// Dynamic shared memory of the tensor-core launches.  xtb_net_create plans with the same arithmetic as launch_rows /
// launch_wgrad, so a layer it puts on the tensor cores always gets a launch that fits.
// bp_rows_kernel: [resident weight blob][ring of n_stages stages][epilogue banks][conv stage-walk table]
// epi_planes: planes the data-gradient epilogue prefetches (bp::dgrad_epi_planes; 0 for the forward kernels), each
// N / 8 chunks x 128 rows x 16 B per bank.  Two banks let the producer fill one tile's operands while the epilogue of
// the tile before reads the other; when two banks would leave fewer than two ring stages it runs with one.
struct RowsSmem { int wres_bytes, stage_bytes, epi_bank_bytes, epi_banks, tab_bytes, n_stages; };
static RowsSmem rows_smem(bool w_res, int w_res_chunks, int w_pitch, int mode, size_t n_stage_ents, size_t n_units, int N,
                          int epi_planes) {
  RowsSmem r;
  r.wres_bytes = w_res ? (int)align_up((size_t)2 * w_res_chunks * w_pitch * 16, 128) : 0;
  r.stage_bytes = bp::RW_STAGE_A + (w_res ? 0 : bp::RW_STAGE_B);
  r.epi_bank_bytes = epi_planes * (N / 8) * bp::RW_A_PLANE;
  const size_t tab = mode == 2 ? 0 : align_up(n_stage_ents * sizeof(bp::StageEnt) + n_units * sizeof(bp::UnitEnt), 128);
  r.tab_bytes = (int)std::min(tab, (size_t)kMaxDynSmem + 1);
  const int room = kMaxDynSmem - 128 - r.wres_bytes - r.tab_bytes;
  auto stages = [&](int banks) { return std::max(0, std::min(bp::RW_MAX_STAGES, (room - banks * r.epi_bank_bytes) / r.stage_bytes)); };
  r.epi_banks = epi_planes ? bp::RW_EPI_BANKS : 0;
  r.n_stages = stages(r.epi_banks);
  if (r.n_stages < 2 && r.epi_banks > 1) { r.epi_banks = 1; r.n_stages = stages(1); }
  return r;
}
// the activation whose derivative a data-gradient epilogue applies: none for the activations past tanh, whose tensors
// collect the gradient wrt their output until act_backward
static inline int dgrad_act(const LayerPlan& lp) { return act_is_ext(lp.src_act) ? 0 : lp.src_act; }
// shared memory of a conv layer's data-gradient launch; accumulate: into a source tensor with another consumer
static RowsSmem conv_dgrad_smem(const LayerPlan& lp, bool accumulate) {
  return rows_smem(lp.w_res, lp.N / 8, lp.K, 1, lp.dg_st.size(), lp.dg_un.size(), lp.n_dg,
                   bp::dgrad_epi_planes(dgrad_act(lp), accumulate));
}
// bp_wgrad_kernel: [WG_STAGES stages][conv (output pixel, accumulator) table]
static size_t wgrad_smem(int mode, int n_opix, int R) {
  return 128 + bp::WG_STAGES * bp::WG_STAGE + (mode == 0 ? align_up((size_t)n_opix * R * sizeof(bp::WgEnt), 128) : 0);
}
// K slices of a dense forward over `tiles` output tiles: as many as fit in ONE wave of CTAs (rounding up instead left a
// few CTAs with two slices: twice the latency), each a whole number of 64-element stages
static int dense_k_slices(int kchunks, int tiles, int* kc_split) {
  *kc_split = kchunks;
  if (tiles < kSMs && kchunks >= 32) {
    const int want = std::min(kSMs / tiles, kchunks / 8);
    if (want > 1) {
      *kc_split = ((kchunks + want - 1) / want + 7) / 8 * 8;
      return (kchunks + *kc_split - 1) / *kc_split;
    }
  }
  return 1;
}
// A conv layer stays on the tensor cores only if its stage tables fit: the forward and data-gradient launches get at
// least two ring stages beside their table (the data gradient with the epilogue buffers of an accumulating launch, the
// largest it can need), the weight-gradient table fits beside the WG_STAGES stages, and no unit needs more stages than
// a UnitEnt counts.  Otherwise it runs on the fp32 kernels.
static bool conv_tables_fit(const LayerPlan& lp, uint32_t max_unit_stages) {
  const ConvGeom& q = lp.q;
  if (max_unit_stages > 255 || lp.fwd_st.size() >= (1u << 24) || lp.dg_st.size() >= (1u << 24)) return false;
  if (rows_smem(lp.w_res, lp.N / 8, lp.K, 0, lp.fwd_st.size(), lp.fwd_un.size(), lp.n_fwd, 0).n_stages < 2) return false;
  if (conv_dgrad_smem(lp, true).n_stages < 2) return false;
  return wgrad_smem(0, q.OH * q.OW, lp.R) <= (size_t)kMaxDynSmem;
}

extern "C" int xtb_net_create(const xtb_net_desc* desc, int max_batch, xtb_net** out) {
  if (!desc || !out || max_batch <= 0) return fail(XTB_ERR_ARG, "xtb_net_create: null/invalid argument");
  if (desc->n_layers <= 0 || desc->n_layers > XTB_MAX_LAYERS) return fail(XTB_ERR_ARG, "n_layers out of range");
  if (desc->input_u8 < 0 || desc->input_u8 > 2) return fail(XTB_ERR_ARG, "input_u8 %d not in 0..2", desc->input_u8);
  auto* net = new xtb_net();
  net->desc = *desc;
  net->max_batch = max_batch;
  net->pitch = (max_batch + 15) / 16 * 16;
  struct Shape { int h, w, c; };
  std::vector<Shape> shp(desc->n_layers + 1);
  std::vector<int> tact(desc->n_layers + 1, 0);
  shp[0] = {desc->in_h, desc->in_w, desc->in_c};
  net->tsize.resize(desc->n_layers + 1);
  net->tsize[0] = desc->in_h * desc->in_w * desc->in_c;
  long long off = 0;
  for (int i = 0; i < desc->n_layers; i++) {
    LayerPlan lp;
    lp.d = desc->layers[i];
    const auto& d = lp.d;
    if (d.src < 0 || d.src > i) { delete net; return fail(XTB_ERR_ARG, "layer %d: bad src %d", i, d.src); }
    if (d.act < XTB_ACT_NONE || d.act > XTB_ACT_GELU) { delete net; return fail(XTB_ERR_ARG, "layer %d: unknown activation %d", i, d.act); }
    if (d.kind == XTB_LOGSTD) {
      // parameter-only: A floats (pi_logstd), no input, no output tensor
      if (d.src != 0) { delete net; return fail(XTB_ERR_ARG, "layer %d: a logstd layer reads no tensor (src must be 0)", i); }
      if (d.cout < 1 || d.cout > MAX_ADIM) { delete net; return fail(XTB_ERR_ARG, "layer %d: logstd width %d not in [1, %d]", i, d.cout, MAX_ADIM); }
      if (d.act != XTB_ACT_NONE) { delete net; return fail(XTB_ERR_ARG, "layer %d: a logstd layer has no activation", i); }
      lp.K = 1; lp.N = d.cout;
      shp[i + 1] = {1, 1, 0};
      net->tsize[i + 1] = 0;
      lp.w_off = off; off += lp.N;
      lp.b_off = off;
      net->L.push_back(lp);
      continue;
    }
    {   // no layer reads the (0-wide) tensor of a logstd layer
      const bool bad_src = d.src > 0 && desc->layers[d.src - 1].kind == XTB_LOGSTD;
      const bool bad_k = d.kind == XTB_DUELING && d.k > 0 && d.k <= i && desc->layers[d.k - 1].kind == XTB_LOGSTD;
      if (bad_src || bad_k) { delete net; return fail(XTB_ERR_ARG, "layer %d: reads the tensor of a logstd layer", i); }
    }
    if (d.kind == XTB_DUELING) {
      // combine of two earlier layers: src = the A-wide stream, k = the 1-wide stream; no parameters
      if (d.src == 0 || d.k == 0) { delete net; return fail(XTB_ERR_ARG, "layer %d: a dueling layer cannot read the observation", i); }
      if (d.k < 0 || d.k > i) { delete net; return fail(XTB_ERR_ARG, "layer %d: dueling 1-wide input %d is not an earlier layer", i, d.k); }
      if (d.k == d.src) { delete net; return fail(XTB_ERR_ARG, "layer %d: dueling inputs must be two different tensors", i); }
      if (net->tsize[d.k] != 1) { delete net; return fail(XTB_ERR_ARG, "layer %d: dueling input %d is %d wide, not 1", i, d.k, net->tsize[d.k]); }
      if (d.act != XTB_ACT_NONE) { delete net; return fail(XTB_ERR_ARG, "layer %d: a dueling layer has no activation", i); }
      if (act_is_ext(tact[d.src]) || act_is_ext(tact[d.k]))
        { delete net; return fail(XTB_ERR_ARG, "layer %d: a dueling layer reads relu / tanh / linear tensors only", i); }
      lp.in_size = lp.out_size = net->tsize[d.src];
      lp.src_act = tact[d.src]; lp.adv_act = tact[d.k];
      shp[i + 1] = {1, 1, lp.out_size};
      net->tsize[i + 1] = lp.out_size;
      lp.w_off = lp.b_off = off;
      net->L.push_back(lp);
      continue;
    }
    Shape is = shp[d.src];
    lp.in_size = is.h * is.w * is.c;
    lp.src_act = tact[d.src];
    if (d.kind == XTB_CONV && !d.pad_same && d.k == is.h && d.k == is.w) {
      // a VALID conv whose window covers the whole map (ImpalaCnnOpt's 11x11) is a dense layer on the
      // HWC-flattened input with the identical [kh*kw*cin, cout] weight matrix
      lp.d.kind = XTB_DENSE;
    }
    if (lp.d.kind == XTB_CONV) {
      if (d.stride != 1 && d.stride != 2 && d.stride != 4) { delete net; return fail(XTB_ERR_ARG, "layer %d: stride must be 1,2,4", i); }
      ConvGeom& g = lp.g;
      g.H = is.h; g.W = is.w; g.C = is.c; g.KH = g.KW = d.k; g.S = d.stride; g.Cout = d.cout;
      if (d.pad_same) {
        same_pad(g.H, d.k, d.stride, &g.OH, &g.padT);
        same_pad(g.W, d.k, d.stride, &g.OW, &g.padL);
        lp.pad = true;
      } else {
        g.OH = (g.H - d.k) / d.stride + 1; g.OW = (g.W - d.k) / d.stride + 1; g.padT = g.padL = 0;
      }
      if (g.OH <= 0 || g.OW <= 0) { delete net; return fail(XTB_ERR_ARG, "layer %d: empty conv output", i); }
      g.K = d.k * d.k * g.C; g.P = g.OH * g.OW;
      g.mP = fastdiv_magic(g.P); g.mOW = fastdiv_magic(g.OW); g.mHW = fastdiv_magic(g.H * g.W); g.mW = fastdiv_magic(g.W);
      lp.K = g.K; lp.N = d.cout; lp.Kd = d.k * d.k * d.cout;
      lp.sshift = d.stride == 1 ? 0 : (d.stride == 2 ? 1 : 2);
      shp[i + 1] = {g.OH, g.OW, d.cout};
      // tables (fp32 path)
      std::vector<int> koff(g.K), kyx(g.K), dkyx(lp.Kd), dco(lp.Kd), wk(lp.Kd);
      for (int ky = 0; ky < d.k; ky++)
        for (int kx = 0; kx < d.k; kx++) {
          for (int ci = 0; ci < g.C; ci++) {
            int k = (ky * d.k + kx) * g.C + ci;
            koff[k] = (ky * g.W + kx) * g.C + ci;
            kyx[k] = pack_yx(ky, kx);
          }
          for (int co = 0; co < d.cout; co++) {
            int k = (ky * d.k + kx) * d.cout + co;
            dkyx[k] = pack_yx(ky, kx);
            dco[k] = co;
            wk[k] = (ky * d.k + kx) * g.C * d.cout + co;
          }
        }
      auto up = [&](int** dst, const std::vector<int>& v) -> cudaError_t {
        cudaError_t e = cudaMalloc(dst, v.size() * sizeof(int));
        if (e != cudaSuccess) return e;
        return cudaMemcpy(*dst, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice);
      };
      cudaError_t e;
      if ((e = up(&lp.koff, koff)) != cudaSuccess || (e = up(&lp.kyx, kyx)) != cudaSuccess ||
          (e = up(&lp.dkyx, dkyx)) != cudaSuccess || (e = up(&lp.dco, dco)) != cudaSuccess ||
          (e = up(&lp.wk, wk)) != cudaSuccess) {
        delete net;
        return fail(XTB_ERR_CUDA, "table upload failed: %s", cudaGetErrorString(e));
      }
      // ---- tensor-core plan
      lp.q = g;
      const bool cout_ok = d.cout % 16 == 0 && d.cout <= 64;
      if (d.src == 0) {
        // uint8 frames, 4 channels, stride 4: space-to-depth canvas [OH+k/4-1, OW+k/4-1] blocks of 64 features
        if (desc->input_u8 && g.C == 4 && d.stride == 4 && d.k % 4 == 0 && g.padL % 2 == 0 && g.W % 4 == 0 && cout_ok) {
          lp.tc = lp.s2d = true;
          lp.k4 = d.k / 4;
          ConvGeom& q = lp.q;
          q.H = g.OH + lp.k4 - 1; q.W = g.OW + lp.k4 - 1; q.C = 64; q.KH = q.KW = lp.k4; q.S = 1; q.padT = q.padL = 0;
        }
      } else if (g.C % 16 == 0 && g.C <= 64 && cout_ok && d.stride <= d.k) {
        lp.tc = true;
      }
      if (lp.tc) {
        const ConvGeom& q = lp.q;
        lp.n_fwd = d.cout; lp.n_dg = q.C;
        lp.run_chunks = q.KW * q.C / 8;
        lp.mts = (lp.run_chunks + 15) / 16;
        lp.R = q.KH * lp.mts;
        if (lp.R > 32 || lp.R * d.cout > 512) lp.tc = lp.s2d = false;
        lp.w_res = (long long)lp.K * lp.N * 4 <= 96 * 1024;
      }
    } else if (lp.d.kind == XTB_DENSE) {
      lp.K = lp.in_size; lp.N = d.cout;
      shp[i + 1] = {1, 1, d.cout};
      if (d.src != 0 && lp.K % 16 == 0 && pick_tile(lp.N) && pick_tile(lp.K)) {
        lp.tc = true;
        lp.n_fwd = pick_tile(lp.N); lp.n_dg = pick_tile(lp.K);
      }
    } else {
      delete net;
      return fail(XTB_ERR_ARG, "layer %d: unknown kind %d", i, d.kind);
    }
    if (lp.N <= 0) { delete net; return fail(XTB_ERR_ARG, "layer %d: zero outputs", i); }
    tact[i + 1] = d.act;
    lp.out_size = shp[i + 1].h * shp[i + 1].w * shp[i + 1].c;
    net->tsize[i + 1] = lp.out_size;
    lp.w_off = off; off += (long long)lp.K * lp.N;
    lp.b_off = off; off += lp.N;
    net->L.push_back(lp);
  }
  net->n_params = off;
  // a tensor-core layer reads its source in batch-planar form: features must come in chunks of 8 (always true for
  // the shapes accepted above; a dense layer after an uncovered odd-width layer falls back)
  for (auto& lp : net->L) if (lp.tc && lp.d.src != 0 && net->tsize[lp.d.src] % 8) lp.tc = false;
  // the weight-blob refresh (bp_wprep_kernel) reads a tensor-core layer's kernel with 16-byte loads
  for (auto& lp : net->L) if (lp.tc && lp.w_off % 4) lp.tc = lp.s2d = false;
  // stage tables of the tensor-core conv layers; a layer whose tables do not fit in shared memory falls back
  for (auto& lp : net->L) if (lp.tc && lp.d.kind == XTB_CONV) {
    if (conv_tables_fit(lp, build_conv_tables(lp))) continue;
    lp.tc = lp.s2d = false;
    lp.fwd_st.clear(); lp.fwd_un.clear(); lp.dg_st.clear(); lp.dg_un.clear(); lp.wg_tab.clear();
  }
  {   // one observation canvas serves every tensor-core first layer: they must agree on its geometry
    const LayerPlan* f = nullptr; bool agree = true;
    for (auto& lp : net->L) if (lp.s2d) {
      if (!f) f = &lp;
      else if (f->q.H != lp.q.H || f->q.W != lp.q.W || f->g.padT != lp.g.padT || f->g.padL != lp.g.padL) agree = false;
    }
    if (!agree) { for (auto& lp : net->L) if (lp.s2d) lp.tc = lp.s2d = false; f = nullptr; }
    if (f) { net->H4 = f->q.H; net->W4 = f->q.W; }
    net->obs_feats = net->H4 * net->W4 * 64;
  }
  // workspace
  size_t w = 0;
  const int nt = desc->n_layers + 1;
  net->out_off.assign(nt, 0); net->gout_off.assign(nt, 0);
  net->obp_off.assign(nt, 0); net->gbp_off.assign(nt, 0); net->z_off.assign(nt, 0);
  net->plane_elems.assign(nt, 0);
  for (int t = 1; t < nt; t++) {
    size_t bytes = align_up((size_t)max_batch * net->tsize[t] * sizeof(float), 256);
    net->out_off[t] = w; w += bytes;
    net->gout_off[t] = w; w += bytes;
    if (net->tsize[t] % 8 == 0) {
      long long pe = (long long)net->tsize[t] * net->pitch;
      net->plane_elems[t] = pe;
      size_t pbytes = align_up((size_t)pe * 2 * sizeof(uint16_t), 256);   // hi + lo
      net->obp_off[t] = w; w += pbytes;
      net->gbp_off[t] = w; w += pbytes;
    }
    const LayerPlan& lt = net->L[t - 1];
    if ((lt.d.kind == XTB_CONV || lt.d.kind == XTB_DENSE) && act_keeps_z(lt.d.act)) { net->z_off[t] = w; w += bytes; }
  }
  net->obs_bp_off = w; w += align_up((size_t)net->obs_feats * net->pitch * sizeof(uint16_t) + 256, 256);
  long long be = 0;
  for (auto& lp : net->L) if (lp.tc) {
    net->any_tc = true;
    lp.blob_off = be; be += (long long)lp.K * lp.N;
    net->blob_segs.push_back(bp::BlobSeg{lp.w_off, lp.blob_off, lp.K, lp.N, lp.s2d ? lp.k4 : 0});
  }
  net->blob_elems = (long long)align_up((size_t)be, 128);
  net->blob_off = w; w += align_up((size_t)net->blob_elems * 2 * sizeof(uint16_t), 256);
  for (auto& lp : net->L) if (lp.tc) {
    if (lp.d.kind == XTB_CONV) {
      lp.part_off = w; w += align_up((size_t)kSMs * lp.R * 128 * lp.N * sizeof(float), 256);
    }
    lp.dbpart_off = w; w += align_up((size_t)kSMs * 64 * sizeof(float), 256);
  }
  for (auto& lp : net->L) if (lp.tc && lp.d.kind == XTB_CONV) {
    auto place = [&](size_t bytes) { size_t o = w; w += align_up(bytes, 256); return o; };
    lp.fwd_st_off = place(lp.fwd_st.size() * sizeof(bp::StageEnt)); lp.fwd_un_off = place(lp.fwd_un.size() * sizeof(bp::UnitEnt));
    lp.dg_st_off = place(lp.dg_st.size() * sizeof(bp::StageEnt)); lp.dg_un_off = place(lp.dg_un.size() * sizeof(bp::UnitEnt));
    lp.wg_off = place(lp.wg_tab.size() * sizeof(bp::WgEnt));
  }
  // split-K partial sums of a dense forward: n_z slabs of [round16(B)][N] with n_z <= kSMs / (N tiles * batch tiles) + 1
  net->splitk_off = w;
  {
    size_t need = 0;
    for (auto& lp : net->L) if (lp.tc && lp.d.kind == XTB_DENSE) {
      size_t rows = (size_t)(kSMs / (lp.N / lp.n_fwd) + 1) * 128 + net->pitch;
      need = std::max(need, rows * lp.N * sizeof(float));
    }
    w += align_up(need + 256, 256);
  }
  for (auto& lp : net->L)
    if ((lp.d.kind == XTB_CONV || lp.d.kind == XTB_DENSE) && act_is_ext(lp.d.act)) {
      lp.act_part_off = w; w += align_up((size_t)ACT_BWD_BLOCKS * lp.N * sizeof(float), 256);
    }
  net->zeros_off = w; w += 4096;
  // per-block parameter-gradient slabs of the fused PPO heads kernel (K <= 512 hidden units, A <= 8 actions)
  net->heads_part_off = w; w += align_up((size_t)kSMs * (512 * 8 + 3 * 512 + 16) * sizeof(float), 256);
  net->segs_off = w; w += align_up(sizeof(bp::BlobSeg) * XTB_MAX_LAYERS, 256);
  net->ws_bytes = w;
  net->cur.assign(nt, TensorForms{});
  *out = net;
  return XTB_OK;
}

extern "C" void xtb_net_destroy(xtb_net* net) {
  if (!net) return;
  drop_graphs_of(net);
  for (auto& lp : net->L) {
    cudaFree(lp.koff); cudaFree(lp.kyx); cudaFree(lp.dkyx); cudaFree(lp.dco); cudaFree(lp.wk);
  }
  delete net;
}

extern "C" long long xtb_net_param_count(const xtb_net* net) { return net ? net->n_params : -1; }

extern "C" int xtb_net_layer_params(const xtb_net* net, int layer, long long* kernel_off, long long* bias_off,
                                    int* k_rows, int* n_cols) {
  if (!net || layer < 0 || layer >= (int)net->L.size()) return fail(XTB_ERR_ARG, "bad layer index");
  const auto& lp = net->L[layer];
  if (kernel_off) *kernel_off = lp.w_off;
  if (bias_off) *bias_off = lp.b_off;
  if (k_rows) *k_rows = lp.K;
  if (n_cols) *n_cols = lp.N;
  return XTB_OK;
}

extern "C" int xtb_net_layer_plan(const xtb_net* net, int layer, xtb_layer_plan* out) {
  if (!net || !out || layer < 0 || layer >= (int)net->L.size()) return fail(XTB_ERR_ARG, "xtb_net_layer_plan: bad argument");
  const LayerPlan& lp = net->L[layer];
  memset(out, 0, sizeof *out);
  out->kind = lp.d.kind;
  if (!lp.tc) return XTB_OK;
  out->tc = 1; out->s2d = lp.s2d; out->w_res = lp.w_res;
  out->n_fwd = lp.n_fwd; out->n_dg = lp.n_dg; out->R = lp.R;
  if (lp.d.kind == XTB_CONV) {
    out->fwd_stages = rows_smem(lp.w_res, lp.N / 8, lp.K, 0, lp.fwd_st.size(), lp.fwd_un.size(), lp.n_fwd, 0).n_stages;
    out->dg_stages = conv_dgrad_smem(lp, false).n_stages;
    for (bp::UnitEnt u : lp.dg_un) out->dg_empty_units += (u >> 24) == 0;
    out->k_slices = 1;
  } else {
    out->fwd_stages = rows_smem(false, 0, lp.K, 2, 0, 0, lp.n_fwd, 0).n_stages;
    out->dg_stages = rows_smem(false, 0, lp.K, 2, 0, 0, lp.n_dg, bp::dgrad_epi_planes(dgrad_act(lp), 0)).n_stages;
    int kc_split;
    out->k_slices = dense_k_slices(lp.K / 8, (lp.N / lp.n_fwd) * ((net->max_batch + 127) / 128), &kc_split);
  }
  return XTB_OK;
}

extern "C" int xtb_net_tensor_size(const xtb_net* net, int t) {
  if (!net || t < 0 || t >= (int)net->tsize.size()) return -1;
  return net->tsize[t];
}

extern "C" size_t xtb_net_workspace_bytes(const xtb_net* net) { return net ? net->ws_bytes : 0; }

static cudaError_t ensure_kernel_attrs();
extern "C" int xtb_net_sync_weights(xtb_net* net, void* stream);
extern "C" int xtb_net_bind_stream(xtb_net* net, float* params, float* grads, void* workspace, size_t workspace_bytes, void* stream) {
  if (!net || !params || !workspace) return fail(XTB_ERR_ARG, "xtb_net_bind: null pointer");
  if (workspace_bytes < net->ws_bytes) return fail(XTB_ERR_ARG, "workspace too small: %zu < %zu", workspace_bytes, net->ws_bytes);
  bool tc_layers = false;
  for (const auto& lp : net->L) tc_layers |= lp.tc;
  if (tc_layers && (uintptr_t)params % 16) return fail(XTB_ERR_ARG, "xtb_net_bind: parameters must be 16-byte aligned");
  drop_graphs_of(net);                     // captured graphs baked the old buffers in
  net->params = params; net->grads = grads; net->ws = (char*)workspace;
  cudaStream_t st = S(stream);
  { cudaError_t ea = ensure_kernel_attrs(); if (ea != cudaSuccess) return fail(XTB_ERR_CUDA, "kernel attributes: %s", cudaGetErrorString(ea)); }
  // Planes start as zeros: rows beyond the current batch are read (never used) by full-tile operand copies and
  // must be finite; the zero buffer feeds out-of-image chunks of padded weight-gradient operands.
  CUDA_TRY(cudaMemsetAsync(net->ws, 0, net->ws_bytes, st));
  if (!net->blob_segs.empty())
    CUDA_TRY(cudaMemcpyAsync(net->ws + net->segs_off, net->blob_segs.data(), net->blob_segs.size() * sizeof(bp::BlobSeg),
                             cudaMemcpyHostToDevice, st));
  for (const auto& lp : net->L) if (lp.tc && lp.d.kind == XTB_CONV) {
    auto up = [&](size_t off, const void* src, size_t bytes) { return bytes ? cudaMemcpyAsync(net->ws + off, src, bytes, cudaMemcpyHostToDevice, st) : cudaSuccess; };
    CUDA_TRY(up(lp.fwd_st_off, lp.fwd_st.data(), lp.fwd_st.size() * sizeof(bp::StageEnt)));
    CUDA_TRY(up(lp.fwd_un_off, lp.fwd_un.data(), lp.fwd_un.size() * sizeof(bp::UnitEnt)));
    CUDA_TRY(up(lp.dg_st_off, lp.dg_st.data(), lp.dg_st.size() * sizeof(bp::StageEnt)));
    CUDA_TRY(up(lp.dg_un_off, lp.dg_un.data(), lp.dg_un.size() * sizeof(bp::UnitEnt)));
    CUDA_TRY(up(lp.wg_off, lp.wg_tab.data(), lp.wg_tab.size() * sizeof(bp::WgEnt)));
  }
  invalidate(net, true, true);
  int rc = xtb_net_sync_weights(net, stream);
  if (rc) return rc;
  // the segment table came from pageable host memory of this call: do not return before it is on the device
  CUDA_TRY(cudaStreamSynchronize(st));
  return XTB_OK;
}
extern "C" int xtb_net_bind(xtb_net* net, float* params, float* grads, void* workspace, size_t workspace_bytes) {
  return xtb_net_bind_stream(net, params, grads, workspace, workspace_bytes, nullptr);
}

extern "C" float* xtb_net_tensor(xtb_net* net, int t) {
  if (!net || !net->ws || t < 1 || t >= (int)net->tsize.size()) return nullptr;
  return out_f32(net, t);
}
extern "C" float* xtb_net_tensor_grad(xtb_net* net, int t) {
  if (!net || !net->ws || t < 1 || t >= (int)net->tsize.size()) return nullptr;
  return gout_f32(net, t);
}

// ------------------------------------------------------------------------------------------
// fp32 GEMM dispatch
// ------------------------------------------------------------------------------------------
template <int BM, int BN, int TM, int TN, class AL, class BL, class EP>
static void launch_cfg(const AL& al, const BL& bl, const EP& ep, int M, int N, int K, int ksplit, cudaStream_t st) {
  constexpr int BK = 16;
  int kc = (K + ksplit - 1) / ksplit;
  kc = (kc + BK - 1) / BK * BK;
  int ks = (K + kc - 1) / kc;
  dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, ks);
  XLAUNCH((gemm_f32_kernel<BM, BN, BK, TM, TN, AL, BL, EP>), grid, (BM / TM) * (BN / TN), 0, st, al, bl, ep, M, N, K, kc);
}

// split_ok: epilogue is atomic-accumulating so K may be partitioned over gridDim.z
template <class AL, class BL, class EP>
static void launch_gemm(const AL& al, const BL& bl, const EP& ep, int M, int N, int K, bool split_ok, cudaStream_t st) {
  auto ctas = [&](int bm, int bn) { return (long long)((M + bm - 1) / bm) * ((N + bn - 1) / bn); };
  int ksplit = 1;
  if (N <= 32) {
    long long c = ctas(128, 32);
    if (c >= kSMs || split_ok) {
      if (split_ok) { ksplit = (int)((2 * kSMs + c - 1) / c); int mx = (K + 63) / 64; if (ksplit > mx) ksplit = mx; if (ksplit < 1) ksplit = 1; }
      launch_cfg<128, 32, 4, 4>(al, bl, ep, M, N, K, ksplit, st);
      return;
    }
    launch_cfg<32, 32, 2, 2>(al, bl, ep, M, N, K, 1, st);
    return;
  }
  long long c = ctas(64, 64);
  if (c >= kSMs || split_ok) {
    if (split_ok) { ksplit = (int)((2 * kSMs + c - 1) / c); int mx = (K + 63) / 64; if (ksplit > mx) ksplit = mx; if (ksplit < 1) ksplit = 1; }
    launch_cfg<64, 64, 4, 4>(al, bl, ep, M, N, K, ksplit, st);
    return;
  }
  launch_cfg<32, 32, 2, 2>(al, bl, ep, M, N, K, 1, st);
}

// ------------------------------------------------------------------------------------------
// tensor-core launches
// ------------------------------------------------------------------------------------------
// Every instantiation of the kernel families that are chosen at run time, written once: the launches pick from these
// tables and ensure_kernel_attrs opts all of them in to the large shared-memory carve-out.
// The accumulator width is a template parameter of the GEMM kernels (wgmma takes N as an immediate): entry N / 16 - 1.
template <int KIND>
static void (*const kRowsKernels[])(bp::RowsArgs, int, int, int, int) = {
    bp::bp_rows_kernel<KIND, 16>, bp::bp_rows_kernel<KIND, 32>, bp::bp_rows_kernel<KIND, 48>, bp::bp_rows_kernel<KIND, 64>};
static void (*const kWgradKernels[])(bp::WgradArgs) = {bp::bp_wgrad_kernel<16>, bp::bp_wgrad_kernel<32>,
                                                       bp::bp_wgrad_kernel<48>, bp::bp_wgrad_kernel<64>};
template <class F, size_t C>
static F by_width(F const (&tab)[C], int n) { return n > 0 && n % 16 == 0 && n / 16 <= (int)C ? tab[n / 16 - 1] : nullptr; }

// Fused-heads instantiations, in the order they are tried: an entry covers K hidden units with K / 32 <= kpl per lane
// and A <= amax actions
template <class F> struct HeadsEnt { int kpl, amax; F kern; };
template <class LOSS>
static const HeadsEnt<void (*)(PpoHeadsArgs)> kHeadsKernels[] = {
    {2, 8, heads_kernel<LOSS, 2, 8>}, {8, 4, heads_kernel<LOSS, 8, 4>}, {8, 8, heads_kernel<LOSS, 8, 8>},
    {16, 4, heads_kernel<LOSS, 16, 4>}};
template <class DIST>
static const HeadsEnt<decltype(&infer_heads_kernel<DIST, 2, 8>)> kInferHeadsKernels[] = {
    {2, 8, infer_heads_kernel<DIST, 2, 8>}, {8, 4, infer_heads_kernel<DIST, 8, 4>}, {8, 8, infer_heads_kernel<DIST, 8, 8>},
    {16, 8, infer_heads_kernel<DIST, 16, 8>}};
template <class E, size_t C>
static const E* heads_pick(const E (&tab)[C], int K, int A) {
  for (const E& e : tab)
    if (K / 32 <= e.kpl && A <= e.amax) return &e;
  return nullptr;
}
// an instantiation covers the heads (the same for every loss / distribution); infer: infer_heads_kernel
static bool heads_fit(int K, int A, bool infer = false) {
  return K % 32 == 0 && (infer ? heads_pick(kInferHeadsKernels<Categorical>, K, A) != nullptr
                               : heads_pick(kHeadsKernels<PpoLoss>, K, A) != nullptr);
}

// opt-in to the large dynamic shared-memory carve-out, once per process and outside any stream capture
static cudaError_t ensure_kernel_attrs() {
  static bool done = false;
  if (done) return cudaSuccess;
  cudaError_t e = cudaSuccess;
  auto opt_in = [&](const void* k) { if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem); };
  for (auto k : kRowsKernels<0>) opt_in((const void*)k);
  for (auto k : kRowsKernels<1>) opt_in((const void*)k);
  for (auto k : kRowsKernels<2>) opt_in((const void*)k);
  for (auto k : kWgradKernels) opt_in((const void*)k);
  for (const auto& h : kHeadsKernels<PpoLoss>) opt_in((const void*)h.kern);
  for (const auto& h : kHeadsKernels<DuelingTdLoss>) opt_in((const void*)h.kern);
  for (const auto& h : kHeadsKernels<PpoGaussLoss>) opt_in((const void*)h.kern);
  done = e == cudaSuccess;
  return e;
}

template <int KIND>
static cudaError_t launch_rows(bp::RowsArgs& a, cudaStream_t st) {
  const auto kern = by_width(kRowsKernels<KIND>, a.N);
  if (!kern) return cudaErrorInvalidValue;
  { cudaError_t e0 = ensure_kernel_attrs(); if (e0 != cudaSuccess) return e0; }
  const int epi_planes = KIND == 2 ? bp::dgrad_epi_planes(a.src_act, a.accumulate) : 0;
  const RowsSmem m = rows_smem(a.w_res != 0, a.w_res_chunks, a.w_pitch, a.mode, (size_t)a.n_stage_ents, (size_t)a.n_units, a.N,
                               epi_planes);
  if (m.n_stages < 2) return cudaErrorInvalidConfiguration;
  const int smem = 128 + m.wres_bytes + m.n_stages * m.stage_bytes + m.epi_banks * m.epi_bank_bytes + m.tab_bytes;
  const int total = a.n_units * a.n_btiles;
  const int grid = std::min(total, kSMs);
  XLAUNCH(kern, grid, bp::RW_THREADS, smem, st, a, m.n_stages, m.stage_bytes, m.wres_bytes, m.epi_banks);
  return cudaPeekAtLastError();
}

// conv (mode 0): grid = R x slices, one accumulator per CTA
static cudaError_t launch_wgrad(const bp::WgradArgs& a, int grid, cudaStream_t st) {
  const auto kern = by_width(kWgradKernels, a.N);
  if (!kern) return cudaErrorInvalidValue;
  { cudaError_t e0 = ensure_kernel_attrs(); if (e0 != cudaSuccess) return e0; }
  const size_t smem = wgrad_smem(a.mode, a.n_opix, a.R);
  if (smem > (size_t)kMaxDynSmem) return cudaErrorInvalidConfiguration;
  XLAUNCH(kern, grid, bp::WG_THREADS, (int)smem, st, a);
  return cudaPeekAtLastError();
}

// Queue the ordered reduction of n_slabs per-CTA slabs (stride `slab` floats, `count` of them each) into the gradient
// bucket at dst_off, or at dst_ptr; flush_reductions runs the queue in one launch.  conv: the slabs are that conv
// layer's weight-gradient accumulators [R][128][N], mapped back to its weight rows.
static void queue_reduction(xtb_net* net, const float* part, int n_slabs, long long slab, int count, long long dst_off,
                            float* dst_ptr = nullptr, const LayerPlan* conv = nullptr) {
  bp::RedSeg r;
  memset(&r, 0, sizeof r);
  r.part = part; r.n_slabs = n_slabs; r.slab = slab; r.count = count; r.kind = conv ? 0 : 1;
  r.dst_off = dst_off; r.dst_ptr = dst_ptr; r.alpha = 1.f;
  if (conv) {
    r.N = conv->N; r.C = conv->q.C; r.KW = conv->q.KW; r.mts = conv->mts; r.s2d_k4 = conv->s2d ? conv->k4 : 0;
    r.alpha = conv->d.src == 0 ? net->desc.scale : 1.f;
  }
  net->pending.push_back(r);
}

// forward of a tensor-core layer.  want_f32: also store the fp32 row-major copy; want_bp: store the planes
static cudaError_t tc_forward(xtb_net* net, int i, int B, bool want_f32, bool want_bp, cudaStream_t st, long long* launches) {
  const LayerPlan& lp = net->L[i];
  const int t = i + 1;
  bp::RowsArgs a;
  memset(&a, 0, sizeof a);
  a.a = lp.d.src == 0 ? obs_bp(net) : out_bp(net, lp.d.src);
  a.a_split = lp.d.src != 0;
  a.w_hi = blob_hi(net, lp); a.w_lo = a.w_hi + net->blob_elems; a.w_pitch = lp.K;
  a.B = B; a.n_btiles = (B + 127) / 128; a.N = lp.n_fwd;
  const bool ext = act_is_ext(lp.d.act);      // linear into fp32; act_fwd_kernel follows (op_forward)
  a.out = want_bp && !ext ? out_bp(net, t) : no_bp();
  a.out_f32 = ext ? pre_buf(net, t) : (want_f32 ? out_f32(net, t) : nullptr);
  a.ld_f32 = net->tsize[t];
  a.bias = net->params + lp.b_off;
  a.alpha = lp.d.src == 0 ? net->desc.scale : 1.f;
  a.act = ext ? 0 : lp.d.act;
  *launches = 1;
  if (lp.d.kind == XTB_CONV) {
    a.mode = 0;
    a.stages = (const bp::StageEnt*)(net->ws + lp.fwd_st_off); a.units = (const bp::UnitEnt*)(net->ws + lp.fwd_un_off);
    a.n_stage_ents = (int)lp.fwd_st.size();
    a.w_res = lp.w_res; a.w_res_chunks = lp.N / 8;
    a.n_units = lp.q.OH * lp.q.OW;
    return launch_rows<0>(a, st);
  }
  a.mode = 2;
  a.kchunks = lp.K / 8; a.n_ntiles = lp.N / lp.n_fwd;
  const int nz = dense_k_slices(a.kchunks, a.n_ntiles * a.n_btiles, &a.kc_split);
  a.n_units = a.n_ntiles * nz;
  if (nz == 1) return launch_rows<0>(a, st);
  a.part = (float*)(net->ws + net->splitk_off);
  const int b_pad = (B + 15) & ~15;
  a.part_z = (long long)b_pad * lp.N; a.ld_part = lp.N;
  cudaError_t e = launch_rows<1>(a, st);
  if (e != cudaSuccess) return e;
  long long pieces = (long long)(lp.N / 8) * b_pad * bp::FIN_ZL;
  XLAUNCH(bp::bp_splitk_finish_kernel, (unsigned)((pieces + 127) / 128), 128, 0, st, (const float*)a.part, nz, a.part_z, B, lp.N,
          a.bias, a.act, a.out_f32, a.out);
  *launches = 2;
  return cudaPeekAtLastError();
}

// data gradient of tensor-core layer i into the planes of its source tensor
static cudaError_t tc_dgrad(xtb_net* net, int i, int B, int accumulate, float* db_part, cudaStream_t st) {
  const LayerPlan& lp = net->L[i];
  const int t = i + 1, s = lp.d.src;
  bp::RowsArgs a;
  memset(&a, 0, sizeof a);
  a.a = gout_bp(net, t); a.a_split = 1;
  a.w_hi = blob_hi(net, lp); a.w_lo = a.w_hi + net->blob_elems; a.w_pitch = lp.K;
  a.B = B; a.n_btiles = (B + 127) / 128; a.N = lp.n_dg;
  a.out = gout_bp(net, s); a.src = out_bp(net, s); a.src_act = dgrad_act(lp); a.accumulate = accumulate; a.db_part = db_part;
  if (lp.d.kind == XTB_CONV) {
    a.mode = 1;
    a.stages = (const bp::StageEnt*)(net->ws + lp.dg_st_off); a.units = (const bp::UnitEnt*)(net->ws + lp.dg_un_off);
    a.n_stage_ents = (int)lp.dg_st.size();
    a.w_res = lp.w_res; a.w_res_chunks = lp.N / 8;
    a.n_units = lp.q.H * lp.q.W;
  } else {
    a.mode = 2;
    a.kchunks = lp.N / 8; a.kc_split = a.kchunks; a.n_ntiles = lp.K / lp.n_dg;
    a.n_units = a.n_ntiles;
  }
  return launch_rows<2>(a, st);
}

// weight gradient of tensor-core layer i; conv layers queue their ordered reduction
static cudaError_t tc_wgrad(xtb_net* net, int i, int B, cudaStream_t st) {
  LayerPlan& lp = net->L[i];
  const int t = i + 1;
  bp::WgradArgs a;
  memset(&a, 0, sizeof a);
  a.x = lp.d.src == 0 ? obs_bp(net) : out_bp(net, lp.d.src);
  a.x_split = lp.d.src != 0;
  a.g = gout_bp(net, t);
  a.zeros = (const bp::bf16*)(net->ws + net->zeros_off);
  a.B = B; a.n_bsub = (B + bp::WG_KB - 1) / bp::WG_KB;
  if (lp.d.kind == XTB_CONV) {
    const ConvGeom& q = lp.q;
    a.mode = 0;
    a.tab = (const bp::WgEnt*)(net->ws + lp.wg_off);
    a.R = lp.R; a.N = lp.N; a.n_opix = q.OH * q.OW; a.n_ntiles = 1;
    a.part = (float*)(net->ws + lp.part_off);
    // one wave: every accumulator gets the same number of CTAs, each adding a slice of the (pixel, sample chunk) list
    const int slices = std::max(1, std::min(kSMs / lp.R, a.n_opix * a.n_bsub));
    queue_reduction(net, a.part, slices, (long long)lp.R * 128 * lp.N, lp.R * 128 * lp.N, lp.w_off, nullptr, &lp);
    return launch_wgrad(a, lp.R * slices, st);
  }
  a.mode = 1;
  a.N = std::min(lp.n_fwd, 64);
  a.x_chunks = lp.K / 8; a.r_tiles = (lp.K + 127) / 128; a.n_ntiles = lp.N / a.N; a.n_opix = 1; a.R = 1;
  a.dw = net->grads + lp.w_off; a.ldw = lp.N; a.k_rows = lp.K;
  return launch_wgrad(a, std::min(kSMs, a.r_tiles * a.n_ntiles), st);
}

// keep the weight blobs of the bound parameters current (after an optimiser step / set_weights)
extern "C" int xtb_net_sync_weights(xtb_net* net, void* stream) {
  if (!net || !net->ws || !net->params) return fail(XTB_ERR_STATE, "xtb_net_sync_weights: net not bound");
  if (net->blob_segs.empty()) return XTB_OK;
  long long mx = 0;
  for (const auto& s : net->blob_segs) mx = std::max(mx, (long long)(s.N / 8) * s.K);
  dim3 grid((unsigned)((mx + 127) / 128), (unsigned)net->blob_segs.size());
  XLAUNCH(bp::bp_wprep_kernel, grid, 128, 0, S(stream), (const float*)net->params, (const bp::BlobSeg*)(net->ws + net->segs_off),
          (bp::bf16*)(net->ws + net->blob_off), net->blob_elems);
  LAUNCH_CHECK();
  return XTB_OK;
}


// ---- representation changes ------------------------------------------------------------------
static int ensure_bp(xtb_net* net, int t, int B, bool grad, cudaStream_t st) {
  const uint8_t f = forms(net, t, grad);
  if (f & kPlanes) return XTB_OK;
  if (!(f & kF32)) return fail(XTB_ERR_STATE, "tensor %d has no current %s", t, grad ? "gradient" : "value");
  const float* src = grad ? gout_f32(net, t) : out_f32(net, t);
  const int F = net->tsize[t], b_pad = (B + 15) & ~15;
  long long pieces = (long long)(F / 8) * b_pad;
  XLAUNCH(bp::bp_split_kernel, (unsigned)((pieces + 127) / 128), 128, 0, st, src, B, F, grad ? gout_bp(net, t) : out_bp(net, t));
  LAUNCH_CHECK();
  wrote(net, t, grad, kBoth);
  return XTB_OK;
}
static int ensure_f32(xtb_net* net, int t, int B, bool grad, cudaStream_t st) {
  const uint8_t f = forms(net, t, grad);
  if (f & kF32) return XTB_OK;
  if (!(f & kPlanes)) return fail(XTB_ERR_STATE, "tensor %d has no current %s", t, grad ? "gradient" : "value");
  float* dst = grad ? gout_f32(net, t) : out_f32(net, t);
  const int F = net->tsize[t];
  long long pieces = (long long)(F / 8) * B;
  XLAUNCH(bp::bp_merge_kernel, (unsigned)((pieces + 127) / 128), 128, 0, st, grad ? gout_bp(net, t) : out_bp(net, t), B, F, dst);
  LAUNCH_CHECK();
  wrote(net, t, grad, kBoth);
  return XTB_OK;
}

// Self-test of the three kernel forms on plain matrices (see tests/test_gpu_tc.py):
//   mode 0: C[M,N] = A[M,K]   * B[K,N]      forward   (rows kernel, weights MN-major; ksplit > 1: split-K partials)
//   mode 1: C[M,N] = A[M,K]   * Bt[N,K]^T   data grad (rows kernel, weights K-major)
//   mode 2: C[M,N] = At[K,M]^T * B[K,N]     weight grad (samples = K are the reduction axis)
extern "C" int xtb_tc_gemm_test(int mode, const float* a, const float* b, float* c, int M, int N, int K, int ksplit,
                                void* stream) {
  if (!a || !b || !c || M <= 0 || N <= 0 || K <= 0) return fail(XTB_ERR_ARG, "xtb_tc_gemm_test: bad argument");
  if (N % 16 || K % 16 || (mode == 2 && M % 16)) return fail(XTB_ERR_ARG, "xtb_tc_gemm_test: N, K (and M for mode 2) must be multiples of 16");
  cudaStream_t st = S(stream);
  // rows (samples): mode 0/1 -> M rows of A; mode 2 -> K rows of At and B
  const int rows = mode == 2 ? K : M;
  const int pitch = (rows + 15) / 16 * 16;
  const int fa = mode == 2 ? M : K;                 // features of the "activation" operand
  const int fb = N;                                  // mode 2: features of B
  const int nt = pick_tile(N);
  if (!nt) return fail(XTB_ERR_ARG, "N must be a multiple of 16");
  bp::bf16 *pa = nullptr, *pw = nullptr, *pc = nullptr; float* part = nullptr; float* bias = nullptr;
  const long long ea = (long long)fa * pitch;
  const long long ew = mode == 2 ? (long long)fb * pitch : (mode == 1 ? (long long)K * ((N + 15) / 16 * 16) : (long long)N * K);   // weight blob / second activation
  const long long ec = (long long)N * pitch;
  CUDA_TRY(cudaMalloc(&pa, 2 * ea * sizeof(bp::bf16)));
  CUDA_TRY(cudaMalloc(&pw, 2 * ew * sizeof(bp::bf16) + 256));
  CUDA_TRY(cudaMalloc(&pc, 2 * ec * sizeof(bp::bf16) + 4096));
  CUDA_TRY(cudaMalloc(&bias, (size_t)std::max(N, 64) * sizeof(float)));
  CUDA_TRY(cudaMemsetAsync(pa, 0, 2 * ea * sizeof(bp::bf16), st));
  CUDA_TRY(cudaMemsetAsync(pw, 0, 2 * ew * sizeof(bp::bf16) + 256, st));
  CUDA_TRY(cudaMemsetAsync(pc, 0, 2 * ec * sizeof(bp::bf16) + 4096, st));
  CUDA_TRY(cudaMemsetAsync(bias, 0, (size_t)std::max(N, 64) * sizeof(float), st));
  bp::BpT ta{pa, ea, pitch}, tw{pw, ew, mode == 2 ? pitch : K}, tcp{pc, ec, pitch};
  auto split = [&](const float* src, int B_, int F_, bp::BpT dst) {
    long long pieces = (long long)(F_ / 8) * ((B_ + 15) & ~15);
    XLAUNCH(bp::bp_split_kernel, (unsigned)((pieces + 127) / 128), 128, 0, st, src, B_, F_, dst);
  };
  cudaError_t e = cudaSuccess;
  if (mode == 0 || mode == 1) {
    split(a, M, K, ta);
    // weight blob = batch-planar W^T with rows k: mode 0: b = W[K][N] -> rows K, features N.  mode 1: b = Bt[N][K]: the
    // kernel computes D[m, n] = sum_k A[m,k] Bt[n,k] with "W"[n][k] = Bt: rows = n (output), features = k (reduction)
    if (mode == 0) { tw.pitch = K; split(b, K, N, tw); }
    else { tw.pitch = (N + 15) / 16 * 16; split(b, N, K, tw); }
    bp::RowsArgs r;
    memset(&r, 0, sizeof r);
    r.a = ta; r.a_split = 1; r.w_hi = pw; r.w_lo = pw + ew; r.w_pitch = tw.pitch;
    r.mode = 2; r.B = M; r.n_btiles = (M + 127) / 128; r.N = nt; r.n_ntiles = N / nt;
    r.kchunks = K / 8; r.kc_split = r.kchunks;
    r.bias = bias; r.alpha = 1.f; r.act = 0;
    if (mode == 0) {
      int nz = 1;
      if (ksplit > 1) { r.kc_split = ((r.kchunks + ksplit - 1) / ksplit + 7) / 8 * 8; nz = (r.kchunks + r.kc_split - 1) / r.kc_split; }
      r.n_units = r.n_ntiles * nz;
      if (nz > 1) {
        CUDA_TRY(cudaMalloc(&part, (size_t)nz * M * N * sizeof(float)));
        r.part = part; r.part_z = (long long)M * N; r.ld_part = N;
        e = launch_rows<1>(r, st);
        long long pieces = (long long)(N / 8) * ((M + 15) & ~15) * bp::FIN_ZL;
        XLAUNCH(bp::bp_splitk_finish_kernel, (unsigned)((pieces + 127) / 128), 128, 0, st, (const float*)part, nz, r.part_z, M, N,
                (const float*)bias, 0, c, no_bp());
      } else {
        r.out_f32 = c; r.ld_f32 = N;
        e = launch_rows<0>(r, st);
      }
    } else {
      r.n_units = r.n_ntiles;
      r.out = tcp; r.src = tcp; r.src_act = 0;
      e = launch_rows<2>(r, st);
      long long pieces = (long long)(N / 8) * M;
      XLAUNCH(bp::bp_merge_kernel, (unsigned)((pieces + 127) / 128), 128, 0, st, tcp, M, N, c);
    }
  } else {
    split(a, K, M, ta);
    split(b, K, N, tw);
    bp::WgradArgs w;
    memset(&w, 0, sizeof w);
    w.x = ta; w.x_split = 1; w.g = tw; w.zeros = pc;
    w.mode = 1; w.N = nt; w.B = K; w.n_bsub = (K + bp::WG_KB - 1) / bp::WG_KB; w.n_opix = 1; w.R = 1;
    w.x_chunks = M / 8; w.r_tiles = (M + 127) / 128; w.n_ntiles = N / nt;
    w.dw = c; w.ldw = N; w.k_rows = M;
    e = launch_wgrad(w, std::min(kSMs, w.r_tiles * w.n_ntiles), st);
  }
  g_launches.fetch_add(4, std::memory_order_relaxed);
  cudaError_t e2 = cudaStreamSynchronize(st);
  cudaFree(pa); cudaFree(pw); cudaFree(pc); cudaFree(bias); cudaFree(part);
  if (e != cudaSuccess) return fail(XTB_ERR_CUDA, "tc gemm launch: %s", cudaGetErrorString(e));
  if (e2 != cudaSuccess) return fail(XTB_ERR_CUDA, "tc gemm run: %s", cudaGetErrorString(e2));
  return XTB_OK;
}

// ------------------------------------------------------------------------------------------
// fp32 CUDA-core layer ops
// ------------------------------------------------------------------------------------------
template <typename T>
static void conv_fwd(const LayerPlan& lp, const T* x, const int32_t* idx, const float* w, const float* b,
                     float alpha, float* out, int B, cudaStream_t st) {
  int M = B * lp.g.P;
  BRowMajor bl{w, lp.N};
  EpiBiasAct ep{out, b, alpha, act_is_ext(lp.d.act) ? 0 : lp.d.act, lp.N, nullptr, 0};
  if (lp.pad) { AIm2col<T, true> al{x, idx, lp.g, lp.koff, lp.kyx}; launch_gemm(al, bl, ep, M, lp.N, lp.K, false, st); }
  else { AIm2col<T, false> al{x, idx, lp.g, lp.koff, lp.kyx}; launch_gemm(al, bl, ep, M, lp.N, lp.K, false, st); }
}
template <typename T>
static void dense_fwd(const LayerPlan& lp, const T* x, const int32_t* idx, const float* w, const float* b,
                      float alpha, float* out, int B, cudaStream_t st) {
  ADense<T> al{x, idx, lp.K};
  BRowMajor bl{w, lp.N};
  EpiBiasAct ep{out, b, alpha, act_is_ext(lp.d.act) ? 0 : lp.d.act, lp.N, nullptr, 0};
  launch_gemm(al, bl, ep, B, lp.N, lp.K, false, st);
}
template <typename T>
static void conv_wgrad(const LayerPlan& lp, const T* x, const int32_t* idx, const float* dy, float alpha,
                       float* dw, int B, cudaStream_t st, bool bias_row = true) {
  int Mr = B * lp.g.P;
  BRowMajor bl{dy, lp.N};
  EpiAtomic ep{dw, alpha, lp.N};
  // rows 0..K-1 scaled by alpha (input decode scale); the bias row (K) must not be scaled:
  // it rides in the same GEMM only when alpha == 1, else colsum_kernel computes it.
  int rows = lp.K + ((alpha == 1.f && bias_row) ? 1 : 0);
  if (lp.pad) { AIm2colT<T, true> al{x, idx, lp.g, lp.koff, lp.kyx, Mr}; launch_gemm(al, bl, ep, rows, lp.N, Mr, true, st); }
  else { AIm2colT<T, false> al{x, idx, lp.g, lp.koff, lp.kyx, Mr}; launch_gemm(al, bl, ep, rows, lp.N, Mr, true, st); }
}
template <typename T>
static void dense_wgrad(const LayerPlan& lp, const T* x, const int32_t* idx, const float* dy, float alpha,
                        float* dw, int B, cudaStream_t st, bool bias_row = true) {
  ADenseT<T> al{x, idx, lp.K, lp.K};
  BRowMajor bl{dy, lp.N};
  EpiAtomic ep{dw, alpha, lp.N};
  launch_gemm(al, bl, ep, lp.K + ((alpha == 1.f && bias_row) ? 1 : 0), lp.N, B, true, st);
}

// bias gradient: db[n] = sum_m dy[m,n]
__global__ void colsum_kernel(const float* __restrict__ dy, int M, int N, float* __restrict__ db) {
  pdl_wait(); pdl_trigger();
  int n = blockIdx.x * 32 + (threadIdx.x & 31);
  int r0 = blockIdx.y * 1024 + (threadIdx.x >> 5);
  float s = 0.f;
  if (n < N)
    for (int m = r0; m < min(M, (int)(blockIdx.y + 1) * 1024); m += 8) s += dy[(long long)m * N + n];
  __shared__ float red[8][33];
  red[threadIdx.x >> 5][threadIdx.x & 31] = s;
  __syncthreads();
  if (threadIdx.x < 32 && n < N) {
    float t = 0.f;
    for (int i = 0; i < 8; i++) t += red[i][threadIdx.x];
    atomicAdd(db + n, t);
  }
}

// ------------------------------------------------------------------------------------------
// per-layer operations (tensor-core kernel when the shape is covered, fp32 kernel otherwise)
// ------------------------------------------------------------------------------------------
// the activation past tanh of tensor t's layer, after its GEMM wrote the pre-activation to pre_buf: fp32 output
static int act_forward(xtb_net* net, int t, int B, cudaStream_t st) {
  const long long n = (long long)B * net->tsize[t];
  const unsigned blocks = (unsigned)std::min<long long>((n + 255) / 256, 8LL * kSMs);
  XLAUNCH(act_fwd_kernel, blocks, 256, 0, st, (const float*)pre_buf(net, t), n, net->L[t - 1].d.act, out_f32(net, t));
  LAUNCH_CHECK();
  wrote(net, t, false, kF32);
  return XTB_OK;
}
// ... and in the backward pass: the gradient wrt its output, summed over its consumers, becomes the gradient wrt its
// pre-activation (act' from the retained pre-activation, or from the output); the layer's bias gradient is queued for
// the ordered reduction
static int act_backward(xtb_net* net, int t, int B, cudaStream_t st) {
  int rc = ensure_f32(net, t, B, true, st);
  if (rc) return rc;
  const LayerPlan& lp = net->L[t - 1];
  const float* u = z_buf(net, t) ? z_buf(net, t) : out_f32(net, t);
  float* part = (float*)(net->ws + lp.act_part_off);
  XLAUNCH(act_bwd_kernel, ACT_BWD_BLOCKS, ACT_BWD_THREADS, 0, st, gout_f32(net, t), u,
          (int)((long long)B * net->tsize[t] / lp.N), lp.N, lp.d.act, part);
  LAUNCH_CHECK();
  queue_reduction(net, part, ACT_BWD_BLOCKS, lp.N, lp.N, lp.b_off);
  wrote(net, t, true, kF32);
  return XTB_OK;
}

// uint8 frame decode (+ minibatch gather) into the space-to-depth observation canvas
static int op_decode(xtb_net* net, const void* obs, const int32_t* idx, int B, cudaStream_t st) {
  if (forms(net, 0, false) & kPlanes) return XTB_OK;
  const LayerPlan* first = nullptr;
  for (const auto& lp : net->L) if (lp.s2d && use_tc(lp)) { first = &lp; break; }
  if (!first) return XTB_OK;
  dim3 grid(4 * net->H4, (B + bp::DEC_SAMPLES - 1) / bp::DEC_SAMPLES);
  const int smem = bp::DEC_SAMPLES * (net->desc.in_w * 4 + 8);
  XLAUNCH(bp::bp_decode_s2d_kernel, grid, bp::DEC_THREADS, smem, st, (const uint8_t*)obs, idx, B, net->desc.in_h, net->desc.in_w, net->H4,
          net->W4, first->g.padT, first->g.padL, net->desc.input_u8 == 2 ? 1 : 0, obs_bp(net));
  LAUNCH_CHECK();
  wrote(net, 0, false, kPlanes);
  return XTB_OK;
}

// f(x) with the observation as the element type its loaders read: int8 (input_u8 == 2), uint8 (1) or float (0)
template <class F>
static void with_obs_type(const xtb_net* net, const void* obs, F&& f) {
  if (net->desc.input_u8 == 2) f((const int8_t*)obs);
  else if (net->desc.input_u8) f((const uint8_t*)obs);
  else f((const float*)obs);
}

// forward of layer i; tc_allowed = parameters are the bound ones (their blobs are current)
static int op_forward(xtb_net* net, int i, const float* P, bool tc_allowed, const void* obs, const int32_t* idx, int B,
                      bool want_f32, cudaStream_t st) {
  const LayerPlan& lp = net->L[i];
  const int t = i + 1;
  float* out = out_f32(net, t);
  const bool ext = act_is_ext(lp.d.act);
  float* pre = ext ? pre_buf(net, t) : out;      // the fp32 kernels write the activation, or the pre-activation (ext)
  const float* w = P + lp.w_off;
  const float* b = P + lp.b_off;
  if (lp.d.kind == XTB_LOGSTD) return XTB_OK;   // parameter-only: no output tensor
  if (lp.d.kind == XTB_DUELING) {
    int rc = ensure_f32(net, lp.d.src, B, false, st);
    if (!rc) rc = ensure_f32(net, lp.d.k, B, false, st);
    if (rc) return rc;
    XLAUNCH(dueling_fwd_kernel, (B + 7) / 8, 256, 0, st, (const float*)out_f32(net, lp.d.src), (const float*)out_f32(net, lp.d.k), B,
            lp.out_size, out);
    LAUNCH_CHECK();
    wrote(net, t, false, kF32);
    return XTB_OK;
  }
  if (tc_allowed && use_tc(lp)) {
    int rc = lp.d.src == 0 ? op_decode(net, obs, idx, B, st) : ensure_bp(net, lp.d.src, B, false, st);
    if (rc) return rc;
    long long nl = 0;
    cudaError_t te = tc_forward(net, i, B, want_f32, true, st, &nl);
    if (te != cudaSuccess) return fail(XTB_ERR_CUDA, "tensor-core forward launch (layer %d): %s", i, cudaGetErrorString(te));
    g_launches.fetch_add(nl, std::memory_order_relaxed);
    if (ext) return act_forward(net, t, B, st);
    wrote(net, t, false, want_f32 ? kBoth : kPlanes);
    return XTB_OK;
  }
  auto gemm = [&](auto x, const int32_t* ix, float alpha) {
    if (lp.d.kind == XTB_CONV) conv_fwd(lp, x, ix, w, b, alpha, pre, B, st);
    else dense_fwd(lp, x, ix, w, b, alpha, pre, B, st);
  };
  if (lp.d.src == 0) {
    with_obs_type(net, obs, [&](auto x) { gemm(x, idx, net->desc.scale); });
  } else {
    int rc = ensure_f32(net, lp.d.src, B, false, st);
    if (rc) return rc;
    gemm((const float*)out_f32(net, lp.d.src), nullptr, 1.f);
  }
  LAUNCH_CHECK();
  if (ext) return act_forward(net, t, B, st);
  wrote(net, t, false, kF32);
  return XTB_OK;
}

static int op_wgrad(xtb_net* net, int i, const void* obs, const int32_t* idx, int B, cudaStream_t st, bool bias_done = false) {
  const LayerPlan& lp = net->L[i];
  if (lp.d.kind == XTB_DUELING || lp.d.kind == XTB_LOGSTD) return XTB_OK;   // no parameters / none fed by a tensor
  int t = i + 1;
  float* dw = net->grads + lp.w_off;
  float* db = net->grads + lp.b_off;
  const bool tc = use_tc(lp);
  if (tc) {
    int rc = ensure_bp(net, t, B, true, st);
    if (rc) return rc;
    rc = lp.d.src == 0 ? op_decode(net, obs, idx, B, st) : ensure_bp(net, lp.d.src, B, false, st);
    if (rc) return rc;
    cudaError_t te = tc_wgrad(net, i, B, st);
    if (te != cudaSuccess) return fail(XTB_ERR_CUDA, "tensor-core wgrad launch (layer %d): %s", i, cudaGetErrorString(te));
  } else {
    int rc = ensure_f32(net, t, B, true, st);
    if (rc) return rc;
    const float* dy = gout_f32(net, t);
    auto gemm = [&](auto x, const int32_t* ix, float alpha) {
      if (lp.d.kind == XTB_CONV) conv_wgrad(lp, x, ix, dy, alpha, dw, B, st, !bias_done);
      else dense_wgrad(lp, x, ix, dy, alpha, dw, B, st, !bias_done);
    };
    if (lp.d.src == 0) {
      with_obs_type(net, obs, [&](auto x) { gemm(x, idx, net->desc.scale); });
    } else {
      rc = ensure_f32(net, lp.d.src, B, false, st);
      if (rc) return rc;
      gemm((const float*)out_f32(net, lp.d.src), nullptr, 1.f);
    }
  }
  LAUNCH_CHECK();
  // bias gradient = column sums of dY over samples (and pixels), from the fp32 copy when it is current.  The fp32 GEMM
  // adds it as one more row unless it scales its input (the observation's decode scale).
  if (bias_done || (!tc && (lp.d.src != 0 || net->desc.scale == 1.f))) return XTB_OK;
  if (forms(net, t, true) & kF32) {
    int Mb = lp.d.kind == XTB_CONV ? B * lp.g.P : B;
    dim3 gridb((lp.N + 31) / 32, (Mb + 1023) / 1024);
    XLAUNCH(colsum_kernel, gridb, 256, 0, st, (const float*)gout_f32(net, t), Mb, lp.N, db);
  } else {
    XLAUNCH(bp::bp_colsum_kernel, (net->tsize[t] / 8 + 3) / 4, 128, 0, st, gout_bp(net, t), B, net->tsize[t], lp.N, db);
  }
  LAUNCH_CHECK();
  return XTB_OK;
}

// data gradient of layer i into its source tensor (gradient wrt the source's pre-activation)
// fuse_db: the epilogue also produces the bias gradient of the layer behind the source tensor (ordered partial sums)
static int op_dgrad(xtb_net* net, int i, int acc, int B, cudaStream_t st, bool fuse_db = false, int acc2 = 0) {
  const LayerPlan& lp = net->L[i];
  int t = i + 1, s = lp.d.src;
  if (lp.d.kind == XTB_DUELING) {   // both inputs; acc2: accumulate into the 1-wide input (tensor d.k)
    const int s2 = lp.d.k;
    int rc = ensure_f32(net, t, B, true, st);
    if (!rc) rc = ensure_f32(net, s, B, false, st);
    if (!rc) rc = ensure_f32(net, s2, B, false, st);
    if (!rc && acc) rc = ensure_f32(net, s, B, true, st);
    if (!rc && acc2) rc = ensure_f32(net, s2, B, true, st);
    if (rc) return rc;
    XLAUNCH(dueling_dgrad_kernel, (B + 7) / 8, 256, 0, st, (const float*)gout_f32(net, t), (const float*)out_f32(net, s),
            (const float*)out_f32(net, s2), B, lp.out_size, lp.src_act, lp.adv_act, acc, acc2, gout_f32(net, s), gout_f32(net, s2));
    LAUNCH_CHECK();
    wrote(net, s, true, kF32); wrote(net, s2, true, kF32);
    return XTB_OK;
  }
  if (use_tc(lp)) {
    int rc = ensure_bp(net, t, B, true, st);
    if (rc) return rc;
    if (dgrad_act(lp) != 0) { rc = ensure_bp(net, s, B, false, st); if (rc) return rc; }
    if (acc) { rc = ensure_bp(net, s, B, true, st); if (rc) return rc; }
    float* dbp = fuse_db ? (float*)(net->ws + lp.dbpart_off) : nullptr;
    cudaError_t te = tc_dgrad(net, i, B, acc, dbp, st);
    if (te != cudaSuccess) return fail(XTB_ERR_CUDA, "tensor-core dgrad launch (layer %d): %s", i, cudaGetErrorString(te));
    LAUNCH_CHECK();
    if (fuse_db) {
      const int units = lp.d.kind == XTB_CONV ? lp.q.H * lp.q.W : lp.K / lp.n_dg;
      queue_reduction(net, dbp, std::min(kSMs, units * ((B + 127) / 128)), lp.n_dg, lp.n_dg, net->L[s - 1].b_off);
    }
    wrote(net, s, true, kPlanes);
    return XTB_OK;
  }
  int rc = ensure_f32(net, t, B, true, st);
  if (rc) return rc;
  rc = ensure_f32(net, s, B, false, st);
  if (rc) return rc;
  if (acc) { rc = ensure_f32(net, s, B, true, st); if (rc) return rc; }
  const float* dy = gout_f32(net, t);
  const float* x = out_f32(net, s);
  float* gsrc = gout_f32(net, s);
  const float* w = net->params + lp.w_off;
  if (lp.d.kind == XTB_CONV) {
    ADgrad al{dy, lp.g, lp.dkyx, lp.dco, lp.sshift};
    BConvDgrad bl{w, lp.wk, lp.N};
    EpiDgrad ep{gsrc, x, dgrad_act(lp), lp.g.C, acc, nullptr, 0};
    launch_gemm(al, bl, ep, B * lp.g.H * lp.g.W, lp.g.C, lp.Kd, false, st);
  } else {
    ADense<float> al{dy, nullptr, lp.N};
    BTransposed bl{w, lp.N};
    EpiDgrad ep{gsrc, x, dgrad_act(lp), lp.K, acc, nullptr, 0};
    launch_gemm(al, bl, ep, B, lp.K, lp.N, false, st);
  }
  LAUNCH_CHECK();
  wrote(net, s, true, kF32);
  return XTB_OK;
}

// queued ordered reductions (conv weight gradients, fused bias gradients) -> flat gradient bucket, one launch
static int flush_reductions(xtb_net* net, cudaStream_t st) {
  if (net->pending.empty()) return XTB_OK;
  bp::RedSegs segs;
  memset(&segs, 0, sizeof segs);
  int mx = 0;
  if (net->pending.size() > bp::RED_MAX) return fail(XTB_ERR_STATE, "too many pending reductions");
  for (size_t k = 0; k < net->pending.size(); k++) { segs.s[k] = net->pending[k]; mx = std::max(mx, net->pending[k].count); }
  dim3 grid((mx + 127) / 128, (unsigned)net->pending.size());
  XLAUNCH(bp::grad_reduce_kernel, grid, 256, 0, st, segs, net->grads);
  LAUNCH_CHECK();
  net->pending.clear();
  return XTB_OK;
}

// ------------------------------------------------------------------------------------------
// forward / backward
// ------------------------------------------------------------------------------------------
// want_f32_mask: bit t set = tensor t is needed in fp32 row-major form (all tensors for the public entry point)
static int net_forward_impl(xtb_net* net, const float* params, const void* obs, const int32_t* gather_idx,
                            int batch, void* stream, unsigned skip_mask, unsigned want_f32_mask);
extern "C" int xtb_net_forward(xtb_net* net, const float* params, const void* obs, const int32_t* gather_idx,
                               int batch, void* stream) {
  return net_forward_impl(net, params, obs, gather_idx, batch, stream, 0u, ~0u);
}
static int net_forward_impl(xtb_net* net, const float* params, const void* obs, const int32_t* gather_idx,
                            int batch, void* stream, unsigned skip_mask, unsigned want_f32_mask) {
  if (!net || !net->ws) return fail(XTB_ERR_STATE, "xtb_net_forward: net not bound");
  if (batch <= 0 || batch > net->max_batch) return fail(XTB_ERR_ARG, "batch %d out of range (max %d)", batch, net->max_batch);
  if (!obs) return fail(XTB_ERR_ARG, "obs is null");
  const float* P = params ? params : net->params;
  const bool tc_allowed = (P == net->params);   // foreign parameters have no weight blobs: fp32 kernels
  cudaStream_t st = S(stream);
  const int nl = (int)net->L.size();
  invalidate(net, true, false);
  for (int i = 0; i < nl; i++) {
    if (skip_mask & (1u << i)) continue;
    const LayerPlan& lp = net->L[i];
    // dense layers write fp32 from the epilogue when asked; conv maps are merged afterwards (the only fp32 readers of
    // conv maps are uncovered layers and the public API)
    bool direct = lp.d.kind == XTB_DENSE && ((want_f32_mask >> (i + 1)) & 1u);
    // ... or when a layer outside the tensor-core path consumes it (exact fp32 instead of hi + lo)
    if (lp.d.kind == XTB_DENSE)
      for (int j = i + 1; j < nl; j++)
        if (reads(net->L[j], i + 1) && !(skip_mask & (1u << j)) && !(tc_allowed && use_tc(net->L[j]))) direct = true;
    int rc = op_forward(net, i, P, tc_allowed, obs, gather_idx, batch, direct, st);
    if (rc) return rc;
  }
  for (int t = 1; t <= nl; t++) {
    if (!((want_f32_mask >> t) & 1u) || (skip_mask & (1u << (t - 1))) || net->tsize[t] == 0) continue;
    int rc = ensure_f32(net, t, batch, false, st);
    if (rc) return rc;
  }
  return XTB_OK;
}

// What a backward pass starts from and does besides the layers' gradients.  Bit t of a mask stands for tensor t, bit i
// of skip for layer i.
struct BackwardOpts {
  const int32_t* heads; int n_heads;   // tensors whose gradient the caller filled: fp32 row-major, wrt the pre-activation
  unsigned heads_bp = 0u;              // ... of these, the ones filled in planes
  unsigned heads_dy = 0u;              // ... the ones (layers with an activation past tanh) filled wrt the output
  unsigned skip = 0u;                  // layers that are not run
  bool zero_grads = true;              // zero the gradient bucket and drop queued reductions (else a fused loss kernel queued its own)
  unsigned bias_done = 0u;             // tensors whose layer's bias gradient is already queued
  float* dobs = nullptr;               // also d loss / d observation, into dobs
  bool all_reduce = false;             // sum the gradient bucket over g_comm when one is installed
  BackwardOpts(const int32_t* h, int n) : heads(h), n_heads(n) {}
};
static int net_backward_impl(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch, void* stream,
                             const BackwardOpts& o);
extern "C" int xtb_net_backward(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch,
                                const int32_t* head_tensors, int n_heads, void* stream) {
  return net_backward_impl(net, obs, gather_idx, batch, stream, BackwardOpts(head_tensors, n_heads));
}
// d loss / d observation is defined for float observations that only dense layers read (decode scale 1)
static int input_grad_check(const xtb_net* net) {
  if (net->desc.input_u8 || net->desc.scale != 1.f) return fail(XTB_ERR_ARG, "input gradient: the observation must be float with scale 1");
  for (const auto& lp : net->L)
    if (lp.d.src == 0 && lp.d.kind != XTB_DENSE && lp.d.kind != XTB_LOGSTD)
      return fail(XTB_ERR_ARG, "input gradient: only dense layers may read the observation");
  return XTB_OK;
}
extern "C" int xtb_net_backward_input(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch,
                                      const int32_t* head_tensors, int n_heads, float* dobs, void* stream) {
  if (!obs || !dobs || !head_tensors) return fail(XTB_ERR_ARG, "xtb_net_backward_input: null pointer");
  BackwardOpts o(head_tensors, n_heads); o.dobs = dobs;
  return net_backward_impl(net, obs, gather_idx, batch, stream, o);
}
static int net_backward_impl(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch, void* stream,
                             const BackwardOpts& o) {
  if (!net || !net->ws || !net->grads) return fail(XTB_ERR_STATE, "xtb_net_backward: net not bound (grads required)");
  if (batch <= 0 || batch > net->max_batch) return fail(XTB_ERR_ARG, "batch out of range");
  if (o.dobs) { int rc = input_grad_check(net); if (rc) return rc; }
  cudaStream_t st = S(stream);
  xtb_comm* comm = o.all_reduce ? g_comm : nullptr;
  const int nl = (int)net->L.size();
  std::vector<char> has_grad(nl + 1, 0), written(nl + 1, 0);
  std::vector<char> dy(nl + 1, 0);          // the gradient is wrt the output of an act_is_ext layer: act_backward pending
  long long early_off = 0, early_cnt = 0;
  invalidate(net, false, true);
  if (o.zero_grads) net->pending.clear();
  for (int h = 0; h < o.n_heads; h++) {
    int t = o.heads[h];
    if (t < 1 || t > nl || net->tsize[t] == 0) return fail(XTB_ERR_ARG, "bad head tensor %d", t);
    has_grad[t] = 1; written[t] = 1; dy[t] = (o.heads_dy >> t) & 1u;
    wrote(net, t, true, (o.heads_bp >> t) & 1u ? kPlanes : kF32);
  }
  if (o.zero_grads) CUDA_TRY(cudaMemsetAsync(net->grads, 0, net->n_params * sizeof(float), st));
  // bias-gradient fusion: the bias gradient of the layer producing tensor s is the column sum of gout(s); when s has
  // exactly one consumer and that consumer's tensor-core data-gradient tile spans exactly the bias vector, its
  // epilogue accumulates the column sums (ordered partial sums, no atomics) and the separate pass is dropped
  std::vector<char> fuse_bias(nl + 1, 0);
  for (int s = 1; s <= nl; s++) {
    if (o.bias_done & (1u << s)) { fuse_bias[s] = 2; continue; }
    const LayerPlan& ps = net->L[s - 1];
    if (act_is_ext(ps.d.act)) continue;       // the column sums would be of the gradient wrt the output
    int consumers = 0, cj = -1;
    for (int j = 0; j < nl; j++) if (reads(net->L[j], s) && !(o.skip & (1u << j))) { consumers++; cj = j; }
    if (consumers != 1) continue;
    const LayerPlan& c = net->L[cj];
    if (!use_tc(c)) continue;
    if (ps.d.kind == XTB_CONV ? c.n_dg == ps.N : (c.d.kind == XTB_DENSE && c.n_dg == ps.N && c.K == ps.N)) fuse_bias[s] = 1;
  }
  for (int i = nl - 1; i >= 0; i--) {
    if (o.skip & (1u << i)) continue;
    const LayerPlan& lp = net->L[i];
    int t = i + 1;
    if (!has_grad[t]) continue;   // tensor does not influence the loss
    const bool act_bwd = dy[t] && act_is_ext(lp.d.act);      // act_backward also queues the bias gradient
    if (act_bwd) { int rc = act_backward(net, t, batch, st); if (rc) return rc; }
    int rc = op_wgrad(net, i, obs, gather_idx, batch, st, fuse_bias[t] != 0 || act_bwd);
    if (rc) return rc;
    // data parallel: a large dense weight gradient is final here (direct store) -- start summing it over ranks now, on
    // the communicator's side stream, while the rest of the backward pass runs
    if (comm && comm->world > 1 && early_cnt == 0 && lp.d.kind == XTB_DENSE && use_tc(lp) && (long long)lp.K * lp.N >= (1 << 16)) {
      early_off = lp.w_off; early_cnt = (long long)lp.K * lp.N;
      rc = comm_fork_allreduce(comm, net->grads + early_off, early_cnt, st);
      if (rc) return rc;
    }
    if (lp.d.kind == XTB_DUELING) {
      const int s = lp.d.src, s2 = lp.d.k;
      rc = op_dgrad(net, i, written[s] ? 1 : 0, batch, st, false, written[s2] ? 1 : 0);
      if (rc) return rc;
      written[s] = written[s2] = 1; has_grad[s] = has_grad[s2] = 1;
    } else if (lp.d.src != 0) {
      int s = lp.d.src;
      rc = op_dgrad(net, i, written[s] ? 1 : 0, batch, st, fuse_bias[s] == 1);
      if (rc) return rc;
      written[s] = 1; has_grad[s] = 1; dy[s] = 1;
    }
  }
  if (o.dobs) {   // d loss / d observation: the data-gradient GEMM of every dense layer reading it, summed in layer order
    bool first = true;
    for (int i = 0; i < nl; i++) {
      const LayerPlan& lp = net->L[i];
      if (lp.d.src != 0 || lp.d.kind != XTB_DENSE || (o.skip & (1u << i))) continue;
      if (!has_grad[i + 1]) continue;
      int rc = ensure_f32(net, i + 1, batch, true, st);
      if (rc) return rc;
      ADense<float> al{(const float*)gout_f32(net, i + 1), nullptr, lp.N};
      BTransposed bl{net->params + lp.w_off, lp.N};
      // linear: the epilogue's activation source is never used (dobs stands in as a valid address)
      EpiDgrad ep{o.dobs, o.dobs, 0, lp.K, first ? 0 : 1, nullptr, 0};
      launch_gemm(al, bl, ep, batch, lp.K, lp.N, false, st);
      LAUNCH_CHECK();
      first = false;
    }
    if (first) CUDA_TRY(cudaMemsetAsync(o.dobs, 0, (size_t)batch * net->tsize[0] * sizeof(float), st));
  }
  int rc = flush_reductions(net, st);
  if (rc || !comm || comm->world == 1) return rc;
  // the rest of the bucket: everything before and after the early range, as one NCCL group
  if (early_cnt == 0) return xtb_comm_allreduce(comm, net->grads, net->n_params, stream);
  int nrc = g_nccl.GroupStart();
  if (!nrc && early_off > 0) nrc = g_nccl.AllReduce(net->grads, net->grads, (size_t)early_off, kNcclFloat, kNcclSum, comm->comm, st);
  const long long tail = net->n_params - (early_off + early_cnt);
  if (!nrc && tail > 0)
    nrc = g_nccl.AllReduce(net->grads + early_off + early_cnt, net->grads + early_off + early_cnt, (size_t)tail, kNcclFloat, kNcclSum, comm->comm, st);
  int erc = g_nccl.GroupEnd();
  if (nrc || erc) return fail(XTB_ERR_CUDA, "ncclAllReduce: %s", g_nccl.GetErrorString(nrc ? nrc : erc));
  return comm_join(comm, st);
}

// Launch ONE kernel of one layer (0 = forward, 1 = weight gradient, 2 = data gradient, 3 = frame decode) on the
// tensors currently in the workspace: lets bench.py time the dominant kernel alone with CUDA events.
extern "C" int xtb_net_bench_layer(xtb_net* net, int layer, int which, const void* obs, const int32_t* gather_idx,
                                   int batch, void* stream) {
  if (!net || !net->ws || !net->grads) return fail(XTB_ERR_STATE, "xtb_net_bench_layer: net not bound");
  if (layer < 0 || layer >= (int)net->L.size() || batch <= 0 || batch > net->max_batch) return fail(XTB_ERR_ARG, "bad layer/batch");
  cudaStream_t st = S(stream);
  // tensors the caller filled through xtb_net_tensor / xtb_net_tensor_grad are fp32 row-major
  for (int t = 1; t <= (int)net->L.size(); t++)
    for (bool grad : {false, true})
      if (forms(net, t, grad) == kNone) wrote(net, t, grad, kF32);
  if (which == 0) return op_forward(net, layer, net->params, true, obs, gather_idx, batch, false, st);
  if (which == 1) { int rc = op_wgrad(net, layer, obs, gather_idx, batch, st, true); net->pending.clear(); return rc; }
  if (which == 2) {
    if (net->L[layer].d.src == 0) return fail(XTB_ERR_ARG, "layer reads the observation: no data gradient");
    int rc = op_dgrad(net, layer, 0, batch, st);
    net->pending.clear();
    return rc;
  }
  if (which == 3) { wrote(net, 0, false, kNone); return op_decode(net, obs, gather_idx, batch, st); }   // decode again
  return fail(XTB_ERR_ARG, "xtb_net_bench_layer: which must be 0..3");
}


// ------------------------------------------------------------------------------------------
// heads, GAE, losses
// ------------------------------------------------------------------------------------------
extern "C" int xtb_categorical_sample(const float* logits, int batch, int adim, const float* uniforms,
                                      uint64_t seed, uint64_t offset, int32_t* action, float* logp, void* stream) {
  if (!logits || !action || !logp || batch <= 0 || adim <= 0) return fail(XTB_ERR_ARG, "xtb_categorical_sample: bad argument");
  XLAUNCH(sample_kernel<Categorical>, (batch + 127) / 128, 128, 0, S(stream), logits, (const float*)nullptr, batch, adim, uniforms,
          seed, offset, (const unsigned long long*)nullptr, 0, action, logp, (const float*)nullptr, (float*)nullptr);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_argmax(const float* q, int batch, int adim, int32_t* action, void* stream) {
  if (!q || !action || batch <= 0 || adim <= 0) return fail(XTB_ERR_ARG, "xtb_argmax: bad argument");
  XLAUNCH(argmax_kernel, (batch + 127) / 128, 128, 0, S(stream), q, batch, adim, action);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_gae(const float* value, const float* reward, const uint8_t* done, int n_env, int n_step,
                       float gamma, float lam, int sign_clip, float* adv, float* old_value, float* target_value,
                       void* stream) {
  if (!value || !reward || !done || !adv || !old_value || !target_value) return fail(XTB_ERR_ARG, "xtb_gae: null pointer");
  if (n_env == 0 || n_step == 0) return XTB_OK;   // empty rollout: nothing to do
  if (n_env < 0 || n_step < 0) return fail(XTB_ERR_ARG, "xtb_gae: negative size");
  int threads = 128;  // 4 envs per block
  int blocks = (n_env * 32 + threads - 1) / threads;
  XLAUNCH(gae_kernel, blocks, threads, 0, S(stream), value, reward, done, n_env, n_step, gamma, lam, sign_clip, adv,
                                                old_value, target_value);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_ppo_loss_grad(const float* logits, const float* v, const int32_t* gather_idx,
                                 const int32_t* action, const float* old_logp, const float* adv,
                                 const float* old_v, const float* target_v, int batch, int adim,
                                 const xtb_ppo_hyper* hp, float inv_count, float* dlogits, float* dv,
                                 float* loss_out, void* stream) {
  if (!logits || !v || !action || !old_logp || !adv || !old_v || !target_v || !hp || !dlogits || !dv || !loss_out)
    return fail(XTB_ERR_ARG, "xtb_ppo_loss_grad: null pointer");
  if (batch <= 0 || adim <= 0 || adim > MAX_ADIM) return fail(XTB_ERR_ARG, "xtb_ppo_loss_grad: batch/adim out of range");
  PpoHyperDev h{hp->clip_ratio, hp->ent_coef, hp->vf_clip, hp->critic_coef};
  XLAUNCH(ppo_loss_kernel, (batch + 127) / 128, 128, 0, S(stream), logits, v, gather_idx, action, old_logp, adv, old_v,
                                                              target_v, batch, adim, h, inv_count, dlogits, dv, loss_out);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_diag_gaussian_sample(const float* mean, const float* log_std, int batch, int adim, const float* normals,
                                        uint64_t seed, uint64_t offset, float* action, float* logp, void* stream) {
  if (!mean || !log_std || !action || !logp || batch <= 0 || adim <= 0 || adim > MAX_ADIM)
    return fail(XTB_ERR_ARG, "xtb_diag_gaussian_sample: bad argument");
  XLAUNCH(sample_kernel<DiagGaussian>, (batch + 127) / 128, 128, 0, S(stream), mean, log_std, batch, adim, normals, seed, offset,
          (const unsigned long long*)nullptr, 0, action, logp, (const float*)nullptr, (float*)nullptr);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_ppo_gauss_loss_grad(const float* mean, const float* v, const float* log_std, const int32_t* gather_idx,
                                       const float* action, const float* old_logp, const float* adv, const float* old_v,
                                       const float* target_v, int batch, int adim, const xtb_ppo_hyper* hp, float inv_count,
                                       float* dmean, float* dv, float* dlog_std, float* loss_out, void* stream) {
  if (!mean || !v || !log_std || !action || !old_logp || !adv || !old_v || !target_v || !hp || !dmean || !dv || !dlog_std || !loss_out)
    return fail(XTB_ERR_ARG, "xtb_ppo_gauss_loss_grad: null pointer");
  if (batch <= 0 || adim <= 0 || adim > MAX_ADIM) return fail(XTB_ERR_ARG, "xtb_ppo_gauss_loss_grad: batch/adim out of range");
  PpoHyperDev h{hp->clip_ratio, hp->ent_coef, hp->vf_clip, hp->critic_coef};
  if (adim <= 8)
    XLAUNCH(ppo_gauss_loss_kernel<8>, 1, GAUSS_LOSS_THREADS, 0, S(stream), mean, v, log_std, gather_idx, action, old_logp, adv, old_v,
            target_v, batch, adim, h, inv_count, dmean, dv, dlog_std, loss_out);
  else
    XLAUNCH(ppo_gauss_loss_kernel<MAX_ADIM>, 1, GAUSS_LOSS_THREADS, 0, S(stream), mean, v, log_std, gather_idx, action, old_logp, adv,
            old_v, target_v, batch, adim, h, inv_count, dmean, dv, dlog_std, loss_out);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_vtrace_loss_grad(const float* tp_logits, const float* baseline, const float* bp_logits,
                                    const int32_t* action, const uint8_t* done, const float* reward,
                                    int n_traj, int step_len, int adim, float gamma, float* dlogits,
                                    float* dbaseline, float* vs_out, float* pg_adv_out, float* loss_out,
                                    void* stream) {
  if (!tp_logits || !baseline || !bp_logits || !action || !done || !reward || !dlogits || !dbaseline || !loss_out)
    return fail(XTB_ERR_ARG, "xtb_vtrace_loss_grad: null pointer");
  if (n_traj <= 0 || step_len < 2 || adim <= 0 || adim > MAX_ADIM) return fail(XTB_ERR_ARG, "xtb_vtrace_loss_grad: bad sizes");
  int threads = 128;
  int blocks = (n_traj * 32 + threads - 1) / threads;
  XLAUNCH(vtrace_kernel, blocks, threads, 0, S(stream), tp_logits, baseline, bp_logits, action, done, reward, n_traj,
                                                   step_len, adim, gamma, dlogits, dbaseline, vs_out, pg_adv_out, loss_out);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_dqn_td_loss_grad(const float* q, const float* q_next_target, const float* q_next_online, const int32_t* idx,
                                    const int32_t* action, const float* reward, const uint8_t* done, const float* disc, int batch,
                                    int adim, float gamma, float huber_delta, float inv_count, float* dq, float* y_out,
                                    float* loss_out, void* stream) {
  if (!q || !q_next_target || !action || !reward || !done || !dq || !loss_out) return fail(XTB_ERR_ARG, "xtb_dqn_td_loss_grad: null pointer");
  if (batch <= 0 || adim <= 0) return fail(XTB_ERR_ARG, "xtb_dqn_td_loss_grad: bad sizes");
  XLAUNCH(dqn_loss_kernel, (batch + 127) / 128, 128, 0, S(stream), q, q_next_target, q_next_online, idx, action, reward, done, disc,
          batch, adim, gamma, huber_delta, inv_count, dq, y_out, loss_out);
  LAUNCH_CHECK();
  return XTB_OK;
}
extern "C" int xtb_dqn_loss_grad(const float* q, const float* q_next_target, const float* q_next_online,
                                 const int32_t* action, const float* reward, const uint8_t* done, int batch,
                                 int adim, float gamma, float inv_count, float* dq, float* y_out,
                                 float* loss_out, void* stream) {
  return xtb_dqn_td_loss_grad(q, q_next_target, q_next_online, nullptr, action, reward, done, nullptr, batch, adim, gamma, 0.f,
                              inv_count, dq, y_out, loss_out, stream);
}
extern "C" int xtb_nstep_returns(const float* reward, const uint8_t* done, int n_env, int n_step, int n, float gamma, float* ret,
                                 float* disc, int32_t* last, uint8_t* done_n, void* stream) {
  if (!reward || !done || !ret || !disc || !last || !done_n) return fail(XTB_ERR_ARG, "xtb_nstep_returns: null pointer");
  if (n_env <= 0 || n_step <= 0 || n <= 0) return fail(XTB_ERR_ARG, "xtb_nstep_returns: bad sizes");
  XLAUNCH(nstep_kernel, (n_env * n_step + 127) / 128, 128, 0, S(stream), reward, done, n_env, n_step, n, gamma, ret, disc, last, done_n);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_softmax(const float* logits, int batch, int adim, float* probs, void* stream) {
  if (!logits || !probs || batch <= 0 || adim <= 0) return fail(XTB_ERR_ARG, "xtb_softmax: bad argument");
  XLAUNCH(softmax_rows_kernel, (batch + 127) / 128, 128, 0, S(stream), logits, batch, adim, probs);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_impala_keras_loss_grad(const float* logits, const float* v, const int32_t* idx, const float* action_mat,
                                          const float* adv, const float* target_v, int batch, int adim, float ent_coef,
                                          float value_weight, float loss_scale, float* dlogits, float* dv, float* loss_out,
                                          void* stream) {
  if (!logits || !v || !action_mat || !adv || !target_v || !dlogits || !dv || !loss_out)
    return fail(XTB_ERR_ARG, "xtb_impala_keras_loss_grad: null pointer");
  if (batch <= 0 || adim <= 0 || adim > MAX_ADIM) return fail(XTB_ERR_ARG, "xtb_impala_keras_loss_grad: batch/adim out of range");
  XLAUNCH(impala_keras_loss_kernel, 1, KERAS_LOSS_THREADS, 0, S(stream), logits, v, idx, action_mat, adv, target_v, batch, adim,
          ent_coef, value_weight, loss_scale, dlogits, dv, loss_out);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_mse_loss_grad(const float* q, const float* y, int batch, int adim, float inv_count, float* dq,
                                 float* loss_out, void* stream) {
  if (!q || !y || !dq || !loss_out || batch <= 0 || adim <= 0) return fail(XTB_ERR_ARG, "xtb_mse_loss_grad: bad argument");
  long long n = (long long)batch * adim;
  XLAUNCH(mse_loss_kernel, (unsigned)((n + 127) / 128), 128, 0, S(stream), q, y, n, inv_count, dq, loss_out);
  LAUNCH_CHECK();
  return XTB_OK;
}

// ------------------------------------------------------------------------------------------
// optimiser
// ------------------------------------------------------------------------------------------
struct xtb_adam {
  long long count = 0;
  float lr, beta1, beta2, eps, clip;
  int clip_mode = 0, n_seg = 0, n_blk = 0;
  float *m = nullptr, *v = nullptr;
  float* mg = nullptr; float rms_rho = 0.f, rms_eps = 0.f;   // centred RMSProp instead of Adam when mg != NULL (m = ms)
  int* blk_seg = nullptr; long long* blk_beg = nullptr; int* blk_len = nullptr;
  double* norm_sq = nullptr; float* seg_scale = nullptr; AdamState* st = nullptr; AdamHyper* hyp = nullptr; unsigned int* ticket = nullptr;
};

// The optimiser kernels read and write every buffer as float4 wherever a chunk starts at a multiple of 4 elements.
static inline bool misaligned16(const void* p) { return (uintptr_t)p % 16 != 0; }

extern "C" int xtb_adam_create(long long count, float lr, float beta1, float beta2, float eps, int clip_mode,
                               float clip, const long long* seg_offsets, int n_seg, float* m, float* v,
                               xtb_adam** out) {
  if (count <= 0 || !m || !v || !out) return fail(XTB_ERR_ARG, "xtb_adam_create: bad argument");
  if (clip_mode != XTB_CLIP_NONE && clip_mode != XTB_CLIP_GLOBAL_NORM && clip_mode != XTB_CLIP_PER_TENSOR)
    return fail(XTB_ERR_ARG, "xtb_adam_create: unknown clip_mode %d", clip_mode);
  // clip / max(norm, clip) climbs the gradient for clip < 0 and is 0/0 for clip = 0 and a zero gradient
  if (clip_mode != XTB_CLIP_NONE && !(clip > 0.f))
    return fail(XTB_ERR_ARG, "xtb_adam_create: clip must be > 0 with a clipping mode (got %g)", (double)clip);
  if (misaligned16(m) || misaligned16(v)) return fail(XTB_ERR_ARG, "xtb_adam_create: m and v must be 16-byte aligned");
  std::vector<long long> seg;
  if (clip_mode == XTB_CLIP_PER_TENSOR) {
    if (!seg_offsets || n_seg <= 0) return fail(XTB_ERR_ARG, "per-tensor clip needs segment offsets");
    seg.assign(seg_offsets, seg_offsets + n_seg + 1);
    if (seg.front() != 0 || seg.back() != count) return fail(XTB_ERR_ARG, "segment offsets must span [0,count]");
    for (int s = 0; s < n_seg; s++)        // a decreasing pair would hand the same parameters to two blocks
      if (seg[s + 1] < seg[s])
        return fail(XTB_ERR_ARG, "xtb_adam_create: segment offsets must not decrease (offset %d: %lld < %lld)", s + 1, seg[s + 1], seg[s]);
  } else {
    seg = {0, count};
  }
  auto* o = new xtb_adam();
  o->count = count; o->lr = lr; o->beta1 = beta1; o->beta2 = beta2; o->eps = eps; o->clip = clip;
  o->clip_mode = clip_mode; o->n_seg = (int)seg.size() - 1; o->m = m; o->v = v;
  std::vector<int> bseg, blen; std::vector<long long> bbeg;
  for (int s = 0; s < o->n_seg; s++)
    for (long long b = seg[s]; b < seg[s + 1]; b += OPT_CHUNK) {
      bseg.push_back(s); bbeg.push_back(b); blen.push_back((int)std::min<long long>(OPT_CHUNK, seg[s + 1] - b));
    }
  o->n_blk = (int)bseg.size();
  AdamState init{1.f, 1.f, 0.f, 0.f, 0u};
  cudaError_t e = cudaSuccess;
  auto chk = [&](cudaError_t r) { if (e == cudaSuccess) e = r; };
  chk(cudaMalloc(&o->blk_seg, o->n_blk * sizeof(int)));
  chk(cudaMalloc(&o->blk_beg, o->n_blk * sizeof(long long)));
  chk(cudaMalloc(&o->blk_len, o->n_blk * sizeof(int)));
  chk(cudaMalloc(&o->norm_sq, o->n_seg * sizeof(double)));
  chk(cudaMalloc(&o->seg_scale, o->n_seg * sizeof(float)));
  chk(cudaMalloc(&o->st, sizeof(AdamState)));
  chk(cudaMalloc(&o->hyp, sizeof(AdamHyper)));
  chk(cudaMalloc(&o->ticket, sizeof(unsigned int)));
  if (e == cudaSuccess) {
    chk(cudaMemcpy(o->blk_seg, bseg.data(), o->n_blk * sizeof(int), cudaMemcpyHostToDevice));
    chk(cudaMemcpy(o->blk_beg, bbeg.data(), o->n_blk * sizeof(long long), cudaMemcpyHostToDevice));
    chk(cudaMemcpy(o->blk_len, blen.data(), o->n_blk * sizeof(int), cudaMemcpyHostToDevice));
    chk(cudaMemset(o->norm_sq, 0, o->n_seg * sizeof(double)));
    chk(cudaMemcpy(o->st, &init, sizeof init, cudaMemcpyHostToDevice));
    chk(cudaMemset(o->ticket, 0, sizeof(unsigned int)));
    AdamHyper hy{lr, beta1, beta2, eps, clip, 0.f};
    chk(cudaMemcpy(o->hyp, &hy, sizeof hy, cudaMemcpyHostToDevice));
    chk(cudaMemset(m, 0, count * sizeof(float)));
    chk(cudaMemset(v, 0, count * sizeof(float)));
  }
  if (e != cudaSuccess) { xtb_adam_destroy(o); return fail(XTB_ERR_CUDA, "xtb_adam_create: %s", cudaGetErrorString(e)); }
  *out = o;
  return XTB_OK;
}

extern "C" void xtb_adam_destroy(xtb_adam* o) {
  if (!o) return;
  drop_graphs_of(o);
  cudaFree(o->blk_seg); cudaFree(o->blk_beg); cudaFree(o->blk_len);
  cudaFree(o->norm_sq); cudaFree(o->seg_scale); cudaFree(o->st); cudaFree(o->hyp); cudaFree(o->ticket);
  delete o;
}

static int adam_step_impl(xtb_adam* o, float* params, const float* grads, float grad_scale, void* stream, xtb_net* net);
extern "C" int xtb_adam_step(xtb_adam* o, float* params, const float* grads, float grad_scale, void* stream) {
  return adam_step_impl(o, params, grads, grad_scale, stream, nullptr);
}
// optimiser step on a network's bound parameters; the same kernel refreshes the weight blobs of its tensor-core layers
extern "C" int xtb_adam_step_net(xtb_adam* o, xtb_net* net, float grad_scale, void* stream) {
  if (!net || !net->ws || !net->params || !net->grads) return fail(XTB_ERR_STATE, "xtb_adam_step_net: net not bound");
  if (!o || o->count != net->n_params) return fail(XTB_ERR_ARG, "xtb_adam_step_net: optimiser/net size mismatch");
  return adam_step_impl(o, net->params, net->grads, grad_scale, stream, net);
}
static int adam_step_impl(xtb_adam* o, float* params, const float* grads, float grad_scale, void* stream, xtb_net* net) {
  if (!o || !params || !grads) return fail(XTB_ERR_ARG, "xtb_adam_step: null pointer");
  if (misaligned16(params) || misaligned16(grads) || misaligned16(o->m) || misaligned16(o->v) || misaligned16(o->mg))
    return fail(XTB_ERR_ARG, "xtb_adam_step: params, grads and the optimiser slots must be 16-byte aligned");
  cudaStream_t st = S(stream);
  XLAUNCH(sqnorm_kernel, (o->n_blk + SQN_GROUP - 1) / SQN_GROUP, OPT_THREADS, 0, st, grads, o->blk_seg, o->blk_beg, o->blk_len, o->n_blk, o->norm_sq, o->ticket, o->st,
          (const AdamHyper*)o->hyp, o->seg_scale, o->n_seg, o->clip_mode, grad_scale);
  LAUNCH_CHECK();
  const bool blobs = net && !net->blob_segs.empty();
  if (o->mg) {
    XLAUNCH(rmsprop_kernel, o->n_blk, OPT_THREADS, 0, st, params, grads, o->m, o->mg, o->blk_seg, o->blk_beg, o->blk_len,
            o->seg_scale, (const AdamHyper*)o->hyp, o->rms_rho, o->rms_eps, blobs ? (const bp::BlobSeg*)(net->ws + net->segs_off) : nullptr,
            blobs ? (int)net->blob_segs.size() : 0, blobs ? (__nv_bfloat16*)(net->ws + net->blob_off) : nullptr, blobs ? net->blob_elems : 0LL);
    LAUNCH_CHECK();
    return XTB_OK;
  }
  XLAUNCH(adam_kernel, o->n_blk, OPT_THREADS, 0, st, params, grads, o->m, o->v, o->blk_seg, o->blk_beg, o->blk_len,
          o->seg_scale, o->st, (const AdamHyper*)o->hyp, blobs ? (const bp::BlobSeg*)(net->ws + net->segs_off) : nullptr,
          blobs ? (int)net->blob_segs.size() : 0, blobs ? (__nv_bfloat16*)(net->ws + net->blob_off) : nullptr, blobs ? net->blob_elems : 0LL);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" const float* xtb_adam_grad_norm(const xtb_adam* o) { return o ? &o->st->grad_norm : nullptr; }
extern "C" int xtb_opt_use_rmsprop(xtb_adam* o, float* mean_grad, float decay, float epsilon) {
  if (!o || !mean_grad) return fail(XTB_ERR_ARG, "xtb_opt_use_rmsprop: null pointer");
  if (misaligned16(mean_grad)) return fail(XTB_ERR_ARG, "xtb_opt_use_rmsprop: mean_grad must be 16-byte aligned");
  if (!(decay > 0.f && decay < 1.f) || !(epsilon > 0.f)) return fail(XTB_ERR_ARG, "xtb_opt_use_rmsprop: decay in (0,1), epsilon > 0");
  drop_graphs_of(o);                       // captured steps baked the Adam kernel in
  {   // slot initial values of tf.train.RMSPropOptimizer: rms = ones, mg = zeros (one-time, synchronous)
    std::vector<float> ones((size_t)o->count, 1.f);
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(o->m, ones.data(), ones.size() * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemset(mean_grad, 0, ones.size() * sizeof(float)));
  }
  o->mg = mean_grad; o->rms_rho = decay; o->rms_eps = epsilon;
  return XTB_OK;
}
extern "C" int xtb_adam_set_lr(xtb_adam* o, float lr) {
  if (!o) return fail(XTB_ERR_ARG, "null optimiser");
  o->lr = lr;
  // device-resident: captured graphs read it at replay time.  Ordered after everything already submitted.
  CUDA_TRY(cudaDeviceSynchronize());
  CUDA_TRY(cudaMemcpy(&o->hyp->lr, &lr, sizeof lr, cudaMemcpyHostToDevice));
  return XTB_OK;
}
extern "C" int xtb_adam_set_decay(xtb_adam* o, float decay) {
  if (!o) return fail(XTB_ERR_ARG, "null optimiser");
  if (!(decay >= 0.f)) return fail(XTB_ERR_ARG, "xtb_adam_set_decay: decay must be >= 0");
  CUDA_TRY(cudaDeviceSynchronize());      // device-resident, like the learning rate
  CUDA_TRY(cudaMemcpy(&o->hyp->decay, &decay, sizeof decay, cudaMemcpyHostToDevice));
  return XTB_OK;
}

// ------------------------------------------------------------------------------------------
// fused PPO learner loop
// ------------------------------------------------------------------------------------------
// CUDA graphs cannot be captured on the legacy default stream, which is what a host that never creates streams
// (stream == NULL) runs on.  Such calls are moved onto a private non-blocking stream of the current device, fenced
// against the legacy stream with events on both sides, so the caller keeps default-stream ordering semantics.
struct EngineStream { cudaStream_t st = nullptr; cudaEvent_t in = nullptr, out = nullptr; };
static EngineStream g_engine_streams[64];
struct StreamScope {
  cudaStream_t st = nullptr;
  EngineStream* es = nullptr;
  int begin(void* stream, bool side_if_null) {
    st = S(stream);
    if (st || !side_if_null) return XTB_OK;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) return fail(XTB_ERR_ARG, "device index %d out of range", dev);
    EngineStream& e = g_engine_streams[dev];
    if (!e.st) {
      CUDA_TRY(cudaStreamCreateWithFlags(&e.st, cudaStreamNonBlocking));
      CUDA_TRY(cudaEventCreateWithFlags(&e.in, cudaEventDisableTiming));
      CUDA_TRY(cudaEventCreateWithFlags(&e.out, cudaEventDisableTiming));
    }
    CUDA_TRY(cudaEventRecord(e.in, nullptr));
    CUDA_TRY(cudaStreamWaitEvent(e.st, e.in, 0));
    es = &e; st = e.st;
    return XTB_OK;
  }
  int end() {
    if (!es) return XTB_OK;
    CUDA_TRY(cudaEventRecord(es->out, es->st));
    CUDA_TRY(cudaStreamWaitEvent(nullptr, es->out, 0));
    es = nullptr;
    return XTB_OK;
  }
};
static int g_fuse_heads = [] { const char* e = getenv("XTB_FUSE_HEADS"); return e ? atoi(e) : 1; }();
extern "C" int xtb_set_fuse_heads(int on) { g_fuse_heads = on; return XTB_OK; }

// ---- CUDA-graph cache of the fused entry points ------------------------------------------------
// A captured graph bakes in every kernel argument, so its key holds everything the capture reads.  capture_key()
// zeroes it and fills the entry point, the owners and the arguments; run_graph() adds the communicator and the
// modes, which every capture reads.  Keys are compared bytewise.
enum GraphTag { kPpoTrain = 1, kImpalaTrain, kDqnTrain, kRolloutInfer, kImpalaKerasFit, kImpalaKerasTrain, kMuzeroTrain,
                kMuzeroInitInfer, kMuzeroRecurInfer, kMuzeroSearch };
struct CaptureKey {
  uint64_t tag;          // entry point
  const void* own[6];    // the objects the capture reads (nets, optimiser, ...) and the communicator (own[5]):
                         // destroying one, or rebinding a net, drops the graph
  uint64_t mode[2];      // kernel-path and fused-heads modes
  uint64_t arg[21];      // every pointer and scalar argument; floats by bit pattern
  bool operator<(const CaptureKey& o) const { return memcmp(this, &o, sizeof(CaptureKey)) < 0; }
};
template <class T> static uint64_t key_word(T v) {
  if constexpr (std::is_same_v<T, float>) { uint32_t u; memcpy(&u, &v, sizeof u); return u; }
  else if constexpr (std::is_same_v<T, double>) { uint64_t u; memcpy(&u, &v, sizeof u); return u; }
  else if constexpr (std::is_pointer_v<T>) return (uint64_t)(uintptr_t)v;
  else return (uint64_t)v;
}
template <size_t N, class... A>
static CaptureKey capture_key(GraphTag tag, const void* const (&owners)[N], A... args) {
  static_assert(N < sizeof(CaptureKey::own) / sizeof(void*), "CaptureKey::own too small");
  static_assert(sizeof...(A) <= sizeof(CaptureKey::arg) / sizeof(uint64_t), "CaptureKey::arg too small");
  CaptureKey k;
  memset(&k, 0, sizeof k);
  k.tag = tag;
  std::copy(owners, owners + N, k.own);
  const uint64_t w[] = {key_word(args)...};
  memcpy(k.arg, w, sizeof w);
  return k;
}
struct GraphVal { cudaGraphExec_t exec; long long kernels; };
static constexpr size_t kMaxCachedGraphs = 256;   // beyond it the cache is emptied (keys are buffer addresses)
static std::map<CaptureKey, GraphVal> g_graphs;
static std::atomic<long long> g_graph_replays{0};
extern "C" long long xtb_graph_replay_count(void) { return g_graph_replays.load(); }

// cached graphs hold raw pointers into their owners: they die with the object (a later object may be allocated at
// the same address) and with a net's binding
static void drop_graphs_of(const void* obj) {
  for (auto it = g_graphs.begin(); it != g_graphs.end();) {
    const auto& own = it->first.own;
    if (std::find(std::begin(own), std::end(own), obj) != std::end(own)) { cudaGraphExecDestroy(it->second.exec); it = g_graphs.erase(it); } else ++it;
  }
}

// use_graph == 0: launch(stream) runs eagerly.  Otherwise the launches are captured once per key, with the global
// state every capture reads added to it, and the graph is replayed.
template <class F>
static int run_graph(CaptureKey key, int use_graph, void* stream, F&& launch) {
  if (!use_graph) return launch(stream);
  key.own[5] = g_comm; key.mode[0] = g_tc_mode; key.mode[1] = g_fuse_heads;
  StreamScope sc;
  int src = sc.begin(stream, true);
  if (src) return src;
  auto it = g_graphs.find(key);
  if (it == g_graphs.end()) {
    cudaStream_t st = sc.st;
    long long before = g_launches.load();
    CUDA_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    int rc = launch((void*)st);
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamEndCapture(st, &graph);
    long long captured = g_launches.load() - before;
    g_launches.store(before);   // captured, not launched yet
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (e != cudaSuccess) return fail(XTB_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    cudaGraphExec_t exec = nullptr;
    e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) return fail(XTB_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(e));
    if (g_graphs.size() >= kMaxCachedGraphs) {     // callers that pass fresh buffers every call must not leak executables
      for (auto& kv : g_graphs) cudaGraphExecDestroy(kv.second.exec);
      g_graphs.clear();
    }
    it = g_graphs.emplace(key, GraphVal{exec, captured}).first;
  }
  CUDA_TRY(cudaGraphLaunch(it->second.exec, sc.st));
  g_launches.fetch_add(it->second.kernels, std::memory_order_relaxed);
  g_graph_replays.fetch_add(1, std::memory_order_relaxed);
  return sc.end();
}

// The epoch x minibatch loop of PPO.train (xt/model/ppo/ppo.py:111-132): minibatch k of epoch e holds rows
// perm[e*N + k*B ...] (the last one ragged).  minibatch(idx, mb, loss) enqueues its forward, loss and backward; the
// optimiser step follows.
template <class STEP>
static int ppo_epoch_loop(xtb_net* net, xtb_adam* opt, int N, int B, int E, const int32_t* perm, float* loss_per_step,
                          void* stream, STEP&& minibatch) {
  int steps_per_epoch = (N + B - 1) / B;
  CUDA_TRY(cudaMemsetAsync(loss_per_step, 0, sizeof(float) * E * steps_per_epoch, S(stream)));
  int step = 0;
  for (int e = 0; e < E; e++) {
    for (int s0 = 0; s0 < N; s0 += B, step++) {
      int mb = std::min(B, N - s0);
      int rc = minibatch(perm + (long long)e * N + s0, mb, loss_per_step + step);
      if (rc) return rc;
      rc = xtb_adam_step_net(opt, net, 1.f, stream);
      if (rc) return rc;
    }
  }
  return XTB_OK;
}

// loss / gradient scale of the training loops that average over the local batch: 1 / world while a communicator sums
// the gradients over ranks, else 1
static float dp_inv_world() { return g_comm ? 1.f / g_comm->world : 1.f; }

// What every learner entry point checks before it launches anything: none of the pointers it needs is NULL (`missing`:
// each caller names its own), the net is bound with gradients, the optimiser spans the trained parameters (n_params,
// 0: the net's; opt NULL: an inference call), the `rows` samples of one forward are in [1, max_rows] (0: the net's
// max_batch) and, for a learner that cannot sum its gradients over ranks (dp_ok false), no communicator is installed.
static int learner_check(const char* fn, bool missing, const xtb_net* net, const xtb_adam* opt, long long rows, bool dp_ok,
                         long long max_rows = 0, long long n_params = 0) {
  if (missing) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (!net->ws || !net->grads) return fail(XTB_ERR_STATE, "%s: net not bound", fn);
  if (!dp_ok && g_comm) return fail(XTB_ERR_STATE, "%s: data-parallel training (communicator) is not supported", fn);
  if (opt && opt->count != (n_params ? n_params : net->n_params))
    return fail(XTB_ERR_ARG, "%s: optimiser/net size mismatch (%lld != %lld)", fn, opt->count, n_params ? n_params : net->n_params);
  if (!max_rows) max_rows = net->max_batch;
  if (rows < 1 || rows > max_rows) return fail(XTB_ERR_ARG, "%s: batch %lld not in [1, %lld]", fn, rows, max_rows);
  return XTB_OK;
}

// Fused PPO heads of tensors pi_t / v_t: both heads are linear dense layers on hidden (non-observation) tensors of equal
// width within the heads_kernel limits (infer: the infer_heads_kernel limits), and the fused-heads mode is on
static bool ppo_heads_fusable(const xtb_net* net, int pi_t, int v_t, bool infer) {
  const LayerPlan& lpi = net->L[pi_t - 1];
  const LayerPlan& lv = net->L[v_t - 1];
  return g_fuse_heads && lpi.d.kind == XTB_DENSE && lv.d.kind == XTB_DENSE && lpi.d.act == 0 && lv.d.act == 0 &&
         lpi.d.src != 0 && lv.d.src != 0 && lpi.K == lv.K && heads_fit(lpi.K, net->tsize[pi_t], infer);
}

// One fused minibatch after the forward of the layers below the heads pi_t / v_t (the PPO heads, or the dueling value /
// adv streams): heads_kernel<LOSS> evaluates both heads, the loss and their backward, writes the gradient wrt the
// hidden tensors (straight into their planes when the hidden layer runs on tensor cores), and its per-block slabs are
// queued for the ordered reduction at the end of the backward pass of the layers below, which follows.  `a` carries
// the loss inputs (idx, rollout arrays, hyper-parameters); the slab's loss goes to *loss_dst; ls_off >= 0: the offset
// of the log_std floats whose gradient the policy adds to the slab (LOSS::kLogStd).
template <class LOSS>
static int heads_fused(xtb_net* net, const void* obs, PpoHeadsArgs& a, int mb, int pi_t, int v_t, unsigned skip,
                       long long ls_off, float* loss_dst, void* stream) {
  const LayerPlan& lpi = net->L[pi_t - 1];
  const LayerPlan& lv = net->L[v_t - 1];
  const int adim = net->tsize[pi_t];
  const int32_t* idx = a.idx;
  CUDA_TRY(cudaMemsetAsync(net->grads, 0, net->n_params * sizeof(float), S(stream)));
  net->pending.clear();
  a.h_pi = out_f32(net, lpi.d.src); a.h_v = out_f32(net, lv.d.src);
  a.g_pi = gout_f32(net, lpi.d.src); a.g_v = gout_f32(net, lv.d.src);
  // hidden-layer gradients go straight into batch-planar planes when the hidden layer runs on tensor cores
  // (a hidden layer with an activation past tanh gets the gradient wrt its output, in fp32, and act_backward follows)
  const bool ext_pi = act_is_ext(lpi.src_act), ext_v = act_is_ext(lv.src_act);
  const bool bp_pi = use_tc(net->L[lpi.d.src - 1]) && net->plane_elems[lpi.d.src] > 0 && !ext_pi;
  const bool bp_v = use_tc(net->L[lv.d.src - 1]) && net->plane_elems[lv.d.src] > 0 && !ext_v;
  a.gp_hi = bp_pi ? gout_bp(net, lpi.d.src).hi : nullptr; a.gp_lo = net->plane_elems[lpi.d.src];
  a.gv_hi = bp_v ? gout_bp(net, lv.d.src).hi : nullptr; a.gv_lo = net->plane_elems[lv.d.src];
  a.pitch = net->pitch;
  a.w_pi = net->params + lpi.w_off; a.b_pi = net->params + lpi.b_off; a.w_v = net->params + lv.w_off; a.b_v = net->params + lv.b_off;
  // the hidden layers' bias gradients (column sums of g) when they are dense and only feed the heads
  auto only_feeds_heads = [&](int tsr) { for (int j = 0; j < (int)net->L.size(); j++) if (reads(net->L[j], tsr) && !(skip & (1u << j))) return false; return true; };
  bool bh_pi_ok = net->L[lpi.d.src - 1].d.kind == XTB_DENSE && only_feeds_heads(lpi.d.src) && !ext_pi;
  bool bh_v_ok = net->L[lv.d.src - 1].d.kind == XTB_DENSE && only_feeds_heads(lv.d.src) && !ext_v;
  a.B = mb; a.K = lpi.K; a.A = adim; a.act_pi = dgrad_act(lpi); a.act_v = dgrad_act(lv); a.shared = lpi.d.src == lv.d.src ? 1 : 0;
  int blocks = std::max(1, std::min(kSMs, (mb + 7) / 8));      // one sample per warp up to 1184 samples
  const int HK = lpi.K, nacc = HK * adim + 3 * HK + adim + 2 + (LOSS::kLogStd ? adim : 0);
  a.part = (float*)(net->ws + net->heads_part_off); a.slab = (nacc + 3) & ~3;
  size_t shb = (size_t)8 * nacc * sizeof(float);
  { cudaError_t ea = ensure_kernel_attrs(); if (ea != cudaSuccess) return fail(XTB_ERR_CUDA, "kernel attributes: %s", cudaGetErrorString(ea)); }
  XLAUNCH(heads_pick(kHeadsKernels<LOSS>, a.K, a.A)->kern, blocks, 256, shb, S(stream), a);
  LAUNCH_CHECK();
  {   // ordered reduction of the per-block slabs (queued; runs with the other partial sums at the end of backward)
    auto seg = [&](int off, int count, long long dst_off, float* dst_ptr = nullptr) {
      queue_reduction(net, a.part + off, blocks, a.slab, count, dst_off, dst_ptr);
    };
    seg(0, HK * adim, lpi.w_off);
    seg(HK * adim, HK, lv.w_off);
    if (bh_pi_ok) seg(HK * adim + HK, HK, net->L[lpi.d.src - 1].b_off);
    if (!a.shared && bh_v_ok) seg(HK * adim + 2 * HK, HK, net->L[lv.d.src - 1].b_off);
    seg(HK * adim + 3 * HK, adim, lpi.b_off);
    seg(HK * adim + 3 * HK + adim, 1, lv.b_off);
    seg(HK * adim + 3 * HK + adim + 1, 1, 0, loss_dst);
    if (LOSS::kLogStd) seg(HK * adim + 3 * HK + adim + 2, adim, ls_off);
  }
  const int32_t srcs[2] = {lpi.d.src, lv.d.src};
  BackwardOpts o(srcs, a.shared ? 1 : 2);
  o.heads_bp = (bp_pi ? (1u << lpi.d.src) : 0u) | (bp_v ? (1u << lv.d.src) : 0u);   // the fused kernel wrote planes there
  o.heads_dy = (ext_pi ? (1u << lpi.d.src) : 0u) | (ext_v ? (1u << lv.d.src) : 0u);
  o.bias_done = (bh_pi_ok ? (1u << lpi.d.src) : 0u) | ((lpi.d.src != lv.d.src && bh_v_ok) ? (1u << lv.d.src) : 0u);
  o.skip = skip; o.zero_grads = false; o.all_reduce = true;
  return net_backward_impl(net, obs, idx, mb, stream, o);
}

// The epoch x minibatch loop of PPO.train for the action distribution DIST.  Under the fused-heads conditions one
// heads_kernel<DIST::Loss> launch per minibatch (a DiagGaussian's log_std gradient is A more slab floats, reduced in
// block order into its slot); otherwise layer by layer: forward, the loss kernel (a DiagGaussian's log_std gradient
// straight into its slot of the zeroed gradient bucket), then the backward pass of the network, which keeps that slot.
template <class DIST>
static int ppo_train_launch(xtb_net* net, xtb_adam* opt, const xtb_ppo_rollout* ro, int N, int B, int E, const int32_t* perm,
                            const xtb_ppo_hyper* hp, int pi_t, int v_t, int ls_t, float* loss_per_step, float inv_world,
                            void* stream) {
  const int32_t heads[2] = {pi_t, v_t};
  const auto* action = static_cast<const typename DIST::Action*>(ro->action);
  const int adim = net->tsize[pi_t];
  const long long ls_off = DIST::kLogStd ? net->L[ls_t - 1].w_off : -1;
  const LayerPlan& lpi = net->L[pi_t - 1];
  const LayerPlan& lv = net->L[v_t - 1];
  const bool fuse = ppo_heads_fusable(net, pi_t, v_t, false);
  const unsigned skip = fuse ? ((1u << (pi_t - 1)) | (1u << (v_t - 1))) : 0u;
  return ppo_epoch_loop(net, opt, N, B, E, perm, loss_per_step, stream, [&](const int32_t* idx, int mb, float* step_loss) -> int {
    // fp32 row-major copies: the hidden tensors the fused heads read, or the head outputs the loss kernel reads
    const unsigned want = fuse ? ((1u << lpi.d.src) | (1u << lv.d.src)) : ((1u << pi_t) | (1u << v_t));
    int rc = net_forward_impl(net, nullptr, ro->obs, idx, mb, stream, skip, want);
    if (rc) return rc;
    if (fuse) {
      PpoHeadsArgs a;
      memset(&a, 0, sizeof a);
      a.idx = idx; a.old_logp = ro->old_logp; a.adv = ro->adv; a.old_v = ro->old_v; a.target_v = ro->target_v;
      if constexpr (DIST::kLogStd) { a.action_f = action; a.log_std = net->params + ls_off; }
      else a.action = action;
      a.logits_out = xtb_net_tensor(net, pi_t); a.v_out = xtb_net_tensor(net, v_t);
      a.hp = PpoHyperDev{hp->clip_ratio, hp->ent_coef, hp->vf_clip, hp->critic_coef}; a.inv_count = inv_world / mb;
      return heads_fused<typename DIST::Loss>(net, ro->obs, a, mb, pi_t, v_t, skip, ls_off, step_loss, stream);
    }
    if constexpr (DIST::kLogStd) {
      CUDA_TRY(cudaMemsetAsync(net->grads, 0, net->n_params * sizeof(float), S(stream)));
      rc = xtb_ppo_gauss_loss_grad(xtb_net_tensor(net, pi_t), xtb_net_tensor(net, v_t), net->params + ls_off, idx, action,
                                   ro->old_logp, ro->adv, ro->old_v, ro->target_v, mb, adim, hp, inv_world / mb,
                                   xtb_net_tensor_grad(net, pi_t), xtb_net_tensor_grad(net, v_t), net->grads + ls_off, step_loss,
                                   stream);
    } else {
      rc = xtb_ppo_loss_grad(xtb_net_tensor(net, pi_t), xtb_net_tensor(net, v_t), idx, action, ro->old_logp, ro->adv,
                             ro->old_v, ro->target_v, mb, adim, hp, inv_world / mb, xtb_net_tensor_grad(net, pi_t),
                             xtb_net_tensor_grad(net, v_t), step_loss, stream);
    }
    if (rc) return rc;
    BackwardOpts o(heads, 2);
    o.zero_grads = !DIST::kLogStd; o.all_reduce = true;   // keep the log_std gradient the loss kernel stored
    return net_backward_impl(net, ro->obs, idx, mb, stream, o);
  });
}

// head tensors of the PPO entry points: pi_t (logits / mean, at most MAX_ADIM wide), v_t (value, 1 wide) and ls_t,
// 0 for Categorical, else the DiagGaussian's logstd layer tensor of the mean's width
static int ppo_heads_check(const char* fn, const xtb_net* net, int pi_t, int v_t, int ls_t) {
  const int nl = (int)net->L.size();
  if (pi_t < 1 || pi_t > nl || v_t < 1 || v_t > nl || net->tsize[v_t] != 1 || net->tsize[pi_t] > MAX_ADIM || ls_t < 0 ||
      ls_t > nl)
    return fail(XTB_ERR_ARG, "%s: bad head tensors", fn);
  if (!ls_t) return XTB_OK;
  const LayerPlan& ls = net->L[ls_t - 1];
  if (ls.d.kind != XTB_LOGSTD || ls.N != net->tsize[pi_t]) return fail(XTB_ERR_ARG, "%s: tensor %d is not a logstd layer of the mean's width", fn, ls_t);
  return XTB_OK;
}

extern "C" int xtb_ppo_train(xtb_net* net, xtb_adam* opt, const xtb_ppo_rollout* ro, int n_sample, int batch_size, int n_epoch,
                             const int32_t* perm, const xtb_ppo_hyper* hp, int pi_t, int v_t, int ls_t, float* loss_per_step,
                             int use_graph, void* stream) {
  const char* fn = "xtb_ppo_train";
  const bool missing = !net || !opt || !ro || !ro->obs || !ro->action || !ro->old_logp || !ro->adv || !ro->old_v || !ro->target_v ||
                       !perm || !hp || !loss_per_step;
  if (int rc = learner_check(fn, missing, net, opt, std::min(batch_size, n_sample), true)) return rc;
  if (n_epoch <= 0) return fail(XTB_ERR_ARG, "%s: bad sizes", fn);
  if (int rc = ppo_heads_check(fn, net, pi_t, v_t, ls_t)) return rc;
  const float inv_world = dp_inv_world();
  return run_graph(capture_key(kPpoTrain, {net, opt}, ro->obs, ro->action, ro->old_logp, ro->adv, ro->old_v, ro->target_v, perm,
                               loss_per_step, n_sample, batch_size, n_epoch, hp->clip_ratio, hp->ent_coef, hp->vf_clip,
                               hp->critic_coef, pi_t, v_t, ls_t),
                   use_graph, stream, [&](void* st) {
    return ls_t ? ppo_train_launch<DiagGaussian>(net, opt, ro, n_sample, batch_size, n_epoch, perm, hp, pi_t, v_t, ls_t,
                                                 loss_per_step, inv_world, st)
                : ppo_train_launch<Categorical>(net, opt, ro, n_sample, batch_size, n_epoch, perm, hp, pi_t, v_t, ls_t,
                                                loss_per_step, inv_world, st);
  });
}

// ------------------------------------------------------------------------------------------
// fused IMPALA / DQN learner steps (graph-captured like xtb_ppo_train; gradients all-reduced when a communicator is set)
// ------------------------------------------------------------------------------------------

// ImpalaCnnOpt.train (xt/model/impala/impala_cnn_opt.py:251-265): forward over n = k * step_len env-major samples,
// V-trace + summed losses (vtrace_kernel), backward, clip + Adam.  With a communicator the losses are sums over the
// GLOBAL batch, so no rescaling: gradients are summed over ranks.  loss_out: device float, accumulated (+=).
extern "C" int xtb_impala_train(xtb_net* net, xtb_adam* opt, const void* obs, const int32_t* gather_idx, const float* bp_logits,
                                const int32_t* action, const uint8_t* done, const float* reward, int n_sample, int step_len,
                                float gamma, int logit_tensor, int base_tensor, float* loss_out, int use_graph, void* stream) {
  const bool missing = !net || !opt || !obs || !bp_logits || !action || !done || !reward || !loss_out;
  if (int rc = learner_check("xtb_impala_train", missing, net, opt, n_sample, true)) return rc;
  const int nl = (int)net->L.size();
  if (logit_tensor < 1 || logit_tensor > nl || base_tensor < 1 || base_tensor > nl || net->tsize[base_tensor] != 1)
    return fail(XTB_ERR_ARG, "xtb_impala_train: bad head tensors");
  if (step_len < 2 || n_sample % step_len) return fail(XTB_ERR_ARG, "xtb_impala_train: bad sizes");
  const int adim = net->tsize[logit_tensor];
  if (adim > MAX_ADIM) return fail(XTB_ERR_ARG, "xtb_impala_train: action dim too large");
  return run_graph(capture_key(kImpalaTrain, {net, opt}, obs, gather_idx, bp_logits, action, done, reward, loss_out,
                               n_sample, step_len, gamma, logit_tensor, base_tensor),
                   use_graph, stream, [&](void* st) -> int {
    int rc = net_forward_impl(net, nullptr, obs, gather_idx, n_sample, st, 0u, (1u << logit_tensor) | (1u << base_tensor));
    if (rc) return rc;
    rc = xtb_vtrace_loss_grad(xtb_net_tensor(net, logit_tensor), xtb_net_tensor(net, base_tensor), bp_logits, action, done, reward,
                              n_sample / step_len, step_len, adim, gamma, xtb_net_tensor_grad(net, logit_tensor),
                              xtb_net_tensor_grad(net, base_tensor), nullptr, nullptr, loss_out, st);
    if (rc) return rc;
    const int32_t heads[2] = {logit_tensor, base_tensor};
    BackwardOpts o(heads, 2); o.all_reduce = true;
    rc = net_backward_impl(net, obs, gather_idx, n_sample, st, o);
    if (rc) return rc;
    return xtb_adam_step_net(opt, net, 1.f, st);
  });
}

// ---- IMPALA with the Keras learner (xt/algorithm/impala/impala.py, xt/model/impala/impala_mlp.py, impala_cnn.py) --------
// One Keras fit epoch (training_arrays.fit_loop, batch_size = fit_batch, shuffle = True) over n rows in a given order:
// minibatch k holds rows row_idx[k*fit_batch ...] (observation rows obs_idx[...]); per minibatch forward, the Keras
// loss (impala_keras_loss_kernel, ragged last batch included), backward and the optimiser step.  *loss_out = the
// epoch loss Keras reports: sum over the rows of the per-row loss / n.
static int keras_fit_launch(xtb_net* net, xtb_adam* opt, const void* obs, const int32_t* obs_idx, const int32_t* row_idx,
                            const float* y, const float* adv, const float* tv, int n, int fit_batch, int lt, int vt, float ent,
                            float* loss_out, void* stream) {
  CUDA_TRY(cudaMemsetAsync(loss_out, 0, sizeof(float), S(stream)));
  const int adim = net->tsize[lt];
  const int32_t heads[2] = {lt, vt};
  for (int s0 = 0; s0 < n; s0 += fit_batch) {
    const int mb = std::min(fit_batch, n - s0);
    int rc = net_forward_impl(net, nullptr, obs, obs_idx + s0, mb, stream, 0u, (1u << lt) | (1u << vt));
    if (rc) return rc;
    rc = xtb_impala_keras_loss_grad(xtb_net_tensor(net, lt), xtb_net_tensor(net, vt), row_idx + s0, y, adv, tv, mb, adim, ent,
                                    0.5f, 1.f / n, xtb_net_tensor_grad(net, lt), xtb_net_tensor_grad(net, vt), loss_out, stream);
    if (rc) return rc;
    rc = net_backward_impl(net, obs, obs_idx + s0, mb, stream, BackwardOpts(heads, 2));
    if (rc) return rc;
    rc = xtb_adam_step_net(opt, net, 1.f, stream);
    if (rc) return rc;
  }
  return XTB_OK;
}

// head tensors of both IMPALA-Keras entry points: logits (at most MAX_ADIM wide) and value (1 wide)
static int keras_heads_check(const char* fn, xtb_net* net, int lt, int vt) {
  const int nl = (int)net->L.size();
  if (lt < 1 || lt > nl || vt < 1 || vt > nl || lt == vt || net->tsize[vt] != 1) return fail(XTB_ERR_ARG, "%s: bad head tensors", fn);
  if (net->tsize[lt] > MAX_ADIM) return fail(XTB_ERR_ARG, "%s: action dim %d > %d", fn, net->tsize[lt], MAX_ADIM);
  return XTB_OK;
}

extern "C" int xtb_impala_keras_fit(xtb_net* net, xtb_adam* opt, const void* obs, const int32_t* order, const float* action_mat,
                                    const float* adv, const float* target_v, int n, int fit_batch, int logit_tensor, int v_tensor,
                                    float ent_coef, float* loss_out, int use_graph, void* stream) {
  const char* fn = "xtb_impala_keras_fit";
  const bool missing = !net || !opt || !obs || !order || !action_mat || !adv || !target_v || !loss_out;
  if (int rc = learner_check(fn, missing, net, opt, std::min(n, fit_batch), false)) return rc;
  if (int rc = keras_heads_check(fn, net, logit_tensor, v_tensor)) return rc;
  return run_graph(capture_key(kImpalaKerasFit, {net, opt}, obs, order, action_mat, adv, target_v, n, fit_batch, logit_tensor,
                               v_tensor, ent_coef, loss_out),
                   use_graph, stream, [&](void* st) {
    return keras_fit_launch(net, opt, obs, order, order, action_mat, adv, target_v, n, fit_batch, logit_tensor, v_tensor, ent_coef,
                            loss_out, st);
  });
}

extern "C" int xtb_impala_keras_train(xtb_net* net, xtb_adam* opt, const xtb_impala_traj* tr, int n_traj, int ep_len, int slice,
                                      int fit_batch, const int32_t* order, int32_t* obs_idx, float gamma, float ent_coef,
                                      int logit_tensor, int v_tensor, float* pg_adv, float* target_v, float* loss_per_slice,
                                      int use_graph, void* stream) {
  const char* fn = "xtb_impala_keras_train";
  const bool missing = !net || !opt || !tr || !tr->obs || !tr->behav_prob || !tr->action_mat || !tr->reward || !tr->done || !order ||
                       !obs_idx || !pg_adv || !target_v || !loss_per_slice;
  const long long n_state = (long long)n_traj * (ep_len + 1), n_train = (long long)n_traj * ep_len;
  if (int rc = learner_check(fn, missing, net, opt, n_state, false)) return rc;
  if (int rc = keras_heads_check(fn, net, logit_tensor, v_tensor)) return rc;
  if (n_traj <= 0 || ep_len <= 0 || slice <= 0 || fit_batch <= 0) return fail(XTB_ERR_ARG, "%s: bad sizes", fn);
  const xtb_impala_traj t = *tr;
  return run_graph(capture_key(kImpalaKerasTrain, {net, opt}, t.obs, t.behav_prob, t.action_mat, t.reward, t.done, n_traj,
                               ep_len, slice, fit_batch, order, obs_idx, gamma, ent_coef, logit_tensor, v_tensor, pg_adv, target_v,
                               loss_per_slice),
                   use_graph, stream, [&](void* st) -> int {
    // 1. target probabilities and values of every state with the weights before this call's updates
    int rc = net_forward_impl(net, nullptr, t.obs, nullptr, (int)n_state, st, 0u, (1u << logit_tensor) | (1u << v_tensor));
    if (rc) return rc;
    // 2. V-trace into pg_adv / target_v
    XLAUNCH(impala_keras_vtrace_kernel, (n_traj * 32 + 127) / 128, 128, 0, S(st), (const float*)xtb_net_tensor(net, logit_tensor),
            (const float*)xtb_net_tensor(net, v_tensor), t.behav_prob, t.action_mat, t.reward, t.done, n_traj, ep_len,
            net->tsize[logit_tensor], gamma, pg_adv, target_v);
    LAUNCH_CHECK();
    // 3. observation row of every training row of the shuffled slices
    XLAUNCH(impala_keras_rows_kernel, (unsigned)((n_train + 255) / 256), 256, 0, S(st), order, (int)n_train, ep_len, obs_idx);
    LAUNCH_CHECK();
    // 4. one Keras fit per BATCH_SIZE slice, in order
    for (long long s0 = 0, k = 0; s0 < n_train; s0 += slice, k++) {
      const int n = (int)std::min<long long>(slice, n_train - s0);
      rc = keras_fit_launch(net, opt, t.obs, obs_idx + s0, order + s0, t.action_mat, pg_adv, target_v, n, fit_batch, logit_tensor,
                            v_tensor, ent_coef, loss_per_slice + k, st);
      if (rc) return rc;
    }
    return XTB_OK;
  });
}

// ---- MuZero (xt/model/muzero/muzero_model.py:103-140, 154-239) -------------------------------------------------------
// The three networks (representation, dynamics, prediction) are separate xtb_nets bound to consecutive slices of one
// parameter buffer and one gradient buffer (the Keras list order of MuzeroBase); the dynamics net's own gradient buffer
// is scratch that each of its K applications fills before it is added to its slice.  The object owns the step's
// device scratch, sized for max_batch samples.
struct xtb_muzero {
  xtb_net *rep = nullptr, *dyn = nullptr, *pred = nullptr;
  xtb_muzero_desc d{};
  int max_batch = 0, K = 0, H = 0, A = 0, Sv = 0, Sr = 0, n_part = 0;
  int act_rep = 0, act_dyn = 0;
  long long n_params = 0;      // floats of the shared parameter buffer
  float* buf = nullptr;
  float *hbuf = nullptr, *xbuf = nullptr, *rlog = nullptr, *dr = nullptr, *tv = nullptr, *tr = nullptr, *dh = nullptr,
        *dx = nullptr, *part = nullptr;
};
static inline int mz_blocks(long long rows) { return (int)((rows + MZ_THREADS / 32 - 1) / (MZ_THREADS / 32)); }

extern "C" int xtb_muzero_create(xtb_net* rep, xtb_net* dyn, xtb_net* pred, const xtb_muzero_desc* desc, int max_batch,
                                 xtb_muzero** out) {
  if (!rep || !dyn || !pred || !desc || !out) return fail(XTB_ERR_ARG, "xtb_muzero_create: null pointer");
  for (xtb_net* n : {rep, dyn, pred})
    if (!n->ws || !n->params || !n->grads) return fail(XTB_ERR_STATE, "xtb_muzero_create: every net must be bound");
  const xtb_muzero_desc& d = *desc;
  const int K = d.unroll;
  if (K < 1 || max_batch < 1) return fail(XTB_ERR_ARG, "xtb_muzero_create: unroll %d / max_batch %d out of range", K, max_batch);
  auto bad_t = [](const xtb_net* n, int t) { return t < 1 || t >= (int)n->tsize.size() || n->tsize[t] == 0; };
  if (bad_t(rep, d.rep_h) || bad_t(dyn, d.dyn_h) || bad_t(dyn, d.dyn_r) || bad_t(pred, d.pred_p) || bad_t(pred, d.pred_v) ||
      d.dyn_h == d.dyn_r || d.pred_p == d.pred_v)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: bad tensor ids");
  const int H = rep->tsize[d.rep_h], A = pred->tsize[d.pred_p], Sv = pred->tsize[d.pred_v], Sr = dyn->tsize[d.dyn_r];
  if (dyn->tsize[d.dyn_h] != H || dyn->tsize[0] != H + A || pred->tsize[0] != H)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: widths disagree (hidden %d, actions %d, dynamics input %d, prediction input %d)", H,
                A, dyn->tsize[0], pred->tsize[0]);
  if (A > MZ_MAX_SUPPORT || Sv > MZ_MAX_SUPPORT || Sr > MZ_MAX_SUPPORT)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: a support or the action count exceeds %d", MZ_MAX_SUPPORT);
  if (!(d.value_max > d.value_min) || !(d.reward_max > d.reward_min)) return fail(XTB_ERR_ARG, "xtb_muzero_create: empty value range");
  for (const xtb_net* n : {dyn, pred}) if (int rc = input_grad_check(n)) return rc;
  const int act_rep = rep->L[d.rep_h - 1].d.act, act_dyn = dyn->L[d.dyn_h - 1].d.act;
  if (act_is_ext(act_rep) || act_is_ext(act_dyn)) return fail(XTB_ERR_ARG, "xtb_muzero_create: hidden states must be relu / tanh / linear");
  for (int t : {d.pred_p, d.pred_v}) if (pred->L[t - 1].d.act != XTB_ACT_NONE || pred->L[t - 1].d.kind != XTB_DENSE)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: policy and value heads must be linear dense layers");
  if (dyn->L[d.dyn_r - 1].d.act != XTB_ACT_NONE || dyn->L[d.dyn_r - 1].d.kind != XTB_DENSE)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: the reward head must be a linear dense layer");
  if (rep->max_batch < max_batch || dyn->max_batch < max_batch || (long long)pred->max_batch < (long long)(K + 1) * max_batch)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: nets hold fewer rows than max_batch (prediction: (unroll + 1) * max_batch)");
  // one parameter buffer [rep | dyn | pred] and one gradient buffer with the same layout; dyn's bound gradients lie outside
  float* g0 = rep->grads;
  const long long o_dyn = dyn->params - rep->params, o_pred = pred->params - rep->params, total = o_pred + pred->n_params;
  if (o_dyn < rep->n_params || o_pred < o_dyn + dyn->n_params || pred->grads != g0 + o_pred)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: nets must be bound to slices [rep | dyn | pred] of one buffer, in order");
  if (dyn->grads + dyn->n_params > g0 && dyn->grads < g0 + total)
    return fail(XTB_ERR_ARG, "xtb_muzero_create: the dynamics net's gradient scratch overlaps the shared gradient buffer");
  auto* m = new xtb_muzero();
  m->rep = rep; m->dyn = dyn; m->pred = pred; m->d = d; m->max_batch = max_batch;
  m->K = K; m->H = H; m->A = A; m->Sv = Sv; m->Sr = Sr; m->act_rep = act_rep; m->act_dyn = act_dyn; m->n_params = total;
  const long long Bm = max_batch, R1 = (long long)(K + 1) * Bm, RK = (long long)K * Bm;
  m->n_part = 2 * mz_blocks(R1) + mz_blocks(RK);
  const long long sizes[] = {R1 * H, RK * (H + A), RK * Sr, RK * Sr, R1 * Sv, RK * Sr, R1 * H, Bm * (H + A), m->n_part};
  float** dst[] = {&m->hbuf, &m->xbuf, &m->rlog, &m->dr, &m->tv, &m->tr, &m->dh, &m->dx, &m->part};
  long long tot = 0;
  for (long long n : sizes) tot += (n + 63) / 64 * 64;
  cudaError_t e = cudaMalloc(&m->buf, tot * sizeof(float));
  if (e != cudaSuccess) { delete m; return fail(XTB_ERR_NOMEM, "xtb_muzero_create: %s", cudaGetErrorString(e)); }
  e = cudaMemset(m->buf, 0, tot * sizeof(float));
  if (e != cudaSuccess) { cudaFree(m->buf); delete m; return fail(XTB_ERR_CUDA, "xtb_muzero_create: %s", cudaGetErrorString(e)); }
  float* p = m->buf;
  for (int i = 0; i < 9; i++) { *dst[i] = p; p += (sizes[i] + 63) / 64 * 64; }
  *out = m;
  return XTB_OK;
}

extern "C" void xtb_muzero_destroy(xtb_muzero* m) {
  if (!m) return;
  drop_graphs_of(m);
  cudaDeviceSynchronize();
  cudaFree(m->buf);
  delete m;
}

// the learner checks of a MuZero entry point (opt NULL: an inference call) over its object's nets and batch limit
static int mz_check(const char* fn, const xtb_muzero* m, bool missing, const xtb_adam* opt, int batch) {
  if (!m) return fail(XTB_ERR_ARG, "%s: null object", fn);
  return learner_check(fn, missing, m->rep, opt, batch, false, m->max_batch, m->n_params);
}

// prediction forward over `rows` hidden states (rows of m->hbuf), then softmax policy / value expectation if asked
static int mz_predict(xtb_muzero* m, const float* hidden, int rows, float* value_out, float* policy_out, cudaStream_t st) {
  const xtb_muzero_desc& d = m->d;
  int rc = net_forward_impl(m->pred, nullptr, hidden, nullptr, rows, st, 0u, (1u << d.pred_p) | (1u << d.pred_v));
  if (rc) return rc;
  if (value_out) {
    XLAUNCH(mz_support_value_kernel, mz_blocks(rows), MZ_THREADS, 0, st, (const float*)xtb_net_tensor(m->pred, d.pred_v), rows, m->Sv,
            d.value_min, d.value_max, value_out);
    LAUNCH_CHECK();
  }
  if (policy_out) {
    XLAUNCH(softmax_rows_kernel, (rows + 127) / 128, 128, 0, st, (const float*)xtb_net_tensor(m->pred, d.pred_p), rows, m->A, policy_out);
    LAUNCH_CHECK();
  }
  return XTB_OK;
}

// initial_inference / value_inference: representation then prediction
static int mz_initial_launch(xtb_muzero* m, const void* obs, int B, float* hidden_out, float* value_out, float* policy_out,
                             cudaStream_t st) {
  int rc = net_forward_impl(m->rep, nullptr, obs, nullptr, B, st, 0u, 1u << m->d.rep_h);
  if (rc) return rc;
  const float* h = xtb_net_tensor(m->rep, m->d.rep_h);
  if (hidden_out) CUDA_TRY(cudaMemcpyAsync(hidden_out, h, (size_t)B * m->H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return mz_predict(m, h, B, value_out, policy_out, st);
}

extern "C" int xtb_muzero_initial_inference(xtb_muzero* m, const void* obs, int batch, float* hidden_out, float* value_out,
                                            float* policy_out, int use_graph, void* stream) {
  if (int rc = mz_check("xtb_muzero_initial_inference", m, !obs, nullptr, batch)) return rc;
  return run_graph(capture_key(kMuzeroInitInfer, {m->rep, m->dyn, m->pred, m}, m, obs, batch, hidden_out, value_out, policy_out),
                   use_graph, stream, [&](void* st) { return mz_initial_launch(m, obs, batch, hidden_out, value_out, policy_out, S(st)); });
}

// recurrent_inference after its input concat(hidden, one_hot(action)) is in m->xbuf: dynamics then prediction
static int mz_dynamics_launch(xtb_muzero* m, int batch, float* hidden_out, float* reward_out, float* value_out, float* policy_out,
                              cudaStream_t st) {
  const xtb_muzero_desc& d = m->d;
  int rc = net_forward_impl(m->dyn, nullptr, m->xbuf, nullptr, batch, st, 0u, (1u << d.dyn_h) | (1u << d.dyn_r));
  if (rc) return rc;
  const float* h = xtb_net_tensor(m->dyn, d.dyn_h);
  if (hidden_out) CUDA_TRY(cudaMemcpyAsync(hidden_out, h, (size_t)batch * m->H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (reward_out) {
    XLAUNCH(mz_support_value_kernel, mz_blocks(batch), MZ_THREADS, 0, st, (const float*)xtb_net_tensor(m->dyn, d.dyn_r), batch, m->Sr,
            d.reward_min, d.reward_max, reward_out);
    LAUNCH_CHECK();
  }
  return mz_predict(m, h, batch, value_out, policy_out, st);
}

extern "C" int xtb_muzero_recurrent_inference(xtb_muzero* m, const float* hidden, const int32_t* action, int batch, float* hidden_out,
                                              float* reward_out, float* value_out, float* policy_out, int use_graph, void* stream) {
  if (int rc = mz_check("xtb_muzero_recurrent_inference", m, !hidden || !action, nullptr, batch)) return rc;
  return run_graph(capture_key(kMuzeroRecurInfer, {m->rep, m->dyn, m->pred, m}, m, hidden, action, batch, hidden_out, reward_out,
                               value_out, policy_out),
                   use_graph, stream, [&](void* sv) -> int {
    cudaStream_t st = S(sv);
    const int H = m->H, A = m->A;
    XLAUNCH(mz_concat_onehot_kernel, std::min(4 * kSMs, (batch * (H + A) + 255) / 256), 256, 0, st, hidden, batch, H, action, 1, 0, A, m->xbuf);
    LAUNCH_CHECK();
    return mz_dynamics_launch(m, batch, hidden_out, reward_out, value_out, policy_out, st);
  });
}

// ---- MuZero tree search (xt/agent/muzero/mcts.py) ---------------------------------------------------------------------
// The device state of up to max_envs trees of up to 1 + max_simulations expanded nodes (MctsTrees), plus the float
// outputs of the inference calls the search makes.
struct xtb_muzero_tree {
  MctsTrees t{};
  int max_sims = 0;
  void* buf = nullptr;
  float *reward = nullptr, *value = nullptr, *policy = nullptr;   // [E], [E], [E, A]
};

extern "C" int xtb_muzero_tree_create(const xtb_muzero* m, int max_envs, int max_simulations, xtb_muzero_tree** out) {
  if (!m || !out) return fail(XTB_ERR_ARG, "xtb_muzero_tree_create: null pointer");
  if (max_envs < 1 || max_simulations < 1 || max_simulations > (1 << 20))
    return fail(XTB_ERR_ARG, "xtb_muzero_tree_create: max_envs %d / max_simulations %d out of range", max_envs, max_simulations);
  const long long E = max_envs, NN = max_simulations + 1, A = m->A, H = m->H;
  // byte sizes, in the order of `dst` below; each piece starts 256-byte aligned
  const long long sizes[] = {NN * E * H * 4, E * NN * 8, E * NN * A * 8, E * NN * A * 8, E * NN * A * 4, E * NN * A * 4, E * 8, E * 4,
                             E * 2 * 8, E * NN * 4, E * NN * 4, E * 4, E * 4, E * 4, E * A * 4};
  auto* tr = new xtb_muzero_tree();
  MctsTrees& t = tr->t;
  void** dst[] = {(void**)&t.hid, (void**)&t.reward, (void**)&t.prior, (void**)&t.vsum, (void**)&t.visits, (void**)&t.child,
                  (void**)&t.root_vsum, (void**)&t.root_visits, (void**)&t.minmax, (void**)&t.path_node, (void**)&t.path_act,
                  (void**)&t.depth, (void**)&tr->reward, (void**)&tr->value, (void**)&tr->policy};
  long long tot = 0;
  for (long long n : sizes) tot += align_up(n, 256);
  cudaError_t e = cudaMalloc(&tr->buf, tot);
  if (e != cudaSuccess) { delete tr; return fail(XTB_ERR_NOMEM, "xtb_muzero_tree_create: %s", cudaGetErrorString(e)); }
  char* p = (char*)tr->buf;
  for (int i = 0; i < 15; i++) { *dst[i] = p; p += align_up(sizes[i], 256); }
  t.E = max_envs; t.NN = (int)NN; t.A = (int)A; t.H = (int)H;
  tr->max_sims = max_simulations;
  *out = tr;
  return XTB_OK;
}

extern "C" void xtb_muzero_tree_destroy(xtb_muzero_tree* tr) {
  if (!tr) return;
  drop_graphs_of(tr);
  cudaDeviceSynchronize();
  cudaFree(tr->buf);
  delete tr;
}

extern "C" int xtb_muzero_search(xtb_muzero* m, xtb_muzero_tree* tr, const void* obs, int n_envs, int num_simulations,
                                 const double* noise, double pb_c_base, double pb_c_init, double discount, double exploration_frac,
                                 int32_t* visit_counts_out, double* root_value_out, int use_graph, void* stream) {
  const char* fn = "xtb_muzero_search";
  if (int rc = mz_check(fn, m, !tr || !obs || !visit_counts_out || !root_value_out, nullptr, n_envs)) return rc;
  if (tr->t.A != m->A || tr->t.H != m->H)
    return fail(XTB_ERR_ARG, "%s: tree made for %d actions / hidden width %d, model has %d / %d", fn, tr->t.A, tr->t.H, m->A, m->H);
  if (n_envs > tr->t.E) return fail(XTB_ERR_ARG, "%s: %d environments, the tree holds %d", fn, n_envs, tr->t.E);
  if (num_simulations < 1 || num_simulations > tr->max_sims)
    return fail(XTB_ERR_ARG, "%s: num_simulations %d not in [1, %d]", fn, num_simulations, tr->max_sims);
  if (!std::isfinite(pb_c_base) || !(pb_c_base > 0)) return fail(XTB_ERR_ARG, "%s: pb_c_base %g is not finite and positive", fn, pb_c_base);
  return run_graph(capture_key(kMuzeroSearch, {m->rep, m->dyn, m->pred, m, tr}, m, tr, obs, n_envs, num_simulations, noise, pb_c_base,
                               pb_c_init, discount, exploration_frac, visit_counts_out, root_value_out),
                   use_graph, stream, [&](void* sv) -> int {
    cudaStream_t st = S(sv);
    const MctsTrees& t = tr->t;
    const int N = n_envs, blocks = (N + MCTS_THREADS / 32 - 1) / (MCTS_THREADS / 32);
    const size_t rows = (size_t)t.E * t.H;   // floats of one node's block of hidden rows
    int rc = mz_initial_launch(m, obs, N, t.hid, nullptr, tr->policy, st);
    if (rc) return rc;
    XLAUNCH(mcts_root_kernel, blocks, MCTS_THREADS, 0, st, t, N, (const float*)tr->policy, noise, exploration_frac);
    LAUNCH_CHECK();
    for (int s = 1; s <= num_simulations; s++) {
      XLAUNCH(mcts_select_kernel, blocks, MCTS_THREADS, 0, st, t, N, pb_c_base, pb_c_init, m->xbuf);
      LAUNCH_CHECK();
      rc = mz_dynamics_launch(m, N, t.hid + s * rows, tr->reward, tr->value, tr->policy, st);
      if (rc) return rc;
      XLAUNCH(mcts_expand_backup_kernel, blocks, MCTS_THREADS, 0, st, t, N, s, (const float*)tr->reward, (const float*)tr->value,
              (const float*)tr->policy, discount);
      LAUNCH_CHECK();
    }
    XLAUNCH(mcts_result_kernel, blocks, MCTS_THREADS, 0, st, t, N, visit_counts_out, root_value_out);
    LAUNCH_CHECK();
    return XTB_OK;
  });
}

// MuzeroModel.train (muzero_model.py:103-140, 154-169) over B samples
static int mz_train_launch(xtb_muzero* m, xtb_adam* opt, const xtb_muzero_batch& bt, int B, float loss_offset, float* loss_out,
                           float* value_out, cudaStream_t st) {
  const xtb_muzero_desc& d = m->d;
  const int K = m->K, H = m->H, A = m->A, Sv = m->Sv, Sr = m->Sr, X = H + A;
  const int R1 = (K + 1) * B, RK = K * B;
  xtb_net *rep = m->rep, *dyn = m->dyn, *pred = m->pred;
  const unsigned dyn_out = (1u << d.dyn_h) | (1u << d.dyn_r);
  const int ew_blocks = std::min(4 * kSMs, (B * X + 255) / 256);
  // two-hot targets: value rows step-major [K+1][B], reward rows [K][B] (the last reward target is not used)
  XLAUNCH(mz_support_project_kernel, mz_blocks(R1), MZ_THREADS, 0, st, bt.target_value, R1, B, K + 1, Sv, d.value_min, d.value_max, m->tv);
  LAUNCH_CHECK();
  XLAUNCH(mz_support_project_kernel, mz_blocks(RK), MZ_THREADS, 0, st, bt.target_reward, RK, B, K + 1, Sr, d.reward_min, d.reward_max, m->tr);
  LAUNCH_CHECK();
  // h_0 = representation(obs); h_{k+1}, r_k = dynamics(concat(h_k, one_hot(a_k)))
  int rc = net_forward_impl(rep, nullptr, bt.obs, nullptr, B, st, 0u, 1u << d.rep_h);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(m->hbuf, xtb_net_tensor(rep, d.rep_h), (size_t)B * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  for (int k = 0; k < K; k++) {
    float* xk = m->xbuf + (size_t)k * B * X;
    XLAUNCH(mz_concat_onehot_kernel, ew_blocks, 256, 0, st, (const float*)(m->hbuf + (size_t)k * B * H), B, H, bt.action, K, k, A, xk);
    LAUNCH_CHECK();
    rc = net_forward_impl(dyn, nullptr, xk, nullptr, B, st, 0u, dyn_out);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(m->hbuf + (size_t)(k + 1) * B * H, xtb_net_tensor(dyn, d.dyn_h), (size_t)B * H * sizeof(float),
                             cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(m->rlog + (size_t)k * B * Sr, xtb_net_tensor(dyn, d.dyn_r), (size_t)B * Sr * sizeof(float),
                             cudaMemcpyDeviceToDevice, st));
  }
  // the K+1 prediction applications as one forward over (K+1) B rows
  rc = net_forward_impl(pred, nullptr, m->hbuf, nullptr, R1, st, 0u, (1u << d.pred_p) | (1u << d.pred_v));
  if (rc) return rc;
  // losses: rows of h_0 at gradient scale 1, the unrolled terms at 1/K
  const float gk = 1.f / K;
  const int n1 = mz_blocks(R1);
  XLAUNCH(mz_support_ce_kernel, n1, MZ_THREADS, 0, st, (const float*)xtb_net_tensor(pred, d.pred_p), R1, A, bt.target_policy, B, K + 1, B,
          gk, 1.f / ((float)B * A), xtb_net_tensor_grad(pred, d.pred_p), m->part);
  LAUNCH_CHECK();
  XLAUNCH(mz_support_ce_kernel, n1, MZ_THREADS, 0, st, (const float*)xtb_net_tensor(pred, d.pred_v), R1, Sv, (const float*)m->tv, B, 0, B,
          gk, 1.f / ((float)B * Sv), xtb_net_tensor_grad(pred, d.pred_v), m->part + n1);
  LAUNCH_CHECK();
  XLAUNCH(mz_support_ce_kernel, mz_blocks(RK), MZ_THREADS, 0, st, (const float*)m->rlog, RK, Sr, (const float*)m->tr, B, 0, 0, gk,
          1.f / ((float)B * Sr), m->dr, m->part + 2 * n1);
  LAUNCH_CHECK();
  XLAUNCH(mz_ordered_sum_kernel, 1, MZ_THREADS, 0, st, (const float*)m->part, 2 * n1 + mz_blocks(RK), loss_offset, loss_out);
  LAUNCH_CHECK();
  // backward: prediction (with d loss / d h_i for every i), the dynamics steps newest first, the representation
  const int32_t pheads[2] = {d.pred_p, d.pred_v}, dheads[2] = {d.dyn_h, d.dyn_r}, rheads[1] = {d.rep_h};
  BackwardOpts po(pheads, 2), dopt(dheads, 2);
  po.dobs = m->dh; dopt.dobs = m->dx;
  rc = net_backward_impl(pred, m->hbuf, nullptr, R1, st, po);
  if (rc) return rc;
  float* gdyn = rep->grads + (dyn->params - rep->params);
  CUDA_TRY(cudaMemsetAsync(gdyn, 0, dyn->n_params * sizeof(float), st));
  for (int k = K - 1; k >= 0; k--) {
    const float* xk = m->xbuf + (size_t)k * B * X;
    if (k < K - 1) { rc = net_forward_impl(dyn, nullptr, xk, nullptr, B, st, 0u, dyn_out); if (rc) return rc; }   // recompute step k
    // d h_{k+1}: prediction + 0.5 x the input gradient of step k+1 (scale_gradient(hidden, 0.5))
    XLAUNCH(mz_hidden_grad_kernel, ew_blocks, 256, 0, st, (const float*)(m->dh + (size_t)(k + 1) * B * H),
            (const float*)(k + 1 < K ? m->dx : nullptr), X, 0.5f, (const float*)xtb_net_tensor(dyn, d.dyn_h), m->act_dyn, B, H,
            xtb_net_tensor_grad(dyn, d.dyn_h));
    LAUNCH_CHECK();
    CUDA_TRY(cudaMemcpyAsync(xtb_net_tensor_grad(dyn, d.dyn_r), m->dr + (size_t)k * B * Sr, (size_t)B * Sr * sizeof(float),
                             cudaMemcpyDeviceToDevice, st));
    rc = net_backward_impl(dyn, xk, nullptr, B, st, dopt);
    if (rc) return rc;
    XLAUNCH(mz_accumulate_kernel, std::min(4 * kSMs, (int)((dyn->n_params + 255) / 256)), 256, 0, st, gdyn, (const float*)dyn->grads,
            dyn->n_params);
    LAUNCH_CHECK();
  }
  // d h_0: prediction + the full input gradient of step 0 (h_0 is not scaled)
  XLAUNCH(mz_hidden_grad_kernel, ew_blocks, 256, 0, st, (const float*)m->dh, (const float*)m->dx, X, 1.f,
          (const float*)xtb_net_tensor(rep, d.rep_h), m->act_rep, B, H, xtb_net_tensor_grad(rep, d.rep_h));
  LAUNCH_CHECK();
  rc = net_backward_impl(rep, bt.obs, nullptr, B, st, BackwardOpts(rheads, 1));
  if (rc) return rc;
  // AdamOptimizer(LR).minimize over the whole buffer, then the weight blobs of the three nets
  rc = adam_step_impl(opt, rep->params, rep->grads, 1.f, st, nullptr);
  for (xtb_net* n : {rep, dyn, pred}) if (!rc) rc = xtb_net_sync_weights(n, st);
  if (rc || !value_out) return rc;
  // post-update value_inference of the batch (the learner's new priorities)
  return mz_initial_launch(m, bt.obs, B, nullptr, value_out, nullptr, st);
}

extern "C" int xtb_muzero_train(xtb_muzero* m, xtb_adam* opt, const xtb_muzero_batch* batch_in, int batch, float loss_offset,
                                float* loss_out, float* value_out, int use_graph, void* stream) {
  const bool missing = !opt || !batch_in || !loss_out || !batch_in->obs || !batch_in->action || !batch_in->target_value ||
                       !batch_in->target_reward || !batch_in->target_policy;
  if (int rc = mz_check("xtb_muzero_train", m, missing, opt, batch)) return rc;
  const xtb_muzero_batch bt = *batch_in;
  if (bt.unroll != m->K) return fail(XTB_ERR_ARG, "xtb_muzero_train: batch unroll %d != model unroll %d", bt.unroll, m->K);
  return run_graph(capture_key(kMuzeroTrain, {m->rep, m->dyn, m->pred, m, opt}, m, bt.obs, bt.action, bt.target_value,
                               bt.target_reward, bt.target_policy, batch, loss_offset, loss_out, value_out),
                   use_graph, stream, [&](void* st) { return mz_train_launch(m, opt, bt, batch, loss_offset, loss_out, value_out, S(st)); });
}

// Dueling head that the fused TD step covers: q_tensor combines two linear dense layers that read the same hidden
// (non-observation) tensor, within the heads_kernel limits, and the fused-heads mode is on.
static bool dueling_fusable(const xtb_net* net, int q_tensor) {
  const LayerPlan& lq = net->L[q_tensor - 1];
  if (!g_fuse_heads || lq.d.kind != XTB_DUELING) return false;
  const LayerPlan& lv = net->L[lq.d.src - 1];
  const LayerPlan& la = net->L[lq.d.k - 1];
  return lv.d.kind == XTB_DENSE && la.d.kind == XTB_DENSE && lv.d.act == 0 && la.d.act == 0 && lv.d.src != 0 &&
         lv.d.src == la.d.src && heads_fit(lv.K, lv.N) && !act_is_ext(lv.src_act);
}

// The online half of the dueling TD step in one heads_kernel launch (heads_fused with the value stream as the pi head
// and the adv stream as the value head): both streams' forward, the combine, TD target and loss, the streams' backward
// and the gradient wrt the hidden tensor; then the backward pass of the layers below.
static int dueling_td_fused(xtb_net* net, const void* obs, const int32_t* idx, const int32_t* action, const float* reward,
                            const uint8_t* done, const float* disc, int n, float gamma, float huber, int q_tensor,
                            const float* qn_t, const float* qn_o, float inv_count, float* loss_out, cudaStream_t st) {
  const LayerPlan& lq = net->L[q_tensor - 1];
  const int h = net->L[lq.d.src - 1].d.src;
  const unsigned skip = (1u << (q_tensor - 1)) | (1u << (lq.d.src - 1)) | (1u << (lq.d.k - 1));
  int rc = net_forward_impl(net, nullptr, obs, idx, n, st, skip, 1u << h);
  if (rc) return rc;
  PpoHeadsArgs a;
  memset(&a, 0, sizeof a);
  a.idx = idx; a.action = action; a.reward = reward; a.done = done; a.disc = disc; a.qn_t = qn_t; a.qn_o = qn_o; a.loss_in = loss_out;
  a.gamma = gamma; a.huber = huber; a.inv_count = inv_count;
  return heads_fused<DuelingTdLoss>(net, obs, a, n, lq.d.src, lq.d.k, skip, -1, loss_out, st);
}

// DQN.train (xt/algorithm/dqn/dqn.py:61-103) on a device replay ring: rows idx[0..n) of (obs, next_obs, action, reward,
// done[, disc]); target-network forward on s', optional double-DQN online forward on s', online forward on s, TD target +
// loss gradient, backward, clip + Adam.  qn_t / qn_o: scratch [n, adim] (qn_o NULL = plain DQN).  Reference mode:
// disc = NULL, huber_delta = 0.  With a communicator every rank holds n of world*n samples: inv_count = 1/(world*n*adim).
extern "C" int xtb_dqn_train(xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                             const int32_t* idx, const int32_t* action, const float* reward, const uint8_t* done,
                             const float* disc, int n_sample, float gamma, float huber_delta, int q_tensor, float* qn_t,
                             float* qn_o, float* loss_out, int use_graph, void* stream) {
  const bool missing = !net || !target || !opt || !obs || !next_obs || !action || !reward || !done || !qn_t || !loss_out;
  if (int rc = learner_check("xtb_dqn_train", missing, net, opt, n_sample, true)) return rc;
  if (!target->ws) return fail(XTB_ERR_STATE, "xtb_dqn_train: target net not bound");
  const int nl = (int)net->L.size();
  if (q_tensor < 1 || q_tensor > nl || (int)target->L.size() != nl) return fail(XTB_ERR_ARG, "xtb_dqn_train: bad head tensor");
  if (n_sample > target->max_batch) return fail(XTB_ERR_ARG, "xtb_dqn_train: batch exceeds the target net's max_batch");
  const int adim = net->tsize[q_tensor];
  const float inv_world = dp_inv_world();
  const bool fuse = dueling_fusable(net, q_tensor);
  return run_graph(capture_key(kDqnTrain, {net, target, opt}, obs, next_obs, idx, action, reward, done, disc, qn_t, qn_o, loss_out,
                               n_sample, gamma, huber_delta, q_tensor),
                   use_graph, stream, [&](void* st) -> int {
    const size_t qbytes = (size_t)n_sample * adim * sizeof(float);
    int rc = net_forward_impl(target, nullptr, next_obs, idx, n_sample, st, 0u, 1u << q_tensor);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(qn_t, xtb_net_tensor(target, q_tensor), qbytes, cudaMemcpyDeviceToDevice, S(st)));
    if (qn_o) {
      rc = net_forward_impl(net, nullptr, next_obs, idx, n_sample, st, 0u, 1u << q_tensor);
      if (rc) return rc;
      CUDA_TRY(cudaMemcpyAsync(qn_o, xtb_net_tensor(net, q_tensor), qbytes, cudaMemcpyDeviceToDevice, S(st)));
    }
    const float inv_count = inv_world / ((float)n_sample * adim);
    if (fuse) {
      rc = dueling_td_fused(net, obs, idx, action, reward, done, disc, n_sample, gamma, huber_delta, q_tensor, qn_t, qn_o,
                            inv_count, loss_out, S(st));
      if (rc) return rc;
    } else {
      rc = net_forward_impl(net, nullptr, obs, idx, n_sample, st, 0u, 1u << q_tensor);
      if (rc) return rc;
      rc = xtb_dqn_td_loss_grad(xtb_net_tensor(net, q_tensor), qn_t, qn_o, idx, action, reward, done, disc, n_sample, adim, gamma,
                                huber_delta, inv_count, xtb_net_tensor_grad(net, q_tensor), nullptr, loss_out, st);
      if (rc) return rc;
      const int32_t heads[1] = {q_tensor};
      BackwardOpts o(heads, 1); o.all_reduce = true;
      rc = net_backward_impl(net, obs, idx, n_sample, st, o);
      if (rc) return rc;
    }
    return xtb_adam_step_net(opt, net, 1.f, st);
  });
}

// ------------------------------------------------------------------------------------------
// rollout inference: T batched policy evaluations over the E stacked observations
// ------------------------------------------------------------------------------------------
// T policy evaluations of the action distribution DIST: per step the forward of the layers below the heads and
// infer_heads_kernel (both heads and the draw) within the fused-inference limits, otherwise every layer and then the
// sampling kernel; the draws are the same either way.  step_idx NULL: step t reads observation rows t*E .. (t+1)*E - 1.
template <class DIST>
static int rollout_infer_launch(xtb_net* net, const void* obs, const int32_t* step_idx, int E, int T, int pi_t, int v_t, int ls_t,
                                uint64_t seed, unsigned long long* offset_dev, typename DIST::Action* action, float* logp,
                                float* value, void* stream) {
  const int adim = net->tsize[pi_t];
  const float* log_std = DIST::kLogStd ? net->params + net->L[ls_t - 1].w_off : nullptr;
  const LayerPlan& lpi = net->L[pi_t - 1];
  const LayerPlan& lv = net->L[v_t - 1];
  const bool fuse = ppo_heads_fusable(net, pi_t, v_t, true);
  const unsigned skip = fuse ? ((1u << (pi_t - 1)) | (1u << (v_t - 1))) : 0u;
  const unsigned want = fuse ? ((1u << lpi.d.src) | (1u << lv.d.src)) : ((1u << pi_t) | (1u << v_t));
  const size_t row_bytes = (size_t)net->tsize[0] * (net->desc.input_u8 ? 1 : sizeof(float));
  float* pi_out = xtb_net_tensor(net, pi_t);
  const float* v_in = xtb_net_tensor(net, v_t);
  for (int t = 0; t < T; t++) {
    const void* obs_t = step_idx ? obs : (const void*)((const char*)obs + (size_t)t * E * row_bytes);
    int rc = net_forward_impl(net, nullptr, obs_t, step_idx ? step_idx + (long long)t * E : nullptr, E, stream, skip, want);
    if (rc) return rc;
    typename DIST::Action* a_t = action + (long long)t * E * DIST::action_width(adim);
    float* lp_t = logp + (long long)t * E; float* v_o = value + (long long)t * E;
    if (fuse) {
      XLAUNCH(heads_pick(kInferHeadsKernels<DIST>, lpi.K, adim)->kern, std::max(1, std::min(kSMs, (E + 7) / 8)), 256, 0, S(stream),
              (const float*)out_f32(net, lpi.d.src), (const float*)out_f32(net, lv.d.src), net->params + lpi.w_off,
              net->params + lpi.b_off, net->params + lv.w_off, net->params + lv.b_off, log_std, E, lpi.K, adim, seed, offset_dev, t,
              a_t, lp_t, v_o, pi_out);
    } else {
      XLAUNCH(sample_kernel<DIST>, (E + 127) / 128, 128, 0, S(stream), pi_out, log_std, E, adim, (const float*)nullptr, seed,
              (uint64_t)0, offset_dev, t, a_t, lp_t, v_in, v_o);
    }
    LAUNCH_CHECK();
  }
  XLAUNCH(bump_counter_kernel, 1, 1, 0, S(stream), offset_dev, T);
  LAUNCH_CHECK();
  return XTB_OK;
}

// the checks of the rollout-inference calls past their own pointers: a bound net, the sizes and the head tensors
static int ppo_infer_check(const char* fn, const xtb_net* net, const unsigned long long* offset_dev, int n_env, int n_step,
                           int pi_t, int v_t, int ls_t) {
  if (!net->ws || !offset_dev) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (n_env <= 0 || n_env > net->max_batch || n_step <= 0) return fail(XTB_ERR_ARG, "%s: bad sizes", fn);
  return ppo_heads_check(fn, net, pi_t, v_t, ls_t);
}

// rollout inference on checked arguments, graphed under one key per argument set
static int ppo_rollout_infer(xtb_net* net, const void* obs, const int32_t* step_idx, int n_env, int n_step, int pi_t, int v_t,
                             int ls_t, uint64_t seed, unsigned long long* offset_dev, void* action, float* logp, float* value,
                             int use_graph, void* stream) {
  return run_graph(capture_key(kRolloutInfer, {net}, obs, step_idx, offset_dev, action, logp, value, n_env, n_step, pi_t, v_t, ls_t,
                               seed),
                   use_graph, stream, [&](void* st) {
    return ls_t ? rollout_infer_launch<DiagGaussian>(net, obs, step_idx, n_env, n_step, pi_t, v_t, ls_t, seed, offset_dev,
                                                     static_cast<float*>(action), logp, value, st)
                : rollout_infer_launch<Categorical>(net, obs, step_idx, n_env, n_step, pi_t, v_t, ls_t, seed, offset_dev,
                                                    static_cast<int32_t*>(action), logp, value, st);
  });
}

extern "C" int xtb_ppo_rollout_infer(xtb_net* net, const void* obs, const int32_t* step_idx, int n_env, int n_step, int pi_t,
                                     int v_t, int ls_t, uint64_t seed, unsigned long long* offset_dev, void* action, float* logp,
                                     float* value, int use_graph, void* stream) {
  const char* fn = "xtb_ppo_rollout_infer";
  if (!net || !obs || !action || !logp || !value) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (int rc = ppo_infer_check(fn, net, offset_dev, n_env, n_step, pi_t, v_t, ls_t)) return rc;
  return ppo_rollout_infer(net, obs, step_idx, n_env, n_step, pi_t, v_t, ls_t, seed, offset_dev, action, logp, value, use_graph,
                           stream);
}

// ------------------------------------------------------------------------------------------
// staging helpers
// ------------------------------------------------------------------------------------------
extern "C" void* xtb_pinned_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { fail(XTB_ERR_NOMEM, "cudaHostAlloc(%zu) failed", bytes); return nullptr; }
  return p;
}
extern "C" void xtb_pinned_free(void* p) { if (p) cudaFreeHost(p); }
extern "C" int xtb_copy_h2d(void* dst, const void* src, size_t bytes, void* stream) {
  CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, S(stream)));
  return XTB_OK;
}
extern "C" int xtb_copy_h2d_staged(void* dst, const void* src, size_t bytes, void* stream) {
  if (bytes && (!dst || !src)) return fail(XTB_ERR_ARG, "xtb_copy_h2d_staged: null pointer");
  CUDA_TRY(xtb::Stager::instance().stage_h2d(dst, src, bytes, S(stream)));
  return XTB_OK;
}
// PPO.predict with host buffers in one call (xt/model/ppo/ppo.py:104-109): staged H2D of the observations, the
// (graphed) rollout inference of one step into the packed block out_dev = [action | logp | value], one D2H of it (and
// of the pi head's output into head_host when set) and a stream synchronise.
extern "C" int xtb_ppo_predict_host(xtb_net* net, const void* obs_host, size_t obs_bytes, void* obs_dev, int n_env, int pi_t,
                                    int v_t, int ls_t, uint64_t seed, unsigned long long* offset_dev, float* out_dev,
                                    float* out_host, float* head_host, int use_graph, void* stream) {
  const char* fn = "xtb_ppo_predict_host";
  if (!net || !obs_host || !obs_dev || !out_dev || !out_host) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (int rc = ppo_infer_check(fn, net, offset_dev, n_env, 1, pi_t, v_t, ls_t)) return rc;
  const size_t aw = ls_t ? net->tsize[pi_t] : 1;   // action floats per env: the DiagGaussian's A, or one int32
  StreamScope sc;
  int src = sc.begin(stream, use_graph != 0);
  if (src) return src;
  CUDA_TRY(xtb::Stager::instance().stage_h2d(obs_dev, obs_host, obs_bytes, sc.st));
  int rc = ppo_rollout_infer(net, obs_dev, nullptr, n_env, 1, pi_t, v_t, ls_t, seed, offset_dev, out_dev, out_dev + aw * n_env,
                             out_dev + (aw + 1) * n_env, use_graph, (void*)sc.st);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(out_host, out_dev, sizeof(float) * (aw + 2) * (size_t)n_env, cudaMemcpyDeviceToHost, sc.st));
  if (head_host)
    CUDA_TRY(cudaMemcpyAsync(head_host, xtb_net_tensor(net, pi_t), sizeof(float) * (size_t)n_env * net->tsize[pi_t],
                             cudaMemcpyDeviceToHost, sc.st));
  CUDA_TRY(cudaStreamSynchronize(sc.st));
  return sc.end();
}
extern "C" int xtb_copy_d2h(void* dst, const void* src, size_t bytes, void* stream) {
  CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, S(stream)));
  return XTB_OK;
}
extern "C" int xtb_stream_sync(void* stream) {
  CUDA_TRY(cudaStreamSynchronize(S(stream)));
  return XTB_OK;
}
