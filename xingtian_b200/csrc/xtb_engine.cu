// xtb_engine.cu -- C-ABI implementation (see include/xtb200.h): the layer engine and what every learner shares, and the
// GRU learners (QMIX, SCC, InfoFlow).  The learners on rl_kernels.cuh are in learners.cu; engine.cuh declares what the
// two sources share.
#include "engine.cuh"

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <memory>
#include <string>

#include "layer_kernels.cuh"
#include "optim.cuh"
#include "qmix.cuh"
#include "agent_act.cuh"
#include "scc.cuh"
#include "episode_replay.cuh"
#include "infoflow.cuh"
#include "stager.cuh"
#include "bp_gemm.cuh"
#include "comm.cuh"
#include <cstdlib>

// ------------------------------------------------------------------------------------------
// errors / bookkeeping
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

extern "C" int xtb_version(void) { return XTB_VERSION; }
extern "C" const char* xtb_last_error(void) { return g_err.c_str(); }
extern "C" long long xtb_launch_count(void) { return g_launches.load(); }

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int carve_scratch(const char* fn, void** buf, const std::vector<Piece>& pieces) {
  size_t tot = 0;
  for (const Piece& pc : pieces) tot += align_up(pc.bytes, 256);
  cudaError_t e = cudaMalloc(buf, tot);
  if (e != cudaSuccess) return fail(XTB_ERR_NOMEM, "%s: %s", fn, cudaGetErrorString(e));
  e = cudaMemset(*buf, 0, tot);
  char* p = (char*)*buf;
  for (const Piece& pc : pieces) {
    *pc.slot = p;
    if (pc.init && e == cudaSuccess) e = cudaMemcpy(p, pc.init, pc.bytes, cudaMemcpyHostToDevice);
    p += align_up(pc.bytes, 256);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(nullptr);
  if (e != cudaSuccess) { cudaFree(*buf); return fail(XTB_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(e)); }
  return XTB_OK;
}

// ---- data-parallel communicator ---------------------------------------------------------------
static NcclApi g_nccl;
xtb_comm* g_comm = nullptr;          // installed communicator: gradients are all-reduced inside the training loops
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
bool reads(const LayerPlan& lp, int t) { return lp.d.src == t || (lp.d.kind == XTB_DUELING && lp.d.k == t); }


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
int g_tc_mode = [] { const char* e = getenv("XTB_TC"); return e ? atoi(e) : 1; }();
extern "C" int xtb_set_tc_mode(int mode) { g_tc_mode = mode; return XTB_OK; }
extern "C" int xtb_get_tc_mode(void) { return g_tc_mode; }

static inline bp::BpT out_bp(const xtb_net* n, int t) { return bp::BpT{(bp::bf16*)(n->ws + n->obp_off[t]), n->plane_elems[t], n->pitch}; }
bp::BpT gout_bp(const xtb_net* n, int t) { return bp::BpT{(bp::bf16*)(n->ws + n->gbp_off[t]), n->plane_elems[t], n->pitch}; }
static inline bp::BpT obs_bp(const xtb_net* n) { return bp::BpT{(bp::bf16*)(n->ws + n->obs_bp_off), 0, n->pitch}; }
static inline bp::BpT no_bp() { return bp::BpT{nullptr, 0, 0}; }
float* out_f32(const xtb_net* n, int t) { return (float*)(n->ws + n->out_off[t]); }
float* gout_f32(const xtb_net* n, int t) { return (float*)(n->ws + n->gout_off[t]); }
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
bool use_tc(const LayerPlan& lp) { return g_tc_mode && lp.tc; }
// The fp32 kernels' index tables of a conv layer, one workspace region [koff K][kyx K][dkyx Kd][dco Kd][wk Kd]: forward
// and weight gradient indexed by k = (ky, kx, ci), data gradient by k = (ky, kx, co)
struct ConvTabs { const int *koff, *kyx, *dkyx, *dco, *wk; };
static inline ConvTabs conv_tabs(const xtb_net* n, const LayerPlan& lp) {
  const int* t = (const int*)(n->ws + lp.im2col_off);
  return ConvTabs{t, t + lp.K, t + 2 * lp.K, t + 2 * lp.K + lp.Kd, t + 2 * lp.K + 2 * lp.Kd};
}

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
int dgrad_act(const LayerPlan& lp) { return act_is_ext(lp.src_act) ? 0 : lp.src_act; }
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
// Split-K plan of a dense tensor-core forward over B rows whose slice count is chosen for split_rows rows (rollout
// inference evaluates several steps per forward and chooses for one step's rows, so that a row's sums do not depend
// on how many steps share the launch): nz slices of kc_split chunks, partial sums in nz slabs of [round16(B)][N] floats.
// The workspace planner sizes the split-K region with it, as the launch uses it.
struct DenseSplit { int nz, kc_split; size_t part_bytes; };
static DenseSplit dense_split(const LayerPlan& lp, int B, int split_rows) {
  DenseSplit d;
  d.nz = dense_k_slices(lp.K / 8, (lp.N / lp.n_fwd) * ((split_rows + 127) / 128), &d.kc_split);
  d.part_bytes = d.nz > 1 ? (size_t)d.nz * ((B + 15) & ~15) * lp.N * sizeof(float) : 0;
  return d;
}
int infer_chunk_steps(int max_batch, int E) { return std::max(1, max_batch / E); }
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
  std::unique_ptr<xtb_net> net(new xtb_net());
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
    if (d.src < 0 || d.src > i) return fail(XTB_ERR_ARG, "layer %d: bad src %d", i, d.src);
    if (d.act < XTB_ACT_NONE || d.act > XTB_ACT_GELU) return fail(XTB_ERR_ARG, "layer %d: unknown activation %d", i, d.act);
    if (d.kind == XTB_LOGSTD) {
      // parameter-only: A floats (pi_logstd), no input, no output tensor
      if (d.src != 0) return fail(XTB_ERR_ARG, "layer %d: a logstd layer reads no tensor (src must be 0)", i);
      if (d.cout < 1 || d.cout > MAX_ADIM) return fail(XTB_ERR_ARG, "layer %d: logstd width %d not in [1, %d]", i, d.cout, MAX_ADIM);
      if (d.act != XTB_ACT_NONE) return fail(XTB_ERR_ARG, "layer %d: a logstd layer has no activation", i);
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
      if (bad_src || bad_k) return fail(XTB_ERR_ARG, "layer %d: reads the tensor of a logstd layer", i);
    }
    if (d.kind == XTB_DUELING) {
      // combine of two earlier layers: src = the A-wide stream, k = the 1-wide stream; no parameters
      if (d.src == 0 || d.k == 0) return fail(XTB_ERR_ARG, "layer %d: a dueling layer cannot read the observation", i);
      if (d.k < 0 || d.k > i) return fail(XTB_ERR_ARG, "layer %d: dueling 1-wide input %d is not an earlier layer", i, d.k);
      if (d.k == d.src) return fail(XTB_ERR_ARG, "layer %d: dueling inputs must be two different tensors", i);
      if (net->tsize[d.k] != 1) return fail(XTB_ERR_ARG, "layer %d: dueling input %d is %d wide, not 1", i, d.k, net->tsize[d.k]);
      if (d.act != XTB_ACT_NONE) return fail(XTB_ERR_ARG, "layer %d: a dueling layer has no activation", i);
      if (act_is_ext(tact[d.src]) || act_is_ext(tact[d.k]))
        return fail(XTB_ERR_ARG, "layer %d: a dueling layer reads relu / tanh / linear tensors only", i);
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
      if (d.stride != 1 && d.stride != 2 && d.stride != 4) return fail(XTB_ERR_ARG, "layer %d: stride must be 1,2,4", i);
      ConvGeom& g = lp.g;
      g.H = is.h; g.W = is.w; g.C = is.c; g.KH = g.KW = d.k; g.S = d.stride; g.Cout = d.cout;
      if (d.pad_same) {
        same_pad(g.H, d.k, d.stride, &g.OH, &g.padT);
        same_pad(g.W, d.k, d.stride, &g.OW, &g.padL);
        lp.pad = true;
      } else {
        g.OH = (g.H - d.k) / d.stride + 1; g.OW = (g.W - d.k) / d.stride + 1; g.padT = g.padL = 0;
      }
      if (g.OH <= 0 || g.OW <= 0) return fail(XTB_ERR_ARG, "layer %d: empty conv output", i);
      g.K = d.k * d.k * g.C; g.P = g.OH * g.OW;
      g.mP = fastdiv_magic(g.P); g.mOW = fastdiv_magic(g.OW); g.mHW = fastdiv_magic(g.H * g.W); g.mW = fastdiv_magic(g.W);
      lp.K = g.K; lp.N = d.cout; lp.Kd = d.k * d.k * d.cout;
      lp.sshift = d.stride == 1 ? 0 : (d.stride == 2 ? 1 : 2);
      shp[i + 1] = {g.OH, g.OW, d.cout};
      // index tables of the fp32 kernels, in the order of ConvTabs
      lp.im2col.resize(2 * g.K + 3 * lp.Kd);
      int *koff = lp.im2col.data(), *kyx = koff + g.K, *dkyx = kyx + g.K, *dco = dkyx + lp.Kd, *wk = dco + lp.Kd;
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
      return fail(XTB_ERR_ARG, "layer %d: unknown kind %d", i, d.kind);
    }
    if (lp.N <= 0) return fail(XTB_ERR_ARG, "layer %d: zero outputs", i);
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
  // a host-built table: its region, and its entry in the list every bind uploads
  auto table = [&](const auto& v) {
    const size_t o = w, bytes = v.size() * sizeof(v[0]);
    w += align_up(bytes, 256);
    if (bytes) net->tables.push_back(HostTable{o, v.data(), bytes});
    return o;
  };
  for (auto& lp : net->L) if (lp.tc && lp.d.kind == XTB_CONV) {
    lp.fwd_st_off = table(lp.fwd_st); lp.fwd_un_off = table(lp.fwd_un);
    lp.dg_st_off = table(lp.dg_st); lp.dg_un_off = table(lp.dg_un);
    lp.wg_off = table(lp.wg_tab);
  }
  // split-K partial sums of a dense forward: the largest over the forwards the net runs, B rows split for E rows with
  // E <= B <= max_batch; a rollout-inference chunk of E environments (the most rows at a given E) covers every B = E
  net->splitk_off = w;
  {
    size_t need = 0;
    for (auto& lp : net->L) if (lp.tc && lp.d.kind == XTB_DENSE)
      for (int E = 1; E <= max_batch; E++)
        need = std::max(need, dense_split(lp, infer_chunk_steps(max_batch, E) * E, E).part_bytes);
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
  if (!net->blob_segs.empty())
    net->tables.push_back(HostTable{net->segs_off, net->blob_segs.data(), net->blob_segs.size() * sizeof(bp::BlobSeg)});
  // every conv layer: the fp32 kernels also run tensor-core layers (xtb_set_tc_mode(0), forwards with other parameters)
  for (auto& lp : net->L) if (lp.d.kind == XTB_CONV) lp.im2col_off = table(lp.im2col);
  net->ws_bytes = w;
  net->cur.assign(nt, TensorForms{});
  *out = net.release();
  return XTB_OK;
}

extern "C" void xtb_net_destroy(xtb_net* net) {
  if (!net) return;
  drop_graphs_of(net);
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
  for (const HostTable& t : net->tables)
    CUDA_TRY(cudaMemcpyAsync(net->ws + t.off, t.data, t.bytes, cudaMemcpyHostToDevice, st));
  invalidate(net, true, true);
  int rc = xtb_net_sync_weights(net, stream);
  if (rc) return rc;
  // the tables are copied from pageable host memory: do not return before they are on the device
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

void queue_reduction(xtb_net* net, const float* part, int n_slabs, long long slab, int count, long long dst_off, float* dst_ptr,
                     const LayerPlan* conv) {
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

// forward of a tensor-core layer over B rows, a dense layer split over K as for split_rows rows (dense_split).
// want_f32: also store the fp32 row-major copy; want_bp: store the planes
static cudaError_t tc_forward(xtb_net* net, int i, int B, int split_rows, bool want_f32, bool want_bp, cudaStream_t st,
                              long long* launches) {
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
  const DenseSplit sp = dense_split(lp, B, split_rows);
  const int nz = sp.nz;
  a.kc_split = sp.kc_split;
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
  const long long ea = (long long)fa * pitch;
  const long long ew = mode == 2 ? (long long)fb * pitch : (mode == 1 ? (long long)K * ((N + 15) / 16 * 16) : (long long)N * K);   // weight blob / second activation
  const long long ec = (long long)N * pitch;
  // mode 0 split-K: nz slices of kc_split K chunks
  const int kchunks = K / 8, kc_split = mode == 0 && ksplit > 1 ? ((kchunks + ksplit - 1) / ksplit + 7) / 8 * 8 : kchunks;
  const int nz = (kchunks + kc_split - 1) / kc_split;
  bp::bf16 *pa, *pw, *pc; float *bias, *part;
  void* buf;
  if (int rc = carve_scratch("xtb_tc_gemm_test", &buf, {{&pa, 2 * ea}, {&pw, 2 * ew + 128}, {&pc, 2 * ec + 2048},
                                                        {&bias, std::max(N, 64)}, {&part, nz > 1 ? (long long)nz * M * N : 0}}))
    return rc;
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
    r.kchunks = kchunks; r.kc_split = kc_split;
    r.bias = bias; r.alpha = 1.f; r.act = 0;
    if (mode == 0) {
      r.n_units = r.n_ntiles * nz;
      if (nz > 1) {
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
  cudaFree(buf);
  if (e != cudaSuccess) return fail(XTB_ERR_CUDA, "tc gemm launch: %s", cudaGetErrorString(e));
  if (e2 != cudaSuccess) return fail(XTB_ERR_CUDA, "tc gemm run: %s", cudaGetErrorString(e2));
  return XTB_OK;
}

// ------------------------------------------------------------------------------------------
// fp32 CUDA-core layer ops
// ------------------------------------------------------------------------------------------
template <typename T>
static void conv_fwd(const xtb_net* net, const LayerPlan& lp, const T* x, const int32_t* idx, const float* w, const float* b,
                     float alpha, float* out, int B, cudaStream_t st) {
  int M = B * lp.g.P;
  BRowMajor bl{w, lp.N};
  EpiBiasAct ep{out, b, alpha, act_is_ext(lp.d.act) ? 0 : lp.d.act, lp.N, nullptr, 0};
  const ConvTabs tab = conv_tabs(net, lp);
  if (lp.pad) { AIm2col<T, true> al{x, idx, lp.g, tab.koff, tab.kyx}; launch_gemm(al, bl, ep, M, lp.N, lp.K, false, st); }
  else { AIm2col<T, false> al{x, idx, lp.g, tab.koff, tab.kyx}; launch_gemm(al, bl, ep, M, lp.N, lp.K, false, st); }
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
static void conv_wgrad(const xtb_net* net, const LayerPlan& lp, const T* x, const int32_t* idx, const float* dy, float alpha,
                       float* dw, int B, cudaStream_t st, bool bias_row = true) {
  int Mr = B * lp.g.P;
  BRowMajor bl{dy, lp.N};
  EpiAtomic ep{dw, alpha, lp.N};
  // rows 0..K-1 scaled by alpha (input decode scale); the bias row (K) must not be scaled:
  // it rides in the same GEMM only when alpha == 1, else colsum_kernel computes it.
  int rows = lp.K + ((alpha == 1.f && bias_row) ? 1 : 0);
  const ConvTabs tab = conv_tabs(net, lp);
  if (lp.pad) { AIm2colT<T, true> al{x, idx, lp.g, tab.koff, tab.kyx, Mr}; launch_gemm(al, bl, ep, rows, lp.N, Mr, true, st); }
  else { AIm2colT<T, false> al{x, idx, lp.g, tab.koff, tab.kyx, Mr}; launch_gemm(al, bl, ep, rows, lp.N, Mr, true, st); }
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

// forward of layer i; tc_allowed = parameters are the bound ones (their blobs are current); split_rows: see tc_forward
static int op_forward(xtb_net* net, int i, const float* P, bool tc_allowed, const void* obs, const int32_t* idx, int B,
                      int split_rows, bool want_f32, cudaStream_t st) {
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
    cudaError_t te = tc_forward(net, i, B, split_rows, want_f32, true, st, &nl);
    if (te != cudaSuccess) return fail(XTB_ERR_CUDA, "tensor-core forward launch (layer %d): %s", i, cudaGetErrorString(te));
    g_launches.fetch_add(nl, std::memory_order_relaxed);
    if (ext) return act_forward(net, t, B, st);
    wrote(net, t, false, want_f32 ? kBoth : kPlanes);
    return XTB_OK;
  }
  auto gemm = [&](auto x, const int32_t* ix, float alpha) {
    if (lp.d.kind == XTB_CONV) conv_fwd(net, lp, x, ix, w, b, alpha, pre, B, st);
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
      if (lp.d.kind == XTB_CONV) conv_wgrad(net, lp, x, ix, dy, alpha, dw, B, st, !bias_done);
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
    const ConvTabs tab = conv_tabs(net, lp);
    ADgrad al{dy, lp.g, tab.dkyx, tab.dco, lp.sshift};
    BConvDgrad bl{w, tab.wk, lp.N};
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
extern "C" int xtb_net_forward(xtb_net* net, const float* params, const void* obs, const int32_t* gather_idx,
                               int batch, void* stream) {
  return net_forward_impl(net, params, obs, gather_idx, batch, stream, 0u, ~0u);
}
int net_forward_impl(xtb_net* net, const float* params, const void* obs, const int32_t* gather_idx, int batch, void* stream,
                     unsigned skip_mask, unsigned want_f32_mask, int split_rows) {
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
    int rc = op_forward(net, i, P, tc_allowed, obs, gather_idx, batch, split_rows ? split_rows : batch, direct, st);
    if (rc) return rc;
  }
  for (int t = 1; t <= nl; t++) {
    if (!((want_f32_mask >> t) & 1u) || (skip_mask & (1u << (t - 1))) || net->tsize[t] == 0) continue;
    int rc = ensure_f32(net, t, batch, false, st);
    if (rc) return rc;
  }
  return XTB_OK;
}

extern "C" int xtb_net_backward(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch,
                                const int32_t* head_tensors, int n_heads, void* stream) {
  return net_backward_impl(net, obs, gather_idx, batch, stream, BackwardOpts(head_tensors, n_heads));
}
int input_grad_check(const xtb_net* net) {
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
int net_backward_impl(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch, void* stream, const BackwardOpts& o) {
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
  if (which == 0) return op_forward(net, layer, net->params, true, obs, gather_idx, batch, batch, false, st);
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
// optimiser
// ------------------------------------------------------------------------------------------

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
  AdamHyper hy{lr, beta1, beta2, eps, clip, 0.f};
  // carve_scratch's synchronize also completes these fills before the call returns
  cudaError_t e = cudaMemset(m, 0, count * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(v, 0, count * sizeof(float));
  if (e != cudaSuccess) { delete o; return fail(XTB_ERR_CUDA, "xtb_adam_create: %s", cudaGetErrorString(e)); }
  if (int rc = carve_scratch("xtb_adam_create", &o->buf, {{&o->blk_seg, o->n_blk, bseg.data()}, {&o->blk_beg, o->n_blk, bbeg.data()},
                                                          {&o->blk_len, o->n_blk, blen.data()}, {&o->norm_sq, o->n_seg},
                                                          {&o->seg_scale, o->n_seg}, {&o->st, 1, &init}, {&o->hyp, 1, &hy},
                                                          {&o->ticket, 1}})) {
    delete o;
    return rc;
  }
  *out = o;
  return XTB_OK;
}

extern "C" void xtb_adam_destroy(xtb_adam* o) {
  if (!o) return;
  drop_graphs_of(o);
  cudaDeviceSynchronize();
  cudaFree(o->buf);
  delete o;
}

extern "C" int xtb_adam_step(xtb_adam* o, float* params, const float* grads, float grad_scale, void* stream) {
  return adam_step_impl(o, params, grads, grad_scale, stream, nullptr);
}
// optimiser step on a network's bound parameters; the same kernel refreshes the weight blobs of its tensor-core layers
extern "C" int xtb_adam_step_net(xtb_adam* o, xtb_net* net, float grad_scale, void* stream) {
  if (!net || !net->ws || !net->params || !net->grads) return fail(XTB_ERR_STATE, "xtb_adam_step_net: net not bound");
  if (!o || o->count != net->n_params) return fail(XTB_ERR_ARG, "xtb_adam_step_net: optimiser/net size mismatch");
  return adam_step_impl(o, net->params, net->grads, grad_scale, stream, net);
}
int adam_step_impl(xtb_adam* o, float* params, const float* grads, float grad_scale, void* stream, xtb_net* net) {
  if (!o || !params || !grads) return fail(XTB_ERR_ARG, "xtb_adam_step: null pointer");
  if (misaligned16(params) || misaligned16(grads) || misaligned16(o->m) || misaligned16(o->v) || misaligned16(o->mg))
    return fail(XTB_ERR_ARG, "xtb_adam_step: params, grads and the optimiser slots must be 16-byte aligned");
  cudaStream_t st = S(stream);
  XLAUNCH(sqnorm_kernel, (o->n_blk + SQN_GROUP - 1) / SQN_GROUP, OPT_THREADS, 0, st, grads, o->blk_seg, o->blk_beg, o->blk_len, o->n_blk, o->norm_sq, o->ticket, o->st,
          (const AdamHyper*)o->hyp, o->seg_scale, o->n_seg, o->clip_mode, grad_scale);
  LAUNCH_CHECK();
  const bool blobs = net && !net->blob_segs.empty();
  if (o->mg || o->rms_plain) {
    XLAUNCH(o->mg ? rmsprop_kernel<true> : rmsprop_kernel<false>, o->n_blk, OPT_THREADS, 0, st, params, grads, o->m, o->mg, o->blk_seg, o->blk_beg, o->blk_len,
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
  o->mg = mean_grad; o->rms_rho = decay; o->rms_eps = epsilon; o->rms_plain = false;
  return XTB_OK;
}
extern "C" int xtb_opt_use_rmsprop_plain(xtb_adam* o, float decay, float epsilon) {
  if (!o) return fail(XTB_ERR_ARG, "xtb_opt_use_rmsprop_plain: null pointer");
  if (!(decay > 0.f && decay < 1.f) || !(epsilon > 0.f)) return fail(XTB_ERR_ARG, "xtb_opt_use_rmsprop_plain: decay in (0,1), epsilon > 0");
  drop_graphs_of(o);
  {   // the `rms` slot of tf.train.RMSPropOptimizer starts at ones (one-time, synchronous)
    std::vector<float> ones((size_t)o->count, 1.f);
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(o->m, ones.data(), ones.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  o->mg = nullptr; o->rms_rho = decay; o->rms_eps = epsilon; o->rms_plain = true;
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
// engine streams, the CUDA-graph cache and the learner checks
// ------------------------------------------------------------------------------------------
struct EngineStream { cudaStream_t st = nullptr; cudaEvent_t in = nullptr, out = nullptr; };
static EngineStream g_engine_streams[64];
int StreamScope::begin(void* stream, bool side_if_null) {
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
int StreamScope::end() {
  if (!es) return XTB_OK;
  CUDA_TRY(cudaEventRecord(es->out, es->st));
  CUDA_TRY(cudaStreamWaitEvent(nullptr, es->out, 0));
  es = nullptr;
  return XTB_OK;
}
int g_fuse_heads = [] { const char* e = getenv("XTB_FUSE_HEADS"); return e ? atoi(e) : 1; }();
extern "C" int xtb_set_fuse_heads(int on) { g_fuse_heads = on; return XTB_OK; }

static constexpr size_t kMaxCachedGraphs = 256;   // beyond it the cache is emptied (keys are buffer addresses)
static std::map<CaptureKey, GraphVal> g_graphs;
static std::atomic<long long> g_graph_replays{0};
static std::atomic<long long> g_graph_captures{0};
extern "C" long long xtb_graph_replay_count(void) { return g_graph_replays.load(); }
extern "C" long long xtb_graph_capture_count(void) { return g_graph_captures.load(); }

const GraphVal* graph_find(const CaptureKey& key) {
  auto it = g_graphs.find(key);
  return it == g_graphs.end() ? nullptr : &it->second;
}
const GraphVal* graph_add(const CaptureKey& key, cudaGraphExec_t exec, long long kernels) {
  if (g_graphs.size() >= kMaxCachedGraphs) {     // callers that pass fresh buffers every call must not leak executables
    for (auto& kv : g_graphs) cudaGraphExecDestroy(kv.second.exec);
    g_graphs.clear();
  }
  g_graph_captures.fetch_add(1, std::memory_order_relaxed);
  return &g_graphs.emplace(key, GraphVal{exec, kernels}).first->second;
}
int graph_launch(const GraphVal& g, cudaStream_t st) {
  CUDA_TRY(cudaGraphLaunch(g.exec, st));
  g_launches.fetch_add(g.kernels, std::memory_order_relaxed);
  g_graph_replays.fetch_add(1, std::memory_order_relaxed);
  return XTB_OK;
}
void drop_graphs_of(const void* obj) {
  for (auto it = g_graphs.begin(); it != g_graphs.end();) {
    const auto& own = it->first.own;
    if (std::find(std::begin(own), std::end(own), obj) != std::end(own)) { cudaGraphExecDestroy(it->second.exec); it = g_graphs.erase(it); } else ++it;
  }
}

float dp_inv_world() { return g_comm ? 1.f / g_comm->world : 1.f; }

int learner_check(const char* fn, bool missing, const xtb_net* net, const xtb_adam* opt, long long rows, bool dp_ok, long long max_rows,
                  long long n_params) {
  if (missing) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (!net->ws || !net->grads) return fail(XTB_ERR_STATE, "%s: net not bound", fn);
  if (!dp_ok && g_comm) return fail(XTB_ERR_STATE, "%s: data-parallel training (communicator) is not supported", fn);
  if (opt && opt->count != (n_params ? n_params : net->n_params))
    return fail(XTB_ERR_ARG, "%s: optimiser/net size mismatch (%lld != %lld)", fn, opt->count, n_params ? n_params : net->n_params);
  if (!max_rows) max_rows = net->max_batch;
  if (rows < 1 || rows > max_rows) return fail(XTB_ERR_ARG, "%s: batch %lld not in [1, %lld]", fn, rows, max_rows);
  return XTB_OK;
}

// ---- The recurrent agent of QMIX and SCC (xt/model/qmix/qmix_tf.py: fc1 -> GRU -> fc2) --------------------------------
// fc1 and fc2 are engine nets bound to the slices [fc1 | gru | fc2] at the front of their object's eval weight set, the
// GRU's kernels and biases at o_gru; other weight sets are read through the nets' foreign-parameter forward.  A training
// batch is B episodes of T = L + 1 steps of n agents: R = B T n agent rows, BL = B L steps and S = B n GRU sequences, G
// of them per CTA of the GRU kernels with smem bytes of shared memory.  Acting steps up to E environments at once (E n
// rows of one step each, agent_act): the forward's scratch holds max(R, E n) rows.
struct QmixAgent {
  xtb_net *fc1 = nullptr, *fc2 = nullptr;
  int B = 0, L = 0, T = 0, n = 0, A = 0, H = 0, R = 0, BL = 0, S = 0, G = 0, E = 1;
  size_t smem = 0;
  long long o_gru = 0, o_fc2 = 0;
  float *xg = nullptr, *xc = nullptr, *hout = nullptr, *rh = nullptr, *dy = nullptr, *dag = nullptr, *dac = nullptr;
  float* xin = nullptr;      // [E n, fc1 input width] the acting inputs
  int32_t* ones = nullptr;   // [E n] sequence lengths of the one-step inference and of acting
};

// layer i of nt is a dense layer on tensor src with activation act
static bool dense_layer(const xtb_net* nt, int i, int src, int act) {
  const LayerPlan& lp = nt->L[i];
  return lp.d.kind == XTB_DENSE && lp.d.src == src && lp.d.act == act;
}

// Sequences per CTA of the GRU kernels for S sequences of width H: enough to cover S in one wave of CTAs, at most 8,
// fewer while their shared memory would not fit
static int gru_group(long long S, int H) {
  int G = (int)std::max(1LL, std::min(8LL, (S + kSMs - 1) / kSMs));
  while (G > 1 && qgru_smem_floats(H, G) * 4 > kMaxDynSmem) G--;
  return G;
}

// The agent's checks and sizes for `batch` episodes of `episode_limit` steps of `n_agents` agents with the GRU at gru_off,
// acting for up to act_envs environments (0: one), into *a: all of them but the nets' row capacity (agent_capacity),
// which the caller checks after its own size bounds.
static int agent_plan(const char* fn, xtb_net* fc1, xtb_net* fc2, int batch, int episode_limit, int n_agents, long long gru_off,
                      int act_envs, QmixAgent* a) {
  for (xtb_net* nt : {fc1, fc2})
    if (!nt->ws || !nt->params || !nt->grads) return fail(XTB_ERR_STATE, "%s: every net must be bound", fn);
  if (fc1->L.size() != 1 || !dense_layer(fc1, 0, 0, XTB_ACT_RELU) || fc1->desc.input_u8 || fc1->desc.scale != 1.f)
    return fail(XTB_ERR_ARG, "%s: fc1 must be one relu dense layer on float agent inputs", fn);
  const int H = fc1->tsize[1];
  if (fc2->L.size() != 1 || !dense_layer(fc2, 0, 0, XTB_ACT_NONE) || fc2->tsize[0] != H)
    return fail(XTB_ERR_ARG, "%s: fc2 must be one linear dense layer on the %d-wide GRU output", fn, H);
  if (int rc = input_grad_check(fc2)) return rc;
  const int A = fc2->tsize[1], n = n_agents;
  if (n < 1 || n > QM_MAX_AGENTS) return fail(XTB_ERR_ARG, "%s: n_agents %d not in [1, %d]", fn, n, QM_MAX_AGENTS);
  if (A < 1 || A > 255) return fail(XTB_ERR_ARG, "%s: n_actions %d not in [1, 255] (actions are uint8 in the reference)", fn, A);
  if (batch < 1 || episode_limit < 1) return fail(XTB_ERR_ARG, "%s: batch %d / episode_limit %d out of range", fn, batch, episode_limit);
  const long long T = episode_limit + 1LL, R = batch * T * n;
  if (R > (1LL << 30) / std::max(3 * H, 1)) return fail(XTB_ERR_ARG, "%s: batch too large", fn);
  if (act_envs < 0 || (long long)act_envs * n > (1LL << 30) / std::max(3 * H, std::max(fc1->tsize[0], 1)))
    return fail(XTB_ERR_ARG, "%s: act_envs %d out of range", fn, act_envs);
  const int S = batch * n, G = gru_group(S, H);
  if (H < 1 || qgru_smem_floats(H, G) * 4 > kMaxDynSmem)
    return fail(XTB_ERR_ARG, "%s: rnn_hidden_dim %d: the GRU weights do not fit in shared memory", fn, H);
  // the gradients at the same offsets as the weights
  const long long o_fc2 = fc2->params - fc1->params, gru_n = 2LL * H * 2 * H + 2 * H + 2LL * H * H + H;
  if (gru_off < fc1->n_params || o_fc2 < gru_off + gru_n || fc2->grads != fc1->grads + o_fc2)
    return fail(XTB_ERR_ARG, "%s: nets must be bound to slices [fc1 | gru | fc2] at the front of one buffer, in order", fn);
  a->fc1 = fc1; a->fc2 = fc2;
  a->B = batch; a->L = episode_limit; a->T = (int)T; a->n = n; a->A = A; a->H = H; a->R = (int)R; a->BL = batch * episode_limit;
  a->S = S; a->G = G; a->smem = qgru_smem_floats(H, G) * 4; a->E = std::max(act_envs, 1);
  a->o_gru = gru_off; a->o_fc2 = o_fc2;
  return XTB_OK;
}

// fc1 and fc2 hold the R rows of a training batch and the E n rows of acting
static int agent_capacity(const char* fn, const QmixAgent& a) {
  if (a.fc1->max_batch < a.R || a.fc2->max_batch < a.R) return fail(XTB_ERR_ARG, "%s: fc1 / fc2 hold fewer rows than a batch (%d)", fn, a.R);
  const long long act_rows = (long long)a.E * a.n;
  if (a.fc1->max_batch < act_rows || a.fc2->max_batch < act_rows)
    return fail(XTB_ERR_ARG, "%s: fc1 / fc2 hold fewer rows than act_envs x n_agents (%lld)", fn, act_rows);
  return XTB_OK;
}

// The GRU kernels' shared-memory opt-in.  It is a property of the kernels, shared by every live QMIX, SCC and InfoFlow
// object: it is set to the most any object may use (one object's own need would shrink it under an earlier object with
// a wider GRU or more sequences per CTA).
static int gru_kernel_attrs(const char* fn) {
  cudaError_t e = cudaFuncSetAttribute(qmix_gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(qmix_gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
  if (e != cudaSuccess) return fail(XTB_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(e));
  return XTB_OK;
}

// The GRU kernels' shared-memory opt-in, then the object's scratch in one carve_scratch into *buf: the agent's pieces,
// with the acting inputs and the one-step sequence lengths, before the object's own `pieces`.  On failure nothing stays
// allocated.
static int agent_alloc(const char* fn, QmixAgent& a, void** buf, std::vector<Piece> pieces) {
  if (int rc = gru_kernel_attrs(fn)) return rc;
  const long long R = a.R, H = a.H, En = (long long)a.E * a.n, F = std::max(R, En);
  const std::vector<int32_t> ones(En, 1);
  pieces.insert(pieces.begin(), {{&a.xg, F * 2 * H}, {&a.xc, F * H}, {&a.hout, F * H}, {&a.rh, R * H}, {&a.dy, R * H},
                                 {&a.dag, R * 2 * H}, {&a.dac, R * H}, {&a.xin, En * a.fc1->tsize[0]}, {&a.ones, En, ones.data()}});
  return carve_scratch(fn, buf, pieces);
}

// The recurrent halves of GRUCell's gates/kernel wg [2H, 2H] and candidate/kernel wc [2H, H] (see GruRec)
static GruRec cell_rec(const float* wg, const float* wc, int H) { return GruRec{wg + 2LL * H * H, wc + (long long)H * H, 2 * H, H, 0, 0}; }

// fc1 -> GRU -> fc2 of the weight set P (NULL: the eval set the nets are bound to) over `rows` agent rows holding
// S = rows / T sequences of T steps; the Q values stay in fc2's output tensor.  h0 / hT: see qmix_gru_fwd_kernel.
static int qmix_agent_forward(QmixAgent& a, const float* P, const float* obs, int rows, int T, const int32_t* seq_len, const float* h0,
                              float* hT, int store, cudaStream_t st) {
  const int H = a.H;
  const float* W = P ? P : a.fc1->params;
  const float *wg = W + a.o_gru, *bg = wg + 2 * H * 2 * H, *wc = bg + 2 * H, *bc = wc + 2 * H * H;
  int rc = net_forward_impl(a.fc1, P, obs, nullptr, rows, st, 0u, 1u << 1);
  if (rc) return rc;
  const float* x = xtb_net_tensor(a.fc1, 1);
  // the input projections of every step: x W[:H] + b for the gates and the candidate
  launch_gemm(ADense<float>{x, nullptr, H}, BRowMajor{wg, 2 * H}, EpiBiasAct{a.xg, bg, 1.f, XTB_ACT_NONE, 2 * H, nullptr, 0}, rows,
              2 * H, H, false, st);
  LAUNCH_CHECK();
  launch_gemm(ADense<float>{x, nullptr, H}, BRowMajor{wc, H}, EpiBiasAct{a.xc, bc, 1.f, XTB_ACT_NONE, H, nullptr, 0}, rows, H, H,
              false, st);
  LAUNCH_CHECK();
  const int S = rows / T, G = a.G;
  XLAUNCH(qmix_gru_fwd_kernel, (S + G - 1) / G, QG_THREADS, a.smem, st, cell_rec(wg, wc, H), a.xg, a.xc, h0, hT, a.hout, a.rh, seq_len, S, T,
          a.n, H, G, store);
  LAUNCH_CHECK();
  return net_forward_impl(a.fc2, P ? P + a.o_fc2 : nullptr, a.hout, nullptr, rows, st, 0u, 1u << 1);
}

// Backward of qmix_agent_forward (store = 1, the eval set, all R rows) from d loss / d Q in fc2's output gradient: fc2
// (with d loss / d GRU output), the GRU in reverse time, its weight gradients as GEMMs over all rows, fc1.
static int qmix_agent_backward(QmixAgent& a, const float* obs, const int32_t* seq_len, cudaStream_t st) {
  const int H = a.H, R = a.R, n = a.n;
  const int32_t one[1] = {1};
  BackwardOpts o2(one, 1);
  o2.dobs = a.dy;
  int rc = net_backward_impl(a.fc2, a.hout, nullptr, R, st, o2);
  if (rc) return rc;
  const float* W = a.fc1->params;
  const float *wg = W + a.o_gru, *wc = wg + 2 * H * 2 * H + 2 * H;
  float* gg = a.fc1->grads + a.o_gru;
  float* gc = gg + 2 * H * 2 * H + 2 * H;
  const int S = a.S, G = a.G;
  XLAUNCH(qmix_gru_bwd_kernel, (S + G - 1) / G, QG_THREADS, a.smem, st, cell_rec(wg, wc, H), (const float*)a.xg, (const float*)a.xc,
          (const float*)a.hout, (const float*)a.dy, a.dag, a.dac, seq_len, S, a.T, a.n, H, G);
  LAUNCH_CHECK();
  const float* x = xtb_net_tensor(a.fc1, 1);
  // [kernel; bias] gradients: [x | h_prev | 1]^T da_gates and [x | r h_prev | 1]^T da_candidate over all rows
  launch_gemm(AGruFeat{x, a.hout, H, n, a.T, 1}, BRowMajor{a.dag, 2 * H}, EpiDgrad{gg, gg, 0, 2 * H, 0, nullptr, 0}, 2 * H + 1, 2 * H,
              R, false, st);
  LAUNCH_CHECK();
  launch_gemm(AGruFeat{x, a.rh, H, n, a.T, 0}, BRowMajor{a.dac, H}, EpiDgrad{gc, gc, 0, H, 0, nullptr, 0}, 2 * H + 1, H, R, false, st);
  LAUNCH_CHECK();
  // d loss / d fc1 pre-activation = relu'(x) (da_gates W_g[:H]^T + da_candidate W_c[:H]^T)
  float* dx = xtb_net_tensor_grad(a.fc1, 1);
  launch_gemm(ADense<float>{a.dag, nullptr, 2 * H}, BTransposed{wg, 2 * H}, EpiDgrad{dx, x, XTB_ACT_RELU, H, 0, nullptr, 0}, R, H, 2 * H,
              false, st);
  LAUNCH_CHECK();
  launch_gemm(ADense<float>{a.dac, nullptr, H}, BTransposed{wc, H}, EpiDgrad{dx, x, XTB_ACT_RELU, H, 1, nullptr, 0}, R, H, H, false, st);
  LAUNCH_CHECK();
  return net_backward_impl(a.fc1, obs, nullptr, R, st, BackwardOpts(one, 1));
}

// One step of the agent for one environment: fc1 -> GRU -> fc2 of the weight set `explore` on obs [n, obs_dim], hidden
// [n, H] read and overwritten, q_out [n, A]
static int qmix_agent_step(QmixAgent& a, const float* explore, const float* obs, float* hidden, float* q_out, cudaStream_t st) {
  int rc = qmix_agent_forward(a, explore, obs, a.n, 1, a.ones, hidden, hidden, 0, st);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(q_out, xtb_net_tensor(a.fc2, 1), (size_t)a.n * a.A * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return XTB_OK;
}

// xtb_qmix_infer and xtb_scc_infer: the agent step of object obj, graph-replayed under the object's tag and owners
template <size_t N>
static int agent_infer(const char* fn, GraphTag tag, const void* const (&owners)[N], const void* obj, QmixAgent& a, const float* explore,
                       const float* obs, float* hidden, float* q_out, int use_graph, void* stream) {
  if (int rc = learner_check(fn, !explore || !obs || !hidden || !q_out, a.fc1, nullptr, a.n, true)) return rc;
  return run_graph(capture_key(tag, owners, obj, explore, obs, hidden, q_out), use_graph, stream,
                   [&](void* st) { return qmix_agent_step(a, explore, obs, hidden, q_out, S(st)); });
}

// xtb_qmix_act and xtb_scc_act: one step of n_envs environments of object obj (agent_act.cuh), graph-replayed under the
// object's tag and owners.  The GRU runs the n_envs n sequences with the sequences per CTA gru_group picks for them.
template <size_t N>
static int agent_act(const char* fn, GraphTag tag, const void* const (&owners)[N], const void* obj, QmixAgent& a, const float* explore,
                     int n_envs, int last_on, int id_on, const float* obs, const int32_t* avail, const int32_t* reset, const double* eps,
                     const double* uniforms, unsigned long long seed, unsigned long long* counter, float* hidden, int32_t* last_action,
                     int32_t* actions, int use_graph, void* stream) {
  const bool missing = !explore || !obs || !avail || !reset || !eps || !hidden || !last_action || !actions || (!uniforms && !counter);
  if (int rc = learner_check(fn, missing, a.fc1, nullptr, 1, true)) return rc;
  if (n_envs < 1 || n_envs > a.E) return fail(XTB_ERR_ARG, "%s: n_envs %d not in [1, %d] (act_envs)", fn, n_envs, a.E);
  const int W = a.fc1->tsize[0], o = W - (last_on ? a.A : 0) - (id_on ? a.n : 0);
  if (o < 1) return fail(XTB_ERR_ARG, "%s: fc1's %d inputs leave no room for the observation", fn, W);
  last_on = last_on ? 1 : 0; id_on = id_on ? 1 : 0;
  return run_graph(capture_key(tag, owners, obj, explore, n_envs, last_on, id_on, obs, avail, reset, eps, uniforms, seed, counter, hidden,
                               last_action, actions),
                   use_graph, stream, [&](void* sv) -> int {
    cudaStream_t st = S(sv);
    const int n = a.n, H = a.H, rows = n_envs * n;
    const long long work = (long long)rows * std::max(W, H);
    XLAUNCH(agent_act_inputs_kernel, (unsigned)std::min<long long>((work + AA_THREADS - 1) / AA_THREADS, 8LL * kSMs), AA_THREADS, 0, st,
            obs, reset, last_action, hidden, uniforms ? nullptr : counter, a.xin, n_envs, n, o, a.A, H, last_on, id_on);
    LAUNCH_CHECK();
    QmixAgent b = a;
    b.G = gru_group(rows, H);
    b.smem = qgru_smem_floats(H, b.G) * 4;
    if (int rc = qmix_agent_forward(b, explore, a.xin, rows, 1, a.ones, hidden, hidden, 0, st)) return rc;
    XLAUNCH(agent_act_select_kernel, (rows + AA_THREADS - 1) / AA_THREADS, AA_THREADS, 0, st, (const float*)xtb_net_tensor(a.fc2, 1), avail,
            eps, uniforms, seed, (const unsigned long long*)counter, actions, last_action, n_envs, n, a.A);
    LAUNCH_CHECK();
    return XTB_OK;
  });
}

// ---- QMIX (xt/model/qmix/qmix_tf.py) ----------------------------------------------------------------------------------
// The agent and the hypernetworks, an engine net bound to the slice after fc2 of the eval weight set; target and explore
// sets are read through the nets' foreign-parameter forward.  The object owns the step's device scratch for the fixed
// batch.
struct xtb_qmix {
  QmixAgent ag;
  xtb_net* hyp = nullptr;
  xtb_qmix_desc d{};
  int E = 0, n_part = 0;
  long long o_hyp = 0, n_params = 0;
  void* buf = nullptr;
  float *qt = nullptr, *w1t = nullptr, *b1t = nullptr, *wft = nullptr, *vt = nullptr, *part = nullptr;
};
// hyper net: tensor ids of the w1, b1, w_final and v heads
static const int kQw1 = 2, kQb1 = 3, kQwf = 5, kQv = 7;

extern "C" int xtb_qmix_create(xtb_net* fc1, xtb_net* fc2, xtb_net* hyp, const xtb_qmix_desc* desc, xtb_qmix** out) {
  const char* fn = "xtb_qmix_create";
  if (!fc1 || !fc2 || !hyp || !desc || !out) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  const xtb_qmix_desc& d = *desc;
  QmixAgent ag;
  if (int rc = agent_plan(fn, fc1, fc2, d.batch, d.episode_limit, d.n_agents, d.gru_off, d.act_envs, &ag)) return rc;
  if (!hyp->ws || !hyp->params || !hyp->grads) return fail(XTB_ERR_STATE, "%s: every net must be bound", fn);
  if (hyp->L.size() != 7 || !dense_layer(hyp, 0, 0, XTB_ACT_RELU) || !dense_layer(hyp, 1, 1, XTB_ACT_NONE) ||
      !dense_layer(hyp, 2, 0, XTB_ACT_NONE) || !dense_layer(hyp, 3, 0, XTB_ACT_RELU) || !dense_layer(hyp, 4, 4, XTB_ACT_NONE) ||
      !dense_layer(hyp, 5, 0, XTB_ACT_RELU) || !dense_layer(hyp, 6, 6, XTB_ACT_NONE))
    return fail(XTB_ERR_ARG, "%s: hyper must be hyper_w1 (2 layers), hyper_b1, hyper_w_final (2 layers), val_for_bias (2 layers)", fn);
  const int E = hyp->tsize[kQb1], n = ag.n;
  if (E < 1 || E > QM_MAX_EMBED || hyp->tsize[kQw1] != E * n || hyp->tsize[kQwf] != E || hyp->tsize[6] != E || hyp->tsize[kQv] != 1)
    return fail(XTB_ERR_ARG, "%s: mixer widths disagree (embed %d must be in [1, %d], w1 embed x n_agents, v 1)", fn, E, QM_MAX_EMBED);
  const long long R = ag.R, BL = ag.BL;
  if (int rc = agent_capacity(fn, ag)) return rc;
  if (hyp->max_batch < BL) return fail(XTB_ERR_ARG, "%s: hyper holds fewer rows than a batch (%lld)", fn, BL);
  // [fc1 | gru | fc2 | hyper] in one buffer, the gradients at the same offsets
  const long long o_hyp = hyp->params - fc1->params;
  if (o_hyp < ag.o_fc2 + fc2->n_params || hyp->grads != fc1->grads + o_hyp)
    return fail(XTB_ERR_ARG, "%s: nets must be bound to slices [fc1 | gru | fc2 | hyper] of one buffer, in order", fn);
  auto* q = new xtb_qmix();
  q->ag = ag; q->hyp = hyp; q->d = d; q->E = E; q->o_hyp = o_hyp; q->n_params = o_hyp + hyp->n_params;
  q->n_part = (int)((BL + QM_THREADS / 32 - 1) / (QM_THREADS / 32));
  if (int rc = agent_alloc(fn, q->ag, &q->buf, {{&q->qt, R * ag.A}, {&q->w1t, BL * n * E}, {&q->b1t, BL * E}, {&q->wft, BL * E},
                                                 {&q->vt, BL}, {&q->part, q->n_part + 2}})) {
    delete q;
    return rc;
  }
  *out = q;
  return XTB_OK;
}

extern "C" void xtb_qmix_destroy(xtb_qmix* q) {
  if (!q) return;
  drop_graphs_of(q);
  cudaDeviceSynchronize();
  cudaFree(q->buf);
  delete q;
}

static int qmix_train_launch(xtb_qmix* q, xtb_adam* opt, const float* target, const xtb_qmix_batch& b, float* loss_out, cudaStream_t st) {
  QmixAgent& a = q->ag;
  const int A = a.A, E = q->E, n = a.n, R = a.R, BL = a.BL;
  xtb_net *fc1 = a.fc1, *fc2 = a.fc2, *hyp = q->hyp;
  const unsigned heads = (1u << kQw1) | (1u << kQb1) | (1u << kQwf) | (1u << kQv);
  // target mixer's hypernetworks on the next states (kept), then the eval ones on the states
  int rc = net_forward_impl(hyp, target + q->o_hyp, b.next_state, nullptr, BL, st, 0u, heads);
  if (rc) return rc;
  const std::pair<int, float*> tcopy[] = {{kQw1, q->w1t}, {kQb1, q->b1t}, {kQwf, q->wft}, {kQv, q->vt}};
  for (const auto& c : tcopy)
    CUDA_TRY(cudaMemcpyAsync(c.second, xtb_net_tensor(hyp, c.first), (size_t)BL * hyp->tsize[c.first] * sizeof(float),
                             cudaMemcpyDeviceToDevice, st));
  rc = net_forward_impl(hyp, nullptr, b.state, nullptr, BL, st, 0u, heads);
  if (rc) return rc;
  // target agent (Q kept), then the eval agent with the activations of its backward
  rc = qmix_agent_forward(a, target, b.obs, R, a.T, b.seq_len, nullptr, nullptr, 0, st);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(q->qt, xtb_net_tensor(fc2, 1), (size_t)R * A * sizeof(float), cudaMemcpyDeviceToDevice, st));
  rc = qmix_agent_forward(a, nullptr, b.obs, R, a.T, b.seq_len, nullptr, nullptr, 1, st);
  if (rc) return rc;
  // mixers, TD loss and the gradients wrt the chosen Q and the hypernet outputs
  float* dq = xtb_net_tensor_grad(fc2, 1);
  float* msum = q->part + q->n_part;
  CUDA_TRY(cudaMemsetAsync(dq, 0, (size_t)R * A * sizeof(float), st));
  XLAUNCH(qmix_mask_sum_kernel, 1, QM_THREADS, 0, st, b.mask, BL, msum);
  LAUNCH_CHECK();
  XLAUNCH(qmix_mix_td_kernel, q->n_part, QM_THREADS, 0, st, (const float*)xtb_net_tensor(fc2, 1), (const float*)q->qt, b.avail, b.actions,
          (const float*)xtb_net_tensor(hyp, kQw1), (const float*)xtb_net_tensor(hyp, kQb1), (const float*)xtb_net_tensor(hyp, kQwf),
          (const float*)xtb_net_tensor(hyp, kQv), (const float*)q->w1t, (const float*)q->b1t, (const float*)q->wft, (const float*)q->vt,
          b.reward, b.terminated, b.mask, (const float*)msum, a.B, a.L, n, A, E, q->d.gamma, q->d.use_double_q, dq, xtb_net_tensor_grad(hyp, kQw1),
          xtb_net_tensor_grad(hyp, kQb1), xtb_net_tensor_grad(hyp, kQwf), xtb_net_tensor_grad(hyp, kQv), q->part);
  LAUNCH_CHECK();
  XLAUNCH(qmix_loss_kernel, 1, 32, 0, st, (const float*)q->part, q->n_part, (const float*)msum, loss_out);
  LAUNCH_CHECK();
  // backward: the hypernetworks, then the agent
  const int32_t hheads[4] = {kQw1, kQb1, kQwf, kQv};
  rc = net_backward_impl(hyp, b.state, nullptr, BL, st, BackwardOpts(hheads, 4));
  if (rc) return rc;
  rc = qmix_agent_backward(a, b.obs, b.seq_len, st);
  if (rc) return rc;
  // clip_by_norm per variable + centred RMSProp over the eval set, then the nets' weight blobs
  rc = adam_step_impl(opt, fc1->params, fc1->grads, 1.f, st, nullptr);
  for (xtb_net* nt : {fc1, fc2, hyp}) if (!rc) rc = xtb_net_sync_weights(nt, st);
  return rc;
}

extern "C" int xtb_qmix_train(xtb_qmix* q, xtb_adam* opt, const float* target, const xtb_qmix_batch* batch, float* loss_out, int use_graph,
                              void* stream) {
  const char* fn = "xtb_qmix_train";
  if (!q) return fail(XTB_ERR_ARG, "%s: null object", fn);
  const bool missing = !opt || !target || !batch || !loss_out || !batch->obs || !batch->seq_len || !batch->avail || !batch->actions ||
                       !batch->state || !batch->next_state || !batch->reward || !batch->terminated || !batch->mask;
  if (int rc = learner_check(fn, missing, q->ag.fc1, opt, q->ag.R, false, q->ag.R, q->n_params)) return rc;
  if (!opt->mg) return fail(XTB_ERR_ARG, "%s: the optimiser must be centred RMSProp (xtb_opt_use_rmsprop)", fn);
  const xtb_qmix_batch b = *batch;
  return run_graph(capture_key(kQmixTrain, {q->ag.fc1, q->ag.fc2, q->hyp, q, opt}, q, target, b.obs, b.seq_len, b.avail, b.actions,
                               b.state, b.next_state, b.reward, b.terminated, b.mask, loss_out),
                   use_graph, stream, [&](void* st) { return qmix_train_launch(q, opt, target, b, loss_out, S(st)); });
}

extern "C" int xtb_qmix_infer(xtb_qmix* q, const float* explore, const float* obs, float* hidden, float* q_out, int use_graph, void* stream) {
  if (!q) return fail(XTB_ERR_ARG, "xtb_qmix_infer: null object");
  return agent_infer("xtb_qmix_infer", kQmixInfer, {q->ag.fc1, q->ag.fc2, q->hyp, q}, q, q->ag, explore, obs, hidden, q_out, use_graph,
                     stream);
}

extern "C" int xtb_qmix_act(xtb_qmix* q, const float* explore, int n_envs, int obs_last_action, int obs_agent_id, const float* obs,
                            const int32_t* avail, const int32_t* reset, const double* epsilon, const double* uniforms,
                            unsigned long long seed, unsigned long long* counter, float* hidden, int32_t* last_action, int32_t* actions,
                            int use_graph, void* stream) {
  if (!q) return fail(XTB_ERR_ARG, "xtb_qmix_act: null object");
  return agent_act("xtb_qmix_act", kQmixAct, {q->ag.fc1, q->ag.fc2, q->hyp, q}, q, q->ag, explore, n_envs, obs_last_action, obs_agent_id,
                   obs, avail, reset, epsilon, uniforms, seed, counter, hidden, last_action, actions, use_graph, stream);
}

// ---- SCC (xt/model/scc/scc_tf.py) ------------------------------------------------------------------------------------
// The agent is QMIX's; the critic's hidden layers are engine nets, one per agent group (multi-channel) or one over the
// whole row, bound to slices of the eval set after fc2; the target critic is read through their foreign-parameter
// forward.  See scc.cuh for the critic layout.
struct xtb_scc {
  QmixAgent ag;
  xtb_net* cn[SCC_MAX_GROUPS] = {};
  xtb_scc_desc d{};
  int ncn = 0, multi = 0, concat = 0, U = 0, D = 0, o = 0, mc = 1, V = 0, C = 0, K = 0, n_part = 0, n_chunk = 0;
  int a0[SCC_MAX_GROUPS + 1] = {};
  long long o_mix = 0, o_head = 0, o_cn[SCC_MAX_GROUPS] = {}, agent_size = 0, n_params = 0;
  void* buf = nullptr;
  float *xs = nullptr, *xm = nullptr, *ht = nullptr, *hm = nullptr, *dv = nullptr, *part = nullptr, *hpart = nullptr;
};

// critic rows of group j (channel rows of the multi-channel critic, whole rows of the single-channel one) for `rows` states
static inline long long scc_rows(const xtb_scc* q, int j, long long rows) { return q->multi ? rows * (q->a0[j + 1] - q->a0[j]) : rows; }
// SccH over a group-major buffer of `rows` states, U floats per channel row
static SccH scc_groups(const xtb_scc* q, const float* base, long long rows, int width) {
  SccH h{};
  h.ng = q->ncn;
  for (int j = 0; j <= q->ncn; j++) h.a0[j] = q->a0[j];
  for (int j = 0; j < q->ncn; j++) h.h[j] = base + (q->multi ? rows * q->a0[j] : 0) * width;
  return h;
}
// SccH over the nets' own second-layer outputs (or their gradients)
static SccH scc_nets(const xtb_scc* q, bool grad) {
  SccH h{};
  h.ng = q->ncn;
  for (int j = 0; j <= q->ncn; j++) h.a0[j] = q->a0[j];
  for (int j = 0; j < q->ncn; j++) h.h[j] = grad ? xtb_net_tensor_grad(q->cn[j], 2) : xtb_net_tensor(q->cn[j], 2);
  return h;
}

extern "C" int xtb_scc_create(xtb_net* fc1, xtb_net* fc2, xtb_net* const* critic, const xtb_scc_desc* desc, xtb_scc** out) {
  const char* fn = "xtb_scc_create";
  if (!fc1 || !fc2 || !critic || !desc || !out) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  const xtb_scc_desc& d = *desc;
  const int n = d.n_agents;
  if (d.n_groups < 0 || d.n_groups > SCC_MAX_GROUPS) return fail(XTB_ERR_ARG, "%s: n_groups %d not in [0, %d]", fn, d.n_groups, SCC_MAX_GROUPS);
  const int ncn = d.n_groups ? d.n_groups : 1;
  int a0[SCC_MAX_GROUPS + 1] = {0};
  if (d.n_groups) {
    for (int j = 0; j < d.n_groups; j++) {
      if (d.group[j] < 1) return fail(XTB_ERR_ARG, "%s: group %d has %d agents", fn, j, d.group[j]);
      a0[j + 1] = a0[j] + d.group[j];
    }
    if (a0[d.n_groups] != n) return fail(XTB_ERR_ARG, "%s: the groups hold %d agents, not n_agents %d", fn, a0[d.n_groups], n);
  } else {
    a0[1] = 1;
  }
  if (d.n_groups && d.channel_merge != 0 && d.channel_merge != 1)
    return fail(XTB_ERR_ARG, "%s: channel_merge %d is neither concat (0) nor add (1)", fn, d.channel_merge);
  if (n > 2 && d.mc_sample_times < 1) return fail(XTB_ERR_ARG, "%s: mc_sample_times %d < 1", fn, d.mc_sample_times);
  QmixAgent ag;
  if (int rc = agent_plan(fn, fc1, fc2, d.batch, d.episode_limit, n, d.gru_off, d.act_envs, &ag)) return rc;
  for (int j = 0; j < ncn; j++)
    if (!critic[j] || !critic[j]->ws || !critic[j]->params || !critic[j]->grads) return fail(XTB_ERR_STATE, "%s: every net must be bound", fn);
  const int A = ag.A;
  const int U = critic[0]->L.empty() ? 0 : critic[0]->tsize[1];
  const int in_w = critic[0]->tsize[0];
  const int D = d.n_groups ? in_w : in_w / n, o = D - A;
  for (int j = 0; j < ncn; j++) {
    const xtb_net* c = critic[j];
    if (c->L.size() != 2 || !dense_layer(c, 0, 0, XTB_ACT_RELU) || !dense_layer(c, 1, 1, XTB_ACT_RELU) || c->desc.input_u8 ||
        c->desc.scale != 1.f || c->tsize[1] != U || c->tsize[2] != U || c->tsize[0] != in_w)
      return fail(XTB_ERR_ARG, "%s: every critic net must be dense(U, relu) -> dense(U, relu) on the same float input", fn);
  }
  if (U < 1 || U > SCC_MAX_UNITS) return fail(XTB_ERR_ARG, "%s: dense_unit_number %d not in [1, %d]", fn, U, SCC_MAX_UNITS);
  if (o < 0 || (!d.n_groups && in_w != n * D))
    return fail(XTB_ERR_ARG, "%s: critic input %d is not n_agents x (obs + n_actions %d)", fn, in_w, A);
  const long long BL = ag.BL;
  const int V = d.n_groups ? 0 : (n <= 2 ? n : 2 * n * d.mc_sample_times);
  if (BL * n * std::max(D, U) * std::max(V, 1) > (1LL << 30)) return fail(XTB_ERR_ARG, "%s: batch too large", fn);
  if (int rc = agent_capacity(fn, ag)) return rc;
  for (int j = 0; j < ncn; j++) {
    const long long need = d.n_groups ? BL * (a0[j + 1] - a0[j]) : BL * std::max(V, 1);
    if (critic[j]->max_batch < need) return fail(XTB_ERR_ARG, "%s: critic net %d holds fewer than %lld rows", fn, j, need);
  }
  // [fc1 | gru | fc2 | critic nets | head kernel, head bias] in one buffer, the gradients at the same offsets
  const int C = d.n_groups ? n : 1, concat = d.n_groups ? d.channel_merge == 0 : 1, K = concat ? C * U : U;
  bool ok = true;
  long long prev = ag.o_fc2 + fc2->n_params, o_cn[SCC_MAX_GROUPS] = {};
  for (int j = 0; j < ncn && ok; j++) {
    o_cn[j] = critic[j]->params - fc1->params;
    ok = o_cn[j] >= prev && critic[j]->grads == fc1->grads + o_cn[j] && o_cn[j] % 4 == 0;
    prev = o_cn[j] + critic[j]->n_params;
  }
  if (!ok || d.head_off < prev || d.head_off % 4 != 0)
    return fail(XTB_ERR_ARG, "%s: nets must be bound to slices [fc1 | gru | fc2 | critic nets | head] of one buffer, in order", fn);
  auto* q = new xtb_scc();
  q->ag = ag; q->d = d;
  for (int j = 0; j < ncn; j++) { q->cn[j] = critic[j]; q->o_cn[j] = o_cn[j]; }
  for (int j = 0; j <= ncn; j++) q->a0[j] = a0[j];
  q->ncn = ncn; q->multi = d.n_groups > 0; q->concat = concat; q->U = U; q->D = D; q->o = o; q->mc = std::max(1, d.mc_sample_times);
  q->V = V; q->C = C; q->K = K;
  q->o_mix = o_cn[0]; q->o_head = d.head_off; q->agent_size = ag.o_fc2 + fc2->n_params;
  q->n_params = d.head_off + K + 1;
  q->n_part = (int)((BL + SCC_THREADS / 32 - 1) / (SCC_THREADS / 32));
  q->n_chunk = (int)((BL + SCC_HG_ROWS - 1) / SCC_HG_ROWS);
  const long long xm_n = q->multi ? BL * n * D : BL * n * D * V, hm_n = q->multi ? BL * n * U : BL * U * V;
  if (int rc = agent_alloc(fn, q->ag, &q->buf, {{&q->xs, BL * n * D}, {&q->xm, std::max(xm_n, 1LL)}, {&q->ht, BL * C * U},
                                                 {&q->hm, std::max(hm_n, 1LL)}, {&q->dv, BL}, {&q->part, 2LL * q->n_part + 2},
                                                 {&q->hpart, (long long)q->n_chunk * (K + 1)}})) {
    delete q;
    return rc;
  }
  *out = q;
  return XTB_OK;
}

extern "C" void xtb_scc_destroy(xtb_scc* q) {
  if (!q) return;
  drop_graphs_of(q);
  cudaDeviceSynchronize();
  cudaFree(q->buf);
  delete q;
}

static unsigned scc_grid(long long total) { return (unsigned)std::min<long long>((total + 255) / 256, 8LL * kSMs); }

static int scc_train_launch(xtb_scc* q, xtb_adam* copt, xtb_adam* aopt, const float* target, const xtb_scc_batch& b, float* loss_out,
                            cudaStream_t st) {
  QmixAgent& a = q->ag;
  const int n = a.n, A = a.A, U = q->U, BL = a.BL, R = a.R;
  // critic inputs (shifted), sum of the mask
  XLAUNCH(scc_inputs_kernel, scc_grid((long long)BL * n * q->D), 256, 0, st, b.raw_obs, b.actions, b.subsets, q->xs, q->xm, a.B, a.L, n,
          q->o, A, q->multi, q->mc, scc_groups(q, nullptr, BL, q->D));
  LAUNCH_CHECK();
  float* msum = q->part + 2 * q->n_part;
  XLAUNCH(qmix_mask_sum_kernel, 1, QM_THREADS, 0, st, b.mask, BL, msum);
  LAUNCH_CHECK();
  // per critic net: the target on the full rows, the eval on the credit rows (both kept), the eval on the full rows
  const SccH xs = scc_groups(q, q->xs, BL, q->D), xm = scc_groups(q, q->xm, BL, q->D);
  const SccH ht = scc_groups(q, q->ht, BL, U), hm = scc_groups(q, q->hm, BL, U);
  for (int j = 0; j < q->ncn; j++) {
    xtb_net* c = q->cn[j];
    const long long rows = scc_rows(q, j, BL), mrows = q->multi ? rows : (long long)BL * q->V;
    int rc = net_forward_impl(c, target + q->o_cn[j], xs.h[j], nullptr, (int)rows, st, 0u, 1u << 2);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync((float*)ht.h[j], xtb_net_tensor(c, 2), (size_t)rows * U * sizeof(float), cudaMemcpyDeviceToDevice, st));
    rc = net_forward_impl(c, nullptr, xm.h[j], nullptr, (int)mrows, st, 0u, 1u << 2);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync((float*)hm.h[j], xtb_net_tensor(c, 2), (size_t)mrows * U * sizeof(float), cudaMemcpyDeviceToDevice, st));
    rc = net_forward_impl(c, nullptr, xs.h[j], nullptr, (int)rows, st, 0u, 1u << 2);
    if (rc) return rc;
  }
  // the eval agent with the activations of its backward
  int rc = qmix_agent_forward(a, nullptr, b.obs, R, a.T, b.seq_len, nullptr, nullptr, 1, st);
  if (rc) return rc;
  // critic head, TD loss, credits, actor loss and their gradients
  float* dq = xtb_net_tensor_grad(a.fc2, 1);
  CUDA_TRY(cudaMemsetAsync(dq, 0, (size_t)R * A * sizeof(float), st));
  const float* P = a.fc1->params;
  SccStep sp{scc_nets(q, false), ht, hm, (long long)BL * U, scc_nets(q, true)};
  XLAUNCH(scc_step_kernel, q->n_part, SCC_THREADS, 0, st, sp, P + q->o_head, target + q->o_head, (const float*)xtb_net_tensor(a.fc2, 1),
          b.actions, b.reward, b.terminated, b.mask, (const float*)msum, a.B, a.L, n, A, U, q->concat, q->multi, q->mc, q->d.gamma,
          q->dv, dq, q->part);
  LAUNCH_CHECK();
  XLAUNCH(scc_head_grad_kernel, dim3(q->n_chunk, (q->K + 1 + 127) / 128), 128, 0, st, sp.eh, (const float*)q->dv, BL, U, q->concat,
          q->hpart);
  LAUNCH_CHECK();
  XLAUNCH(scc_reduce_kernel, (q->K + 2 + 127) / 128, 128, 0, st, (const float*)q->hpart, q->n_chunk, q->K, a.fc1->grads + q->o_head,
          (const float*)q->part, q->n_part, (const float*)msum, n, loss_out);
  LAUNCH_CHECK();
  // backward: the critic nets, then the agent
  const int32_t two[1] = {2};
  for (int j = 0; j < q->ncn; j++) {
    rc = net_backward_impl(q->cn[j], xs.h[j], nullptr, (int)scc_rows(q, j, BL), st, BackwardOpts(two, 1));
    if (rc) return rc;
  }
  rc = qmix_agent_backward(a, b.obs, b.seq_len, st);
  if (rc) return rc;
  // Adam over the critic slice, RMSProp over the agent slice (each with its clip_by_norm), then the nets' weight blobs
  rc = adam_step_impl(copt, a.fc1->params + q->o_mix, a.fc1->grads + q->o_mix, 1.f, st, nullptr);
  if (!rc) rc = adam_step_impl(aopt, a.fc1->params, a.fc1->grads, 1.f, st, nullptr);
  for (int j = 0; j < q->ncn && !rc; j++) rc = xtb_net_sync_weights(q->cn[j], st);
  for (xtb_net* nt : {a.fc1, a.fc2}) if (!rc) rc = xtb_net_sync_weights(nt, st);
  return rc;
}

// xtb_scc_train's and xtb_scc_replay_train's checks of the object and both optimisers
static int scc_learner_check(const char* fn, const xtb_scc* q, bool missing, const xtb_adam* critic_opt, const xtb_adam* actor_opt) {
  if (int rc = learner_check(fn, missing, q->ag.fc1, actor_opt, q->ag.R, false, q->ag.R, q->agent_size)) return rc;
  if (critic_opt->count != q->n_params - q->o_mix)
    return fail(XTB_ERR_ARG, "%s: critic optimiser size %lld != %lld", fn, critic_opt->count, q->n_params - q->o_mix);
  if (critic_opt->mg || critic_opt->rms_plain) return fail(XTB_ERR_ARG, "%s: the critic optimiser must be Adam", fn);
  if (!actor_opt->rms_plain) return fail(XTB_ERR_ARG, "%s: the actor optimiser must be uncentred RMSProp (xtb_opt_use_rmsprop_plain)", fn);
  return XTB_OK;
}

extern "C" int xtb_scc_train(xtb_scc* q, xtb_adam* critic_opt, xtb_adam* actor_opt, const float* target, const xtb_scc_batch* batch,
                             float* loss_out, int use_graph, void* stream) {
  const char* fn = "xtb_scc_train";
  if (!q) return fail(XTB_ERR_ARG, "%s: null object", fn);
  const bool missing = !critic_opt || !actor_opt || !target || !batch || !loss_out || !batch->obs || !batch->raw_obs || !batch->seq_len ||
                       !batch->actions || !batch->reward || !batch->terminated || !batch->mask || (!q->multi && q->ag.n > 2 && !batch->subsets);
  if (int rc = scc_learner_check(fn, q, missing, critic_opt, actor_opt)) return rc;
  const xtb_scc_batch b = *batch;
  return run_graph(capture_key(kSccTrain, {q->ag.fc1, q->cn[0], q, critic_opt, actor_opt}, q, target, b.obs, b.raw_obs, b.seq_len,
                               b.actions, b.reward, b.terminated, b.mask, b.subsets, loss_out),
                   use_graph, stream, [&](void* st) { return scc_train_launch(q, critic_opt, actor_opt, target, b, loss_out, S(st)); });
}

extern "C" int xtb_scc_infer(xtb_scc* q, const float* explore, const float* obs, float* hidden, float* q_out, int use_graph, void* stream) {
  if (!q) return fail(XTB_ERR_ARG, "xtb_scc_infer: null object");
  return agent_infer("xtb_scc_infer", kSccInfer, {q->ag.fc1, q->ag.fc2, q}, q, q->ag, explore, obs, hidden, q_out, use_graph, stream);
}

extern "C" int xtb_scc_act(xtb_scc* q, const float* explore, int n_envs, int obs_last_action, int obs_agent_id, const float* obs,
                           const int32_t* avail, const int32_t* reset, const double* epsilon, const double* uniforms,
                           unsigned long long seed, unsigned long long* counter, float* hidden, int32_t* last_action, int32_t* actions,
                           int use_graph, void* stream) {
  if (!q) return fail(XTB_ERR_ARG, "xtb_scc_act: null object");
  return agent_act("xtb_scc_act", kSccAct, {q->ag.fc1, q->ag.fc2, q}, q, q->ag, explore, n_envs, obs_last_action, obs_agent_id, obs,
                   avail, reset, epsilon, uniforms, seed, counter, hidden, last_action, actions, use_graph, stream);
}

extern "C" int xtb_scc_critic(xtb_scc* q, const float* states, int rows, float* v_out, int use_graph, void* stream) {
  const char* fn = "xtb_scc_critic";
  if (!q) return fail(XTB_ERR_ARG, "%s: null object", fn);
  if (int rc = learner_check(fn, !states || !v_out, q->ag.fc1, nullptr, rows, true, q->ag.BL)) return rc;
  return run_graph(capture_key(kSccCritic, {q->ag.fc1, q->cn[0], q}, q, states, rows, v_out), use_graph, stream, [&](void* sv) -> int {
    cudaStream_t st = S(sv);
    const float* in = states;
    const int n = q->ag.n;
    if (q->multi) {
      XLAUNCH(scc_split_kernel, scc_grid((long long)rows * n * q->D), 256, 0, st, states, q->xs, rows, n, q->D,
              scc_groups(q, nullptr, rows, q->D));
      LAUNCH_CHECK();
      in = q->xs;
    }
    const SccH xs = scc_groups(q, in, rows, q->D);
    for (int j = 0; j < q->ncn; j++) {
      int rc = net_forward_impl(q->cn[j], nullptr, xs.h[j], nullptr, (int)scc_rows(q, j, rows), st, 0u, 1u << 2);
      if (rc) return rc;
    }
    XLAUNCH(scc_value_kernel, (rows + SCC_THREADS / 32 - 1) / (SCC_THREADS / 32), SCC_THREADS, 0, st, scc_nets(q, false),
            (const float*)(q->ag.fc1->params + q->o_head), rows, q->U, q->concat, v_out);
    LAUNCH_CHECK();
    return XTB_OK;
  });
}

// ---- QMIX / SCC episode replay (episode_replay.cuh) -------------------------------------------------------------------
// The ring and the drawn ids are one device allocation; `count` mirrors the stored slots so that a draw past them is
// refused before a launch.
struct xtb_episode_replay {
  EprDev d{};
  int capacity = 0, count = 0;
  void* buf = nullptr;
  int32_t* ids = nullptr;   // [capacity] the episode ids of the current call
};

extern "C" int xtb_episode_replay_create(int capacity, int episode_limit, int n_agents, int n_actions, int obs_dim, int state_dim,
                                         int obs_last_action, int obs_agent_id, xtb_episode_replay** out) {
  const char* fn = "xtb_episode_replay_create";
  if (!out) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (capacity < 1 || episode_limit < 1 || n_agents < 1 || n_agents > QM_MAX_AGENTS || n_actions < 1 || n_actions > 255 ||
      obs_dim < 0 || state_dim < 1 || (obs_last_action != 0 && obs_last_action != 1) || (obs_agent_id != 0 && obs_agent_id != 1))
    return fail(XTB_ERR_ARG, "%s: capacity %d / episode_limit %d / n_agents %d / n_actions %d / obs_dim %d / state_dim %d / switches %d %d "
                "out of range", fn, capacity, episode_limit, n_agents, n_actions, obs_dim, state_dim, obs_last_action, obs_agent_id);
  EprDev d{};
  d.T = episode_limit + 1; d.n = n_agents; d.o = obs_dim; d.S = state_dim; d.A = n_actions;
  d.last_action = obs_last_action; d.agent_id = obs_agent_id;
  d.width = obs_dim + (obs_last_action ? n_actions : 0) + (obs_agent_id ? n_agents : 0);
  const long long row = epr_layout(d);
  if (row > (1LL << 40) / capacity) return fail(XTB_ERR_ARG, "%s: %d episodes of %lld bytes are too large", fn, capacity, row);
  auto* r = new xtb_episode_replay();
  r->d = d;
  if (int rc = carve_scratch(fn, &r->buf, {{&r->d.ring, capacity * row}, {&r->ids, (long long)capacity}})) {
    delete r;
    return rc;
  }
  r->capacity = capacity;
  *out = r;
  return XTB_OK;
}

extern "C" void xtb_episode_replay_destroy(xtb_episode_replay* r) {
  if (!r) return;
  drop_graphs_of(r);
  cudaDeviceSynchronize();
  cudaFree(r->buf);
  delete r;
}

extern "C" long long xtb_episode_replay_row_bytes(const xtb_episode_replay* r) { return r ? r->d.row_bytes : 0; }

static int epr_check(const char* fn, const xtb_episode_replay* r, bool missing) {
  if (!r || missing) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (g_comm) return fail(XTB_ERR_STATE, "%s: data-parallel training (communicator) is not supported", fn);
  return XTB_OK;
}

extern "C" int xtb_episode_replay_add(xtb_episode_replay* r, int slot, const void* row, long long bytes, void* stream) {
  const char* fn = "xtb_episode_replay_add";
  if (int rc = epr_check(fn, r, !row)) return rc;
  const EprDev& d = r->d;
  if (slot < 0 || slot >= r->capacity) return fail(XTB_ERR_ARG, "%s: slot %d not in [0, %d)", fn, slot, r->capacity);
  if (bytes != d.row_bytes) return fail(XTB_ERR_ARG, "%s: a row is %lld bytes, not %lld", fn, d.row_bytes, bytes);
  // the batch reads the actions as indices and the filled sum as a sequence length: both are checked here
  const uint8_t* h = static_cast<const uint8_t*>(row);
  for (long long i = 0; i < (long long)(d.T - 1) * d.n; i++) {
    int32_t a;
    memcpy(&a, h + d.o_act + 4 * i, 4);
    if (a < 0 || a >= d.A) return fail(XTB_ERR_ARG, "%s: action %d not in [0, %d)", fn, a, d.A);
  }
  uint64_t sum = 0;   // int64 addition wraps as NumPy's does
  for (int t = 0; t < d.T; t++) {
    int64_t f;
    memcpy(&f, h + d.o_filled + 8 * t, 8);
    sum += (uint64_t)f;
  }
  if ((int64_t)sum < 0 || (int64_t)sum > d.T) return fail(XTB_ERR_ARG, "%s: filled sums to %lld, not in [0, %d]", fn, (long long)(int64_t)sum, d.T);
  CUDA_TRY(xtb::Stager::instance().stage_h2d(d.ring + (long long)slot * d.row_bytes, row, (size_t)bytes, S(stream)));
  r->count = std::max(r->count, slot + 1);
  return XTB_OK;
}

// B ids, each a stored slot, into the replay's id buffer (one staged upload on `stream`)
static int epr_ids(const char* fn, xtb_episode_replay* r, int B, const int32_t* ids, void* stream) {
  if (B < 1 || B > r->count) return fail(XTB_ERR_ARG, "%s: batch %d not in [1, %d stored episodes]", fn, B, r->count);
  for (int b = 0; b < B; b++)
    if (ids[b] < 0 || ids[b] >= r->count) return fail(XTB_ERR_ARG, "%s: id %d not in [0, %d)", fn, ids[b], r->count);
  CUDA_TRY(xtb::Stager::instance().stage_h2d(r->ids, ids, sizeof(int32_t) * B, S(stream)));
  return XTB_OK;
}

static int epr_gather_launch(xtb_episode_replay* r, int B, const xtb_episode_batch& o, int32_t* max_t, cudaStream_t st) {
  if (o.seq_len || max_t) {
    XLAUNCH(epr_seq_len_kernel, 1, 256, 0, st, r->d, (const int32_t*)r->ids, B, o.seq_len, max_t);
    LAUNCH_CHECK();
  }
  XLAUNCH(epr_gather_kernel, dim3(r->d.T, B), kEprThreads, 0, st, r->d, (const int32_t*)r->ids, o);
  LAUNCH_CHECK();
  return XTB_OK;
}

// the replay's episodes are the agent's training batch
static int epr_agent_check(const char* fn, const xtb_episode_replay* r, const QmixAgent& a, int B) {
  if (B != a.B) return fail(XTB_ERR_ARG, "%s: batch %d is not the model's %d", fn, B, a.B);
  const EprDev& d = r->d;
  if (d.n != a.n || d.A != a.A || d.T != a.T || d.width != a.fc1->tsize[0])
    return fail(XTB_ERR_ARG, "%s: replay (%d agents, %d actions, %d steps, inputs %d wide) does not match the model (%d, %d, %d, %d)", fn,
                d.n, d.A, d.T, d.width, a.n, a.A, a.T, a.fc1->tsize[0]);
  return XTB_OK;
}

extern "C" int xtb_episode_replay_gather(xtb_episode_replay* r, int batch, const int32_t* ids, const xtb_episode_batch* out, int32_t* max_t_out,
                                         void* stream) {
  const char* fn = "xtb_episode_replay_gather";
  if (int rc = epr_check(fn, r, !ids || !out)) return rc;
  if (int rc = epr_ids(fn, r, batch, ids, stream)) return rc;
  return epr_gather_launch(r, batch, *out, max_t_out, S(stream));
}

extern "C" int xtb_qmix_replay_train(xtb_episode_replay* r, xtb_qmix* q, xtb_adam* opt, const float* target, int batch, const int32_t* ids,
                                     const xtb_qmix_batch* bufs, float* loss_out, int32_t* max_t_out, int use_graph, void* stream) {
  const char* fn = "xtb_qmix_replay_train";
  if (!q) return fail(XTB_ERR_ARG, "%s: null object", fn);
  const bool missing = !ids || !opt || !target || !bufs || !loss_out || !max_t_out || !bufs->obs || !bufs->seq_len || !bufs->avail ||
                       !bufs->actions || !bufs->state || !bufs->next_state || !bufs->reward || !bufs->terminated || !bufs->mask;
  if (int rc = epr_check(fn, r, missing)) return rc;
  if (int rc = learner_check(fn, false, q->ag.fc1, opt, q->ag.R, false, q->ag.R, q->n_params)) return rc;
  if (!opt->mg) return fail(XTB_ERR_ARG, "%s: the optimiser must be centred RMSProp (xtb_opt_use_rmsprop)", fn);
  if (int rc = epr_agent_check(fn, r, q->ag, batch)) return rc;
  if (r->d.S != q->hyp->tsize[0]) return fail(XTB_ERR_ARG, "%s: replay states are %d wide, the mixer's %d", fn, r->d.S, q->hyp->tsize[0]);
  if (int rc = epr_ids(fn, r, batch, ids, stream)) return rc;
  const xtb_qmix_batch b = *bufs;
  const xtb_episode_batch o{const_cast<float*>(b.obs), nullptr, const_cast<int32_t*>(b.seq_len), const_cast<float*>(b.avail),
                            const_cast<int32_t*>(b.actions), const_cast<float*>(b.state), const_cast<float*>(b.next_state),
                            const_cast<float*>(b.reward), const_cast<float*>(b.terminated), const_cast<float*>(b.mask)};
  return run_graph(capture_key(kQmixReplayTrain, {q->ag.fc1, q->ag.fc2, q->hyp, q, opt, r}, r, q, target, batch, b.obs, b.seq_len, b.avail,
                               b.actions, b.state, b.next_state, b.reward, b.terminated, b.mask, loss_out, max_t_out),
                   use_graph, stream, [&](void* sv) -> int {
    int rc = epr_gather_launch(r, batch, o, max_t_out, S(sv));
    return rc ? rc : qmix_train_launch(q, opt, target, b, loss_out, S(sv));
  });
}

extern "C" int xtb_scc_replay_train(xtb_episode_replay* r, xtb_scc* q, xtb_adam* critic_opt, xtb_adam* actor_opt, const float* target, int batch,
                                    const int32_t* ids, const xtb_scc_batch* bufs, float* loss_out, int32_t* max_t_out, int use_graph,
                                    void* stream) {
  const char* fn = "xtb_scc_replay_train";
  if (!q) return fail(XTB_ERR_ARG, "%s: null object", fn);
  const bool missing = !ids || !critic_opt || !actor_opt || !target || !bufs || !loss_out || !max_t_out || !bufs->obs || !bufs->raw_obs ||
                       !bufs->seq_len || !bufs->actions || !bufs->reward || !bufs->terminated || !bufs->mask ||
                       (!q->multi && q->ag.n > 2 && !bufs->subsets);
  if (int rc = epr_check(fn, r, missing)) return rc;
  if (int rc = scc_learner_check(fn, q, false, critic_opt, actor_opt)) return rc;
  if (int rc = epr_agent_check(fn, r, q->ag, batch)) return rc;
  if (r->d.o != q->o) return fail(XTB_ERR_ARG, "%s: replay observations are %d wide, the critic's %d", fn, r->d.o, q->o);
  if (int rc = epr_ids(fn, r, batch, ids, stream)) return rc;
  const xtb_scc_batch b = *bufs;
  const xtb_episode_batch o{const_cast<float*>(b.obs), const_cast<float*>(b.raw_obs), const_cast<int32_t*>(b.seq_len), nullptr,
                            const_cast<int32_t*>(b.actions), nullptr, nullptr, const_cast<float*>(b.reward), const_cast<float*>(b.terminated),
                            const_cast<float*>(b.mask)};
  return run_graph(capture_key(kSccReplayTrain, {q->ag.fc1, q->cn[0], q, critic_opt, actor_opt, r}, r, q, target, batch, b.obs, b.raw_obs,
                               b.seq_len, b.actions, b.reward, b.terminated, b.mask, b.subsets, loss_out, max_t_out),
                   use_graph, stream, [&](void* sv) -> int {
    int rc = epr_gather_launch(r, batch, o, max_t_out, S(sv));
    return rc ? rc : scc_train_launch(q, critic_opt, actor_opt, target, b, loss_out, S(sv));
  });
}

// ---- InfoFlow recommender DQN (xt/model/dqn/dqn_rec_model.py, xt/algorithm/dqn/dqn_infoflw_alg.py) -------------------
// One flat weight buffer [gru | gru_1 | dense | dense_1 | q_value] (TF variable order, every slice 256-byte aligned):
// each GRU is Keras's kernel [U, 3U], recurrent_kernel [U, 3U] and bias [3U] (gates [z | r | h]), the head (dense,
// dense_1, q_value) an engine net bound to the slice at head_off, the gradients at the same offsets.  The frozen
// embedding table lives outside it.  GRU i of S sequences runs on 5 S step rows (row s * 5 + t).  The object's scratch
// grows with the sequences (transitions, or rows of a predict) and head input rows a call needs; a growth drops the
// object's graphs.
struct xtb_infoflow {
  xtb_infoflow_desc d{};
  int U = 0, D = 0, Du = 0;
  int s_cap = 0, r_cap = 0;      // scratch capacity: GRU sequences, head input rows
  void* buf = nullptr;
  float *xs[2] = {}, *xg[2] = {}, *xc[2] = {}, *hout[2] = {}, *rh[2] = {}, *hT[2] = {}, *dy[2] = {};
  float *dag = nullptr, *dac = nullptr, *x = nullptr, *dx = nullptr, *target = nullptr;
  int32_t *len5 = nullptr, *iota = nullptr;
};

static long long if_gru_floats(long long U) { return 6 * U * U + 3 * U; }

extern "C" int xtb_infoflow_create(const xtb_infoflow_desc* desc, xtb_infoflow** out) {
  const char* fn = "xtb_infoflow_create";
  if (!desc || !out || !desc->table) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  const xtb_infoflow_desc& d = *desc;
  if (d.user_dim < 1 || d.item_dim < 1 || d.emb_dim < 1 || d.vocab < 1 || d.batch < 1)
    return fail(XTB_ERR_ARG, "%s: user_dim %d, item_dim %d, emb_dim %d, vocab %d and batch %d must be positive", fn, d.user_dim,
                d.item_dim, d.emb_dim, d.vocab, d.batch);
  if (d.last_act < XTB_ACT_NONE || d.last_act > XTB_ACT_GELU) return fail(XTB_ERR_ARG, "%s: last_act %d is not an xtb_act", fn, d.last_act);
  const long long U = (long long)d.item_dim * d.emb_dim;
  if (U > 4096 || qgru_smem_floats((int)U, 1) * 4 > kMaxDynSmem)
    return fail(XTB_ERR_ARG, "%s: item_dim x emb_dim = %lld GRU units: the GRU weights do not fit in shared memory (at most 137)", fn, U);
  const long long gn = if_gru_floats(U);
  if (d.gru_off != 0 || d.gru1_off < gn || d.head_off < d.gru1_off + gn || d.gru1_off % 64 || d.head_off % 64)
    return fail(XTB_ERR_ARG, "%s: the weights must be slices [gru | gru_1 | head] from offset 0, each 64-float aligned", fn);
  auto* f = new xtb_infoflow();
  f->d = d; f->U = (int)U; f->Du = d.user_dim * d.emb_dim; f->D = f->Du + 3 * f->U;
  *out = f;
  return XTB_OK;
}

extern "C" void xtb_infoflow_destroy(xtb_infoflow* f) {
  if (!f) return;
  drop_graphs_of(f);
  cudaDeviceSynchronize();
  cudaFree(f->buf);
  delete f;
}

// Scratch for S sequences and `rows` head input rows (grow-only; a growth drops the object's graphs)
static int if_reserve(const char* fn, xtb_infoflow* f, int S, int rows) {
  if (S <= f->s_cap && rows <= f->r_cap) return XTB_OK;
  const int sc = std::max(S, f->s_cap), rc = std::max(rows, f->r_cap);
  drop_graphs_of(f);
  CUDA_TRY(cudaDeviceSynchronize());
  cudaFree(f->buf);
  f->buf = nullptr; f->s_cap = f->r_cap = 0;
  if (int rc = gru_kernel_attrs(fn)) return rc;
  const long long R = 5LL * sc, U = f->U, D = f->D;
  std::vector<int32_t> len5(sc, IF_HIST), iota(sc + 1LL);
  for (int i = 0; i <= sc; i++) iota[i] = i;
  std::vector<Piece> pieces;
  for (int i = 0; i < 2; i++)
    pieces.insert(pieces.end(), {{&f->xs[i], R * U}, {&f->xg[i], R * 2 * U}, {&f->xc[i], R * U}, {&f->hout[i], R * U},
                                 {&f->rh[i], R * U}, {&f->hT[i], sc * U}, {&f->dy[i], R * U}});
  pieces.insert(pieces.end(), {{&f->dag, R * 2 * U}, {&f->dac, R * U}, {&f->x, (long long)rc * D}, {&f->dx, (long long)sc * D},
                               {&f->target, (long long)sc}, {&f->len5, (long long)sc, len5.data()},
                               {&f->iota, sc + 1LL, iota.data()}});
  if (int r = carve_scratch(fn, &f->buf, pieces)) return r;
  f->s_cap = sc; f->r_cap = rc;
  return XTB_OK;
}

// The head: dense (relu) on the D-wide rows, dense_1 (relu), q_value (1 wide, last_act)
static int if_head_check(const char* fn, const xtb_infoflow* f, const xtb_net* head) {
  if (!head) return fail(XTB_ERR_ARG, "%s: null head", fn);
  if (!head->ws || !head->params || !head->grads) return fail(XTB_ERR_STATE, "%s: head not bound", fn);
  if (head->L.size() != 3 || !dense_layer(head, 0, 0, XTB_ACT_RELU) || !dense_layer(head, 1, 1, XTB_ACT_RELU) ||
      !dense_layer(head, 2, 2, f->d.last_act) || head->tsize[0] != f->D || head->tsize[3] != 1 || head->desc.input_u8 ||
      head->desc.scale != 1.f)
    return fail(XTB_ERR_ARG, "%s: head must be dense (relu), dense_1 (relu), q_value (1 wide, last_act) on %d-wide float rows", fn, f->D);
  return XTB_OK;
}

// GRU i's recurrent weights in place (Keras GRU v1: recurrent_kernel [U, 3U] = [z | r | h], hard_sigmoid gates)
static GruRec if_rec(const xtb_infoflow* f, const float* W) {
  const float* rec = W + 3LL * f->U * f->U;
  return GruRec{rec, rec + 2 * f->U, 3 * f->U, 3 * f->U, f->U, 1};
}

// GRU kernels' sequences per CTA for S sequences and their shared memory
static int if_group(int U, int S, size_t* smem) {
  int g = std::max(1, std::min(8, (S + kSMs - 1) / kSMs));
  while (g > 1 && qgru_smem_floats(U, g) * 4 > kMaxDynSmem) g--;
  *smem = qgru_smem_floats(U, g) * 4;
  return g;
}

// Both GRUs of the weights P over S sequences from the ids click / noclick [S, 5 item_dim]: hT[i] = the last outputs
// (return_sequences=False); with `store`, the activations of the backward pass
static int if_grus(xtb_infoflow* f, const float* P, const int32_t* click, const int32_t* noclick, int S, int store, cudaStream_t st) {
  const int U = f->U, R = 5 * S;
  const long long n = (long long)R * U;
  XLAUNCH(infoflow_gather_kernel, (int)std::min<long long>(4 * kSMs, (2 * n + IF_THREADS - 1) / IF_THREADS), IF_THREADS, 0, st, click,
          noclick, f->d.table, n, f->d.emb_dim, f->xs[0], f->xs[1]);
  LAUNCH_CHECK();
  size_t smem = 0;
  const int g = if_group(U, S, &smem);
  for (int i = 0; i < 2; i++) {
    const float* W = P + (i ? f->d.gru1_off : f->d.gru_off);
    const float* bias = W + 6LL * U * U;
    // the input projections: x kernel[:, :2U] + bias[:2U] ([z | r]) and x kernel[:, 2U:] + bias[2U:]
    launch_gemm(ADense<float>{f->xs[i], nullptr, U}, BRowMajor{W, 3 * U}, EpiBiasAct{f->xg[i], bias, 1.f, XTB_ACT_NONE, 2 * U, nullptr, 0},
                R, 2 * U, U, false, st);
    LAUNCH_CHECK();
    launch_gemm(ADense<float>{f->xs[i], nullptr, U}, BRowMajor{W + 2 * U, 3 * U},
                EpiBiasAct{f->xc[i], bias + 2 * U, 1.f, XTB_ACT_NONE, U, nullptr, 0}, R, U, U, false, st);
    LAUNCH_CHECK();
    XLAUNCH(qmix_gru_fwd_kernel, (S + g - 1) / g, QG_THREADS, smem, st, if_rec(f, W), f->xg[i], f->xc[i], (const float*)nullptr, f->hT[i],
            f->hout[i], f->rh[i], (const int32_t*)f->len5, S, IF_HIST, 1, U, g, store);
    LAUNCH_CHECK();
  }
  return XTB_OK;
}

// Head input rows into f->x (see infoflow_rows_kernel) and the head's forward over `rows` of them
static int if_rows_forward(xtb_infoflow* f, xtb_net* head, const int32_t* user, const int32_t* item, const int32_t* off, int B, int rows,
                           cudaStream_t st) {
  XLAUNCH(infoflow_rows_kernel, std::min(4 * kSMs, (rows + IF_THREADS / 32 - 1) / (IF_THREADS / 32)), IF_THREADS, 0, st, user, item, off,
          (const float*)f->hT[0], (const float*)f->hT[1], f->d.table, B, rows, f->d.user_dim, f->d.item_dim, f->d.emb_dim, f->x);
  LAUNCH_CHECK();
  return net_forward_impl(head, nullptr, f->x, nullptr, rows, st, 0u, 1u << 3);
}

static int if_train_launch(xtb_infoflow* f, xtb_net* head, xtb_adam* opt, const xtb_infoflow_batch& b, int cap, float* loss_out,
                           float* target_out, cudaStream_t st) {
  const int B = f->d.batch, U = f->U, R = 5 * B;
  float* P = head->params - f->d.head_off;
  float* Gr = head->grads - f->d.head_off;
  // target pass (dqn_infoflw_alg.py:94-153): the online net's Q of every candidate row of the next states, the
  // next-state GRUs once per transition, then the segmented max and the TD target
  float* target = target_out ? target_out : f->target;
  int rc = XTB_OK;
  if (b.label) {
    if (target_out) CUDA_TRY(cudaMemcpyAsync(target_out, b.label, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, st));
    target = const_cast<float*>(b.label);
  } else {
    rc = if_grus(f, P, b.next_click, b.next_noclick, B, 0, st);
    if (!rc) rc = if_rows_forward(f, head, b.next_user, b.cand_item, b.cand_off, B, cap, st);
    if (rc) return rc;
    XLAUNCH(infoflow_td_kernel, (B + IF_THREADS / 32 - 1) / (IF_THREADS / 32), IF_THREADS, 0, st, (const float*)xtb_net_tensor(head, 3),
            b.cand_off, b.reward, b.done, B, f->d.gamma, target);
    LAUNCH_CHECK();
  }
  // model.fit of the one minibatch: forward, mse (the pre-update loss) and backward
  rc = if_grus(f, P, b.click, b.noclick, B, 1, st);
  if (!rc) rc = if_rows_forward(f, head, b.user, b.item, f->iota, B, B, st);
  if (rc) return rc;
  const int act = f->d.last_act;
  XLAUNCH(infoflow_mse_kernel, 1, IF_THREADS, 0, st, (const float*)xtb_net_tensor(head, 3), (const float*)target, B, act,
          act_is_ext(act) ? 0 : 1, xtb_net_tensor_grad(head, 3), loss_out);
  LAUNCH_CHECK();
  const int32_t qh[1] = {3};
  BackwardOpts o(qh, 1);
  o.heads_dy = 1u << 3;
  o.dobs = f->dx;
  rc = net_backward_impl(head, f->x, nullptr, B, st, o);
  if (rc) return rc;
  // the GRUs from the h_click / h_noclick slices of d loss / d input (the embedding is frozen: nothing flows further)
  size_t smem = 0;
  const int g = if_group(U, B, &smem);
  for (int i = 0; i < 2; i++) {
    CUDA_TRY(cudaMemcpy2DAsync(f->dy[i] + (IF_HIST - 1) * U, (size_t)IF_HIST * U * sizeof(float), f->dx + f->Du + i * U,
                               (size_t)f->D * sizeof(float), (size_t)U * sizeof(float), B, cudaMemcpyDeviceToDevice, st));
    const long long o_w = i ? f->d.gru1_off : f->d.gru_off;
    XLAUNCH(qmix_gru_bwd_kernel, (B + g - 1) / g, QG_THREADS, smem, st, if_rec(f, P + o_w), (const float*)f->xg[i], (const float*)f->xc[i],
            (const float*)f->hout[i], (const float*)f->dy[i], f->dag, f->dac, (const int32_t*)f->len5, B, IF_HIST, 1, U, g);
    LAUNCH_CHECK();
    // [kernel; recurrent_kernel; bias] gradients, [3U] columns apart: [x | h_prev | 1]^T d[z|r] into columns [0, 2U) and
    // [x | r h_prev | 1]^T d h^ into columns [2U, 3U)
    float* gw = Gr + o_w;
    launch_gemm(AGruFeat{f->xs[i], f->hout[i], U, 1, IF_HIST, 1}, BRowMajor{f->dag, 2 * U}, EpiDgrad{gw, gw, 0, 3 * U, 0, nullptr, 0},
                2 * U + 1, 2 * U, R, false, st);
    LAUNCH_CHECK();
    launch_gemm(AGruFeat{f->xs[i], f->rh[i], U, 1, IF_HIST, 0}, BRowMajor{f->dac, U}, EpiDgrad{gw + 2 * U, gw + 2 * U, 0, 3 * U, 0, nullptr, 0},
                2 * U + 1, U, R, false, st);
    LAUNCH_CHECK();
  }
  // Keras Adam over [gru | gru_1 | head], then the head's weight blobs
  rc = adam_step_impl(opt, P, Gr, 1.f, st, nullptr);
  if (!rc) rc = xtb_net_sync_weights(head, st);
  return rc;
}

extern "C" int xtb_infoflow_train(xtb_infoflow* f, xtb_net* head, xtb_adam* opt, const xtb_infoflow_batch* batch, float* loss_out,
                                  float* target_out, int use_graph, void* stream) {
  const char* fn = "xtb_infoflow_train";
  if (!f) return fail(XTB_ERR_ARG, "%s: null object", fn);
  if (int rc = if_head_check(fn, f, head)) return rc;
  const bool missing = !opt || !batch || !loss_out || !batch->user || !batch->click || !batch->noclick || !batch->item ||
                       (!batch->label && (!batch->next_user || !batch->next_click || !batch->next_noclick || !batch->cand_off ||
                                          !batch->cand_item || !batch->reward || !batch->done));
  const int B = f->d.batch;
  if (int rc = learner_check(fn, missing, head, opt, B, false, 0, f->d.head_off + head->n_params)) return rc;
  const xtb_infoflow_batch b = *batch;
  if (b.n_cand < 0 || b.cand_cap < std::max(b.n_cand, B) || b.cand_cap > head->max_batch)
    return fail(XTB_ERR_ARG, "%s: cand_cap %d must hold n_cand %d and the batch %d, and the head %d rows", fn, b.cand_cap, b.n_cand, B,
                head->max_batch);
  if (int rc = if_reserve(fn, f, B, b.cand_cap)) return rc;
  return run_graph(capture_key(kInfoflowTrain, {head, f, opt}, f, b.user, b.click, b.noclick, b.item, b.next_user, b.next_click,
                               b.next_noclick, b.cand_off, b.cand_item, b.reward, b.done, b.label, b.cand_cap, loss_out, target_out),
                   use_graph, stream, [&](void* st) { return if_train_launch(f, head, opt, b, b.cand_cap, loss_out, target_out, S(st)); });
}

extern "C" int xtb_infoflow_predict(xtb_infoflow* f, xtb_net* head, const int32_t* user, const int32_t* click, const int32_t* noclick,
                                    const int32_t* item, int n, float* q_out, int use_graph, void* stream) {
  const char* fn = "xtb_infoflow_predict";
  if (!f) return fail(XTB_ERR_ARG, "%s: null object", fn);
  if (int rc = if_head_check(fn, f, head)) return rc;
  if (int rc = learner_check(fn, !user || !click || !noclick || !item || !q_out, head, nullptr, n, true)) return rc;
  if (int rc = if_reserve(fn, f, n, n)) return rc;
  return run_graph(capture_key(kInfoflowPredict, {head, f}, f, user, click, noclick, item, n, q_out), use_graph, stream, [&](void* sv) -> int {
    cudaStream_t st = S(sv);
    const float* P = head->params - f->d.head_off;
    int rc = if_grus(f, P, click, noclick, n, 0, st);
    if (!rc) rc = if_rows_forward(f, head, user, item, f->iota, n, n, st);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(q_out, xtb_net_tensor(head, 3), (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return XTB_OK;
  });
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
extern "C" int xtb_copy_d2h(void* dst, const void* src, size_t bytes, void* stream) {
  CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, S(stream)));
  return XTB_OK;
}
extern "C" int xtb_stream_sync(void* stream) {
  CUDA_TRY(cudaStreamSynchronize(S(stream)));
  return XTB_OK;
}
