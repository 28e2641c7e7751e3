// engine.cuh -- what the engine's sources share (xtb_engine.cu, learners.cu): the native objects' structs, the process
// state and the host functions one source defines and the other calls.  The C ABI is include/xtb200.h; this header is
// private to the library.
#pragma once
#include "../../include/xtb200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <type_traits>
#include <vector>

#include "bp_tables.cuh"
#include "gemm_f32.cuh"

namespace xtb { struct AdamState; struct AdamHyper; }
using namespace xtb;

static const int kSMs = 132;                    // H100 SXM: persistent kernels size their grids to one wave
static const int kMaxDynSmem = 232448 - 3072;   // 227 KiB per CTA minus the kernels' static shared memory (<= 3 KiB)

// ---- the layer engine's plan of a net and its workspace -------------------------------------------------------------
struct LayerPlan {
  xtb_layer_desc d;
  ConvGeom g{};          // conv only
  int in_size = 0;       // floats per sample of the source tensor
  int out_size = 0;
  int K = 0, N = 0;      // weight matrix [K,N]
  long long w_off = 0, b_off = 0;
  int src_act = 0;       // activation of the producing layer of the source tensor
  int adv_act = 0;       // dueling: activation of the producing layer of the 1-wide stream (tensor d.k)
  // conv: index tables of the fp32 kernels (see ConvTabs) and their workspace offset
  std::vector<int> im2col; size_t im2col_off = 0;
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

// Which forms of a tensor's value, and of its gradient, hold the current data: bits of the fp32 row-major buffer and
// of the batch-planar planes.  Tensor 0 is the observation: its planes are the decoded-frame canvas.
enum Form : uint8_t { kNone = 0, kF32 = 1, kPlanes = 2, kBoth = 3 };
struct TensorForms { uint8_t val = kNone, grad = kNone; };

// A table built on the host by xtb_net_create and the workspace byte offset it is uploaded to by every bind
struct HostTable { size_t off; const void* data; size_t bytes; };

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
  std::vector<HostTable> tables;          // the segment table, the stage walks and the im2col tables, in the workspace
  bool any_tc = false;
  float* params = nullptr; float* grads = nullptr; char* ws = nullptr;
  std::vector<TensorForms> cur;           // per tensor: changed only by wrote() / invalidate() / ensure_f32 / ensure_bp
  std::vector<bp::RedSeg> pending;        // ordered reductions queued by the running backward pass
};

// Everything below stays inside the library: the exported names are the C ABI's xtb_* alone, so a same-named symbol
// elsewhere in the process (a `fail`, a `g_comm`) can neither bind to these nor take their place.
#pragma GCC visibility push(hidden)

// ---- errors and launch counting ---------------------------------------------------------------------------------------
extern std::atomic<long long> g_launches;   // kernels launched (or replayed in a graph): xtb_launch_count
// sets the message of xtb_last_error and returns code
int fail(int code, const char* fmt, ...);
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
inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- Scratch of the native objects ------------------------------------------------------------------------------------
// One piece of an object's device scratch: the pointer it is carved into, its length in elements of that pointer's type
// and, optionally, the host contents it starts with (otherwise zeros)
struct Piece {
  void** slot;
  size_t bytes;
  const void* init;
  template <class T> Piece(T** p, long long count, const T* init = nullptr)
      : slot(reinterpret_cast<void**>(p)), bytes((size_t)count * sizeof(T)), init(init) {}
};
// An object's scratch as one cudaMalloc into *buf, every piece 256-byte aligned and filled.  The fill runs on the legacy
// stream, which a non-blocking stream is not ordered after, so the call returns only once it is complete.  On failure
// nothing is left allocated.
int carve_scratch(const char* fn, void** buf, const std::vector<Piece>& pieces);

// ---- process state ----------------------------------------------------------------------------------------------------
extern xtb_comm* g_comm;   // installed communicator (xtb_set_grad_comm): gradients are all-reduced inside the training loops
extern int g_tc_mode;      // 1 = tensor cores where the shape is covered, 0 = fp32 CUDA-core kernels only (XTB_TC, xtb_set_tc_mode)
extern int g_fuse_heads;   // the fused heads kernels run where they apply (XTB_FUSE_HEADS, xtb_set_fuse_heads)

// ---- the layer engine -------------------------------------------------------------------------------------------------
// layer `lp` reads tensor t: through src, or as the second (1-wide) input of a dueling layer
bool reads(const LayerPlan& lp, int t);

// fp32 row-major value / gradient of tensor t, [max_batch][tsize]
float* out_f32(const xtb_net* n, int t);
float* gout_f32(const xtb_net* n, int t);
// batch-planar planes of the gradient of tensor t
bp::BpT gout_bp(const xtb_net* n, int t);
// layer lp runs on the tensor cores in the current mode
bool use_tc(const LayerPlan& lp);
// the activation whose derivative a data-gradient epilogue applies: none for the activations past tanh, whose tensors
// collect the gradient wrt their output until act_backward
int dgrad_act(const LayerPlan& lp);
// Steps per forward of rollout inference over E environments: as many as fit max_batch rows, at least one
int infer_chunk_steps(int max_batch, int E);
// Queue the ordered reduction of n_slabs per-CTA slabs (stride `slab` floats, `count` of them each) into the gradient
// bucket at dst_off, or at dst_ptr; the backward pass runs the queue in one launch.  conv: the slabs are that conv
// layer's weight-gradient accumulators [R][128][N], mapped back to its weight rows.
void queue_reduction(xtb_net* net, const float* part, int n_slabs, long long slab, int count, long long dst_off,
                     float* dst_ptr = nullptr, const LayerPlan* conv = nullptr);

// ------------------------------------------------------------------------------------------
// fp32 GEMM dispatch
// ------------------------------------------------------------------------------------------
template <int BM, int BN, int TM, int TN, class AL, class BL, class EP>
void launch_cfg(const AL& al, const BL& bl, const EP& ep, int M, int N, int K, int ksplit, cudaStream_t st) {
  constexpr int BK = 16;
  int kc = (K + ksplit - 1) / ksplit;
  kc = (kc + BK - 1) / BK * BK;
  int ks = (K + kc - 1) / kc;
  dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, ks);
  XLAUNCH((gemm_f32_kernel<BM, BN, BK, TM, TN, AL, BL, EP>), grid, (BM / TM) * (BN / TN), 0, st, al, bl, ep, M, N, K, kc);
}

// split_ok: epilogue is atomic-accumulating so K may be partitioned over gridDim.z
template <class AL, class BL, class EP>
void launch_gemm(const AL& al, const BL& bl, const EP& ep, int M, int N, int K, bool split_ok, cudaStream_t st) {
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

// ---- forward / backward -----------------------------------------------------------------------------------------------
// want_f32_mask: bit t set = tensor t is needed in fp32 row-major form (all tensors for the public entry point).
// split_rows: the rows the dense split-K forwards are planned for (tc_forward); 0 = batch
int net_forward_impl(xtb_net* net, const float* params, const void* obs, const int32_t* gather_idx, int batch, void* stream,
                     unsigned skip_mask, unsigned want_f32_mask, int split_rows = 0);
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
int net_backward_impl(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch, void* stream, const BackwardOpts& o);
// d loss / d observation is defined for float observations that only dense layers read (decode scale 1)
int input_grad_check(const xtb_net* net);

// ---- optimiser --------------------------------------------------------------------------------------------------------
struct xtb_adam {
  long long count = 0;
  float lr, beta1, beta2, eps, clip;
  int clip_mode = 0, n_seg = 0, n_blk = 0;
  float *m = nullptr, *v = nullptr;
  float* mg = nullptr; float rms_rho = 0.f, rms_eps = 0.f;   // centred RMSProp instead of Adam when mg != NULL (m = ms)
  bool rms_plain = false;                                    // uncentred RMSProp instead of Adam (m = ms, mg unused)
  int* blk_seg = nullptr; long long* blk_beg = nullptr; int* blk_len = nullptr;
  double* norm_sq = nullptr; float* seg_scale = nullptr; AdamState* st = nullptr; AdamHyper* hyp = nullptr; unsigned int* ticket = nullptr;
  void* buf = nullptr;                                       // the one allocation the pointers above are carved from
};
// one optimiser step over params / grads; net: also refresh the weight blobs of its tensor-core layers
int adam_step_impl(xtb_adam* o, float* params, const float* grads, float grad_scale, void* stream, xtb_net* net);

// ---- learner entry points ---------------------------------------------------------------------------------------------
// loss / gradient scale of the training loops that average over the local batch: 1 / world while a communicator sums
// the gradients over ranks, else 1
float dp_inv_world();
// What every learner entry point checks before it launches anything: none of the pointers it needs is NULL (`missing`:
// each caller names its own), the net is bound with gradients, the optimiser spans the trained parameters (n_params,
// 0: the net's; opt NULL: an inference call), the `rows` samples of one forward are in [1, max_rows] (0: the net's
// max_batch) and, for a learner that cannot sum its gradients over ranks (dp_ok false), no communicator is installed.
int learner_check(const char* fn, bool missing, const xtb_net* net, const xtb_adam* opt, long long rows, bool dp_ok,
                  long long max_rows = 0, long long n_params = 0);

// CUDA graphs cannot be captured on the legacy default stream, which is what a host that never creates streams
// (stream == NULL) runs on.  Such calls are moved onto a private non-blocking stream of the current device, fenced
// against the legacy stream with events on both sides, so the caller keeps default-stream ordering semantics.
struct EngineStream;
struct StreamScope {
  cudaStream_t st = nullptr;
  EngineStream* es = nullptr;
  int begin(void* stream, bool side_if_null);
  int end();
};

// ---- CUDA-graph cache of the fused entry points ------------------------------------------------
// A captured graph bakes in every kernel argument, so its key holds everything the capture reads.  capture_key()
// zeroes it and fills the entry point, the owners and the arguments; run_graph() adds the communicator and the
// modes, which every capture reads.  Keys are compared bytewise.
enum GraphTag { kPpoTrain = 1, kImpalaTrain, kDqnTrain, kRolloutInfer, kImpalaKerasFit, kImpalaKerasTrain, kMuzeroTrain,
                kMuzeroInitInfer, kMuzeroRecurInfer, kMuzeroSearch, kQmixTrain, kQmixInfer,
                kSccTrain, kSccInfer, kSccCritic, kDqnTrainWeighted, kDqnPerTrain, kInfoflowTrain, kInfoflowPredict, kMuzeroReplayTrain,
                kQmixReplayTrain, kSccReplayTrain, kQmixAct, kSccAct };
struct CaptureKey {
  uint64_t tag;          // entry point
  const void* own[7];    // the objects the capture reads (nets, optimiser, ...) and the communicator (own[6]):
                         // destroying one, or rebinding a net, drops the graph
  uint64_t mode[2];      // kernel-path and fused-heads modes
  uint64_t arg[21];      // every pointer and scalar argument; floats by bit pattern
  bool operator<(const CaptureKey& o) const { return memcmp(this, &o, sizeof(CaptureKey)) < 0; }
};
template <class T> uint64_t key_word(T v) {
  if constexpr (std::is_same_v<T, float>) { uint32_t u; memcpy(&u, &v, sizeof u); return u; }
  else if constexpr (std::is_same_v<T, double>) { uint64_t u; memcpy(&u, &v, sizeof u); return u; }
  else if constexpr (std::is_pointer_v<T>) return (uint64_t)(uintptr_t)v;
  else return (uint64_t)v;
}
template <size_t N, class... A>
CaptureKey capture_key(GraphTag tag, const void* const (&owners)[N], A... args) {
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

// The cache of captured graphs (xtb_engine.cu).  Cached graphs hold raw pointers into their owners: they die with the object (a
// later object may be allocated at the same address) and with a net's binding.
struct GraphVal { cudaGraphExec_t exec; long long kernels; };
const GraphVal* graph_find(const CaptureKey& key);
// caches a captured graph of `kernels` launches (emptying the cache first when it is full)
const GraphVal* graph_add(const CaptureKey& key, cudaGraphExec_t exec, long long kernels);
int graph_launch(const GraphVal& g, cudaStream_t st);
void drop_graphs_of(const void* obj);

// use_graph == 0: launch(stream) runs eagerly.  Otherwise the launches are captured once per key, with the global
// state every capture reads added to it, and the graph is replayed.
template <class F>
int run_graph(CaptureKey key, int use_graph, void* stream, F&& launch) {
  if (!use_graph) return launch(stream);
  key.own[6] = g_comm; key.mode[0] = g_tc_mode; key.mode[1] = g_fuse_heads;
  StreamScope sc;
  int src = sc.begin(stream, true);
  if (src) return src;
  const GraphVal* g = graph_find(key);
  if (!g) {
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
    g = graph_add(key, exec, captured);
  }
  int rc = graph_launch(*g, sc.st);
  if (rc) return rc;
  return sc.end();
}

#pragma GCC visibility pop
