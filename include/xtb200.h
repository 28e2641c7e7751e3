/*
 * xtb200.h -- C-ABI of libxtb200.so, the H100 (sm_90a) engine behind XingTian's
 * Model / Algorithm plugin API.
 *
 * The reference (huawei-noah/xingtian, /root/reference) has NO native boundary:
 * its hot path is Python composing TensorFlow-1.15 ops.  Each entry point below
 * names the reference Python interface it replaces (file:line, relative to the
 * reference root).  All pointers are plain device pointers unless the name ends
 * in `_host`; sizes are element counts unless they say bytes; `stream` is a
 * cudaStream_t passed as void* (NULL = legacy default stream).  Storage is
 * caller-owned (the Python host allocates it as torch.Tensor storage); the
 * library never frees caller memory.  Every function returns 0 on success and a
 * negative xtb_status otherwise; xtb_last_error() gives the thread-local message
 * (the Python shim raises RuntimeError with it -- reference behaviour: exceptions
 * propagate, xt/train.py:159-178).
 */
#ifndef XTB200_H_
#define XTB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XTB_VERSION 101

enum xtb_status {
  XTB_OK = 0,
  XTB_ERR_ARG = -1,     /* bad argument / unsupported configuration */
  XTB_ERR_CUDA = -2,    /* a CUDA runtime call or kernel launch failed */
  XTB_ERR_STATE = -3,   /* object not bound / wrong call order */
  XTB_ERR_NOMEM = -4
};

enum xtb_layer_kind { XTB_CONV = 0, XTB_DENSE = 1, XTB_DUELING = 2, XTB_LOGSTD = 3 };
/* Hidden-layer activations: the keys of ACTIVATION_MAP (xt/model/model_utils.py:8-19) with TF 1.15's semantics, plus
 * NONE (linear).  xtb_net_create rejects any other value with XTB_ERR_ARG.
 *   SIGMOID    1 / (1 + e^-x)                                   tf.math.sigmoid
 *   SOFTSIGN   x / (1 + |x|)                                    tf.nn.softsign
 *   SOFTPLUS   log(1 + e^x) = max(x, 0) + log1p(e^-|x|)         tf.nn.softplus
 *   LEAKY_RELU x > 0 ? x : 0.2 x                                tf.nn.leaky_relu (default alpha 0.2)
 *   ELU        x > 0 ? x : e^x - 1                              tf.nn.elu (alpha 1)
 *   SELU       1.0507009873554805 * (x > 0 ? x : 1.6732632423543772 (e^x - 1))   tf.nn.selu
 *   SWISH      x * sigmoid(x)                                   tf.nn.swish
 *   GELU       0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))  the reference's tanh form, xt/model/tf_utils.py:157-166
 * The GEMM epilogues apply RELU, TANH and NONE.  A layer with one of the others runs its GEMM linear into fp32 and one
 * elementwise launch applies the activation; the backward sums the gradients of its consumers wrt its output and one
 * elementwise launch multiplies by the derivative.  That derivative is taken from the output y, except for SOFTSIGN,
 * SWISH and GELU, which y does not determine well (or at all): their layers keep the pre-activation in a workspace
 * buffer of their own, written by every forward (xtb_net_workspace_bytes includes it).  A dueling layer reads only
 * RELU / TANH / NONE tensors. */
enum xtb_act {
  XTB_ACT_NONE = 0, XTB_ACT_RELU = 1, XTB_ACT_TANH = 2, XTB_ACT_SIGMOID = 3, XTB_ACT_SOFTSIGN = 4, XTB_ACT_SOFTPLUS = 5,
  XTB_ACT_LEAKY_RELU = 6, XTB_ACT_ELU = 7, XTB_ACT_SELU = 8, XTB_ACT_SWISH = 9, XTB_ACT_GELU = 10
};

#define XTB_MAX_LAYERS 16

/* One Keras layer of the reference networks.
 * conv : Conv2D(cout, (k,k), strides=(stride,stride), padding = pad_same ? 'same' : 'valid')
 *        NHWC activations, HWIO kernel  (xt/model/model_utils.py:91-97,
 *        xt/model/impala/impala_cnn_opt.py:120-137, xt/model/dqn/dqn_cnn.py:49-51)
 * dense: Dense(n) on the HWC-flattened source (model_utils.py:83-88, :63-65)
 * dueling: the dueling Q combine of DqnCnn / DqnMlp with model_config {dueling: True} (xt/model/dqn/dqn_cnn.py:55-58,
 *        dqn_mlp.py:51-54,80-87): Q = adv + (value - mean over actions of value).  No parameters and no activation
 *        (act must be XTB_ACT_NONE).  `src` is the A-wide "value" tensor and `k` holds the tensor id of the 1-wide "adv"
 *        tensor (the only layer kind with a second input); both must be outputs of earlier layers, never the
 *        observation, and different tensors.  The output is A wide.  xtb_net_layer_params reports 0 rows and 0 columns
 *        for it.  xtb_dqn_train runs a dueling q_tensor in one fused kernel when both streams are linear dense layers
 *        on one hidden tensor (see xtb_dqn_train).
 * logstd: the state-independent `pi_logstd` variable of PPO with action_type DiagGaussian (xt/model/ppo/ppo.py:75-78:
 *        tf.get_variable('pi_logstd', shape=(1, A), initializer=zeros)).  A parameter-only layer: it owns `cout` = A
 *        floats, reads no tensor (src must be 0) and produces none (its tensor is 0 wide, so no layer may read it and it
 *        cannot be a backward head); act must be XTB_ACT_NONE and 1 <= cout <= 32.  xtb_net_layer_params reports 1 row
 *        and A columns with bias_off = kernel_off + A (it has no bias).  It takes part in clipping, the optimiser and
 *        the gradient bucket like every other parameter; the PPO calls below read it by offset when it is their
 *        logstd_tensor. */
typedef struct xtb_layer_desc {
  int32_t kind;      /* xtb_layer_kind */
  int32_t src;       /* tensor id of the input: 0 = observation, i+1 = output of layer i */
  int32_t act;       /* xtb_act */
  int32_t k;         /* conv kernel size */
  int32_t stride;    /* conv stride (1, 2 or 4) */
  int32_t cout;      /* conv filters / dense units */
  int32_t pad_same;  /* conv: 1 = TF 'SAME' padding, 0 = 'VALID' */
} xtb_layer_desc;

typedef struct xtb_net_desc {
  int32_t input_u8;        /* 1: uint8 observation decoded as x*scale (model_utils.py:187-189); 2: int8 observation (each
                              byte b read as b < 128 ? b : b - 256, then times scale: uint8 frames fed to the int8
                              placeholder of MuzeroCnn with obs_type int8); 0: float; other values XTB_ERR_ARG */
  float scale;             /* 1/255 for uint8 Atari frames, 1 for float observations */
  int32_t in_h, in_w, in_c; /* observation HWC; vectors use 1,1,dim */
  int32_t n_layers;
  xtb_layer_desc layers[XTB_MAX_LAYERS];
} xtb_net_desc;

typedef struct xtb_net xtb_net;

/* ---- library ---------------------------------------------------------------- */
int xtb_version(void);
const char* xtb_last_error(void);
/* Number of kernels this library has launched in the calling process (all threads). */
long long xtb_launch_count(void);
/* Number of CUDA-graph replays (fused training loop / rollout inference) the library has issued. */
long long xtb_graph_replay_count(void);

/* ---- network: replaces XTModel's TF graph (xt/model/model.py:30-127) ---------- */
/* Flat fp32 parameter layout: per layer, kernel [K,N] (HWIO flattened) then bias [N];
 * identical to iterating TFVariables' ordered dict (xt/model/tf_utils.py:84-102). */
int xtb_net_create(const xtb_net_desc* desc, int max_batch, xtb_net** out);
void xtb_net_destroy(xtb_net* net);
long long xtb_net_param_count(const xtb_net* net);
/* offsets (in floats) of layer `layer`'s kernel and bias inside the flat buffer, and K,N */
int xtb_net_layer_params(const xtb_net* net, int layer, long long* kernel_off, long long* bias_off,
                         int* k_rows, int* n_cols);
/* How xtb_net_create planned layer `layer` (read-only; changes nothing that runs).  Every field but `kind` is 0 for a
 * layer on the fp32 CUDA-core kernels.  A layer planned onto the tensor cores runs there while xtb_get_tc_mode() is 1. */
typedef struct xtb_layer_plan {
  int32_t kind;           /* xtb_layer_kind after planning: a VALID conv whose window covers the whole map is dense */
  int32_t tc;             /* 1: the wgmma (tensor-core) kernels run this layer */
  int32_t s2d;            /* first layer run as a stride-1 conv over the space-to-depth canvas of uint8 frames */
  int32_t w_res;          /* conv: the weight blob stays resident in shared memory; 0: it streams through the ring */
  int32_t n_fwd, n_dg;    /* accumulator columns of a forward / data-gradient tile */
  int32_t R;              /* conv: weight-gradient accumulators (filter row x 128-feature tile) */
  int32_t fwd_stages;     /* ring stages of the forward launch */
  int32_t dg_stages;      /* ring stages of the data-gradient launch */
  int32_t dg_empty_units; /* conv: input pixels that no filter tap reaches (their data gradient is zero) */
  int32_t k_slices;       /* K slices (split-K) of a dense forward at max_batch samples; 1 for a conv */
} xtb_layer_plan;
int xtb_net_layer_plan(const xtb_net* net, int layer, xtb_layer_plan* out);
/* floats per sample of tensor `t` (0 = observation) */
int xtb_net_tensor_size(const xtb_net* net, int t);
size_t xtb_net_workspace_bytes(const xtb_net* net);
/* params/grads: [param_count] floats; workspace: xtb_net_workspace_bytes() bytes */
/* A net with tensor-core layers needs `params` 16-byte aligned (XTB_ERR_ARG otherwise). */
int xtb_net_bind(xtb_net* net, float* params, float* grads, void* workspace, size_t workspace_bytes);
/* same, with the initialisation work (workspace clear, weight blobs) ordered on `stream`; returns after it completed */
int xtb_net_bind_stream(xtb_net* net, float* params, float* grads, void* workspace, size_t workspace_bytes, void* stream);
/* Every tensor the tensor-core kernels read is kept as two bf16 planes (hi = bf16(x), lo = bf16(x-hi)) next
 * to its fp32 copy.  The planes of the bound parameters are refreshed by xtb_net_bind, by the fused training
 * loops after each optimiser step, and by this call -- which a host that writes the parameter buffer itself
 * (set_weights, target-network sync, an external optimiser step) must make before the next forward. */
int xtb_net_sync_weights(xtb_net* net, void* stream);
/* activation / activation-gradient buffer of tensor t (t>=1), [batch, tensor_size] floats */
float* xtb_net_tensor(xtb_net* net, int t);
float* xtb_net_tensor_grad(xtb_net* net, int t);
/* Forward over `batch` samples. obs: [rows, H,W,C] uint8 or float; if gather_idx != NULL sample b
 * reads observation row gather_idx[b] (the minibatch gather of xt/model/ppo/ppo.py:123-128 folded
 * into the first layer's loads).  `params` NULL = the bound parameters (else e.g. a target net,
 * xt/algorithm/dqn/dqn.py:57). */
int xtb_net_forward(xtb_net* net, const float* params, const void* obs, const int32_t* gather_idx,
                    int batch, void* stream);
/* Backward: consumes d(loss)/d(pre-activation) already written into xtb_net_tensor_grad() of the
 * head tensors, zeroes and fills the bound grads buffer.  Replaces
 * optimizer.compute_gradients (xt/model/ppo/ppo.py:99). */
int xtb_net_backward(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch,
                     const int32_t* head_tensors, int n_heads, void* stream);

/* ---- policy head: replaces CategoricalDist (xt/model/tf_dist.py:89-130) and
 *      PPO.predict's fetches (xt/model/ppo/ppo.py:104-109) ---------------------- */
/* action = argmax(logits - log(-log u)); u from `uniforms` [batch,adim] if non-NULL, else
 * Philox4x32-10(seed, offset).  logp = log-softmax(logits)[action]. */
int xtb_categorical_sample(const float* logits, int batch, int adim, const float* uniforms,
                           uint64_t seed, uint64_t offset, int32_t* action, float* logp, void* stream);
/* argmax over the last axis (DQN greedy action, xt/algorithm/algorithm.py:124-135) */
int xtb_argmax(const float* q, int batch, int adim, int32_t* action, void* stream);

/* ---- GAE: replaces PPO.data_proc (xt/agent/ppo/ppo.py:77-106) ------------------- */
/* value [E,T+1], reward [E,T], done [E,T] (uint8) -> adv, old_value, target_value [E,T].
 * sign_clip != 0 applies np.sign to rewards (xt/agent/ppo/atari_ppo.py:46). */
int xtb_gae(const float* value, const float* reward, const uint8_t* done, int n_env, int n_step,
            float gamma, float lam, int sign_clip, float* adv, float* old_value, float* target_value,
            void* stream);

/* ---- PPO loss: replaces actor_loss_with_entropy + critic_loss
 *      (xt/model/ppo/__init__.py:4-25, combined xt/model/ppo/ppo.py:87-92) --------- */
typedef struct xtb_ppo_hyper {
  float clip_ratio;   /* LOSS_CLIPPING */
  float ent_coef;     /* ENTROPY_LOSS */
  float vf_clip;      /* VF_CLIP */
  float critic_coef;  /* CRITIC_LOSS_COEF */
} xtb_ppo_hyper;
/* logits [B,A], v [B]; rollout arrays are indexed through gather_idx (NULL = identity).
 * inv_count = 1/B_global (mean over the *global* minibatch when sharded, SURVEY 8(e)).
 * Writes dlogits [B,A], dv [B]; atomically adds this minibatch's loss to *loss_out. */
int xtb_ppo_loss_grad(const float* logits, const float* v, const int32_t* gather_idx,
                      const int32_t* action, const float* old_logp, const float* adv,
                      const float* old_v, const float* target_v, int batch, int adim,
                      const xtb_ppo_hyper* hp, float inv_count, float* dlogits, float* dv,
                      float* loss_out, void* stream);

/* ---- V-trace: replaces vtrace.from_logic_outputs + vtrace_loss
 *      (xt/model/impala/vtrace.py:39-115, impala_cnn_opt.py:188-196, :299-351) ------ */
/* Flat env-major inputs [n_traj*step_len,...]; the last step of every trajectory is dropped
 * from the loss and its baseline is the bootstrap (split_batches drop_last).  Writes
 * dlogits [N,A], dbaseline [N] (zeros on dropped rows), optional vs/pg_adv [N], adds loss. */
int xtb_vtrace_loss_grad(const float* tp_logits, const float* baseline, const float* bp_logits,
                         const int32_t* action, const uint8_t* done, const float* reward,
                         int n_traj, int step_len, int adim, float gamma, float* dlogits,
                         float* dbaseline, float* vs_out, float* pg_adv_out, float* loss_out,
                         void* stream);

/* ---- DQN TD target + MSE: replaces DQN.train's target loop and Keras 'mse'
 *      (xt/algorithm/dqn/dqn.py:79-97, xt/model/dqn/dqn_cnn.py:60-61) ---------------- */
/* q [B,A] online Q(s); q_next_target [B,A]; q_next_online NULL or [B,A] (double DQN).
 * Writes dq [B,A] = 2/(B*A)*(q[b,a]-y) on the taken action, td target y [B] (optional), adds loss. */
int xtb_dqn_loss_grad(const float* q, const float* q_next_target, const float* q_next_online,
                      const int32_t* action, const float* reward, const uint8_t* done, int batch,
                      int adim, float gamma, float inv_count, float* dq, float* y_out,
                      float* loss_out, void* stream);

/* Same target/loss with the options BASELINE.json's north_star names (defaults = the reference): rows may be indexed
 * through idx (minibatch rows of a replay ring); disc != NULL is a per-row bootstrap discount (gamma^n of an n-step
 * return, 0 = the window hit a terminal step); huber_delta > 0 selects the Huber loss instead of the squared error. */
int xtb_dqn_td_loss_grad(const float* q, const float* q_next_target, const float* q_next_online, const int32_t* idx,
                         const int32_t* action, const float* reward, const uint8_t* done, const float* disc, int batch,
                         int adim, float gamma, float huber_delta, float inv_count, float* dq, float* y_out,
                         float* loss_out, void* stream);
/* n-step returns over env-major trajectories [n_env][n_step] (north_star "n-step TD-target kernel"; the reference's
 * DQN is 1-step, xt/algorithm/dqn/dqn.py:86-97): ret = sum_{k<m} gamma^k r_{t+k}, m = steps to the first terminal
 * (inclusive), n, or the end of the segment; disc = gamma^m or 0 after a terminal; last = row whose next-state
 * bootstraps; done_n = window contains a terminal. */
int xtb_nstep_returns(const float* reward, const uint8_t* done, int n_env, int n_step, int n, float gamma, float* ret,
                      float* disc, int32_t* last, uint8_t* done_n, void* stream);

/* Keras model.train_on_batch(states, y) with loss='mse' (xt/model/model.py:77-82,
 * xt/model/dqn/dqn_cnn.py:60-61): loss = mean over B*A of (q-y)^2, dq = 2*(q-y)*inv_count. */
int xtb_mse_loss_grad(const float* q, const float* y, int batch, int adim, float inv_count, float* dq,
                      float* loss_out, void* stream);
/* probs[b] = softmax(logits[b]) (the `output_actions` softmax of ImpalaMlp / ImpalaCnn.predict). */
int xtb_softmax(const float* logits, int batch, int adim, float* probs, void* stream);
/* Keras loss of ImpalaMlp / ImpalaCnn (impala_loss + value_weight * mse) on p = softmax(logits[b]) and v[b], data row
 * r = idx[b] (NULL: b) of action_mat / adv / target_v:
 *   l_b = mean_i [adv_r (-y_ri log(p_i + 1e-10)) - ent_coef (-p_i log(p_i + 1e-10))] + value_weight (v_b - target_v_r)^2
 * dlogits / dv: gradient of mean_b l_b, through log(p + 1e-10) and the softmax Jacobian.  *loss_out += loss_scale *
 * sum_b l_b, summed in a fixed order (one block, no atomics).  adim <= 32. */
int xtb_impala_keras_loss_grad(const float* logits, const float* v, const int32_t* idx, const float* action_mat,
                               const float* adv, const float* target_v, int batch, int adim, float ent_coef,
                               float value_weight, float loss_scale, float* dlogits, float* dv, float* loss_out,
                               void* stream);

/* ---- optimiser: replaces tf.train.AdamOptimizer + clip_by_global_norm
 *      (xt/model/ppo/ppo.py:97-102, impala_cnn_opt.py:198-217) and Keras
 *      Adam(clipnorm) (xt/model/dqn/dqn_cnn.py:60) ----------------------------------- */
typedef struct xtb_adam xtb_adam;
enum xtb_clip_mode { XTB_CLIP_NONE = 0, XTB_CLIP_GLOBAL_NORM = 1, XTB_CLIP_PER_TENSOR = 2 };
/* m, v: [count] floats, 16-byte aligned (caller-owned, zero-initialised by this call); seg_offsets: n_seg+1
 * non-decreasing boundaries of the tensors inside the flat buffer, from 0 to count (used by XTB_CLIP_PER_TENSOR; equal
 * neighbours make an empty tensor).  clip_mode is one of xtb_clip_mode, and clip > 0 unless it is XTB_CLIP_NONE.
 * Any other argument returns XTB_ERR_ARG before a CUDA call. */
int xtb_adam_create(long long count, float lr, float beta1, float beta2, float eps, int clip_mode,
                    float clip, const long long* seg_offsets, int n_seg, float* m, float* v,
                    xtb_adam** out);
void xtb_adam_destroy(xtb_adam* opt);
/* grad_scale multiplies the gradient before clipping (1 normally). After the call
 * *xtb_adam_grad_norm() holds the pre-clip global norm of grad_scale * grads (device float).  params and grads must be
 * 16-byte aligned (XTB_ERR_ARG, launching nothing, otherwise). */
int xtb_adam_step(xtb_adam* opt, float* params, const float* grads, float grad_scale, void* stream);
/* Same step on a bound network's parameters/gradients; the kernel also refreshes the weights' bf16 planes. */
int xtb_adam_step_net(xtb_adam* opt, xtb_net* net, float grad_scale, void* stream);
const float* xtb_adam_grad_norm(const xtb_adam* opt);
int xtb_adam_set_lr(xtb_adam* opt, float lr);
/* Keras OptimizerV2 `decay` (xt/model/impala/impala_cnn.py: Adam(lr, clipnorm=40, decay=5.12e-9)): every later Adam step
 * uses lr / (1 + decay * iterations), iterations = the steps this optimiser took before it.  Device-resident like the
 * learning rate; 0 (the default) leaves the step exactly as without it. */
int xtb_adam_set_decay(xtb_adam* opt, float decay);
/* Switch the optimiser handle to tf.train.RMSPropOptimizer(lr, decay, epsilon, centered=True) (momentum 0), the
 * `opt_type: rmsprop` branch of xt/model/impala/impala_cnn_opt.py:205-206: the `m` buffer of xtb_adam_create becomes the
 * mean-square slot and `mean_grad` (count floats, 16-byte aligned) the mean-gradient slot; this call sets them to
 * ones / zeros as TF initialises them; `v` is unused.  Clipping, chunking and the weight-blob refresh are those of the Adam step. */
int xtb_opt_use_rmsprop(xtb_adam* opt, float* mean_grad, float decay, float epsilon);

/* ---- fused learner loops -------------------------------------------------------- */
/* use_graph != 0 (xtb_ppo_train, xtb_impala_train, xtb_dqn_train, xtb_ppo_rollout_infer and xtb_ppo_predict_host built
 * on it): the call's launches are captured once as a CUDA graph and replayed.  A graph is keyed on every
 * argument plus the kernel-path mode (xtb_set_tc_mode), the fused-heads mode (xtb_set_fuse_heads) and the installed
 * communicator (xtb_set_grad_comm), so a mode change takes effect at the next call.  It is dropped when its net,
 * target net, optimiser or communicator is destroyed, or when its net is rebound (xtb_net_bind). */
/* The PPO calls (xtb_ppo_train, xtb_ppo_rollout_infer, xtb_ppo_predict_host) take the policy's heads as tensor ids:
 * pi_tensor (the logits, or the DiagGaussian mean: at most 32 wide), v_tensor (the value, 1 wide) and logstd_tensor,
 * which selects the action distribution, as PPO's action_type does (xt/model/ppo/ppo.py:62-95):
 *   0        Categorical (see xtb_categorical_sample, xtb_ppo_loss_grad); actions are int32, one per sample;
 *   > 0      DiagGaussian (see xtb_diag_gaussian_sample, xtb_ppo_gauss_loss_grad): the tensor id (layer index + 1) of an
 *            XTB_LOGSTD layer as wide as pi_tensor; actions are A floats per sample.
 * Any other value, or a logstd_tensor that is not such a layer, returns XTB_ERR_ARG before a launch.
 * Fused heads: when both heads are linear dense layers on hidden (not observation) tensors of equal width K, K is a
 * multiple of 32, and the fused-heads mode is on (xtb_set_fuse_heads), one kernel evaluates both heads --
 *   training:  with the loss and their backward, for A <= 8 and K <= 256 or A <= 4 and K <= 512; its per-block partial
 *              sums, a log_std gradient included, are reduced in block order, so with tensor-core trunk layers the
 *              step is bitwise reproducible;
 *   inference: with the draw, for A <= 8 and K <= 512.
 * Every other shape runs layer by layer (forward, the loss or sampling kernel, backward); the draws are the same. */
/* PPO.train (xt/model/ppo/ppo.py:111-132): for every minibatch slice of `perm`
 * (device int32 [n_epoch*n_sample], the host-generated np.random.shuffle order) run
 * forward, loss, backward, clip, Adam.  loss_per_step: device float [n_epoch*ceil(N/B)].  Without fused heads a
 * DiagGaussian's log_std gradient goes straight into its slot of the bound gradient buffer.
 * All launches go to `stream`. */
typedef struct xtb_ppo_rollout {
  const void* obs;            /* [N, H,W,C] uint8 / float */
  const void* action;         /* behaviour actions: int32 [N] (Categorical) or float [N, A] (DiagGaussian) */
  const float* old_logp;      /* [N] */
  const float* adv;           /* [N] */
  const float* old_v;         /* [N] */
  const float* target_v;      /* [N] */
} xtb_ppo_rollout;
int xtb_ppo_train(xtb_net* net, xtb_adam* opt, const xtb_ppo_rollout* ro, int n_sample, int batch_size, int n_epoch,
                  const int32_t* perm, const xtb_ppo_hyper* hp, int pi_tensor, int v_tensor, int logstd_tensor,
                  float* loss_per_step, int use_graph, void* stream);

/* ImpalaCnnOpt.train (xt/model/impala/impala_cnn_opt.py:251-265) as one captured step: forward over n_sample =
 * k*step_len env-major rows (rows gather_idx[b] of obs when non-NULL), in-graph V-trace + summed losses, backward,
 * clip_by_global_norm + Adam.  *loss_out += loss (device float). */
int xtb_impala_train(xtb_net* net, xtb_adam* opt, const void* obs, const int32_t* gather_idx, const float* bp_logits,
                     const int32_t* action, const uint8_t* done, const float* reward, int n_sample, int step_len,
                     float gamma, int logit_tensor, int base_tensor, float* loss_out, int use_graph, void* stream);
/* DQN.train (xt/algorithm/dqn/dqn.py:61-103) as one captured step over rows idx[0..n_sample) of a device replay ring:
 * target forward on next_obs, optional double-DQN online forward (qn_o != NULL), online forward on obs, TD target +
 * loss gradient (see xtb_dqn_td_loss_grad for disc / huber_delta), backward, per-tensor clip + Adam.
 * qn_t, qn_o: scratch [n_sample, adim].  *loss_out += loss.
 * When q_tensor is an XTB_DUELING layer whose two streams are linear dense layers reading the same hidden tensor (not
 * the observation), the hidden width K is a multiple of 32 with A <= 8 and K <= 256, or A <= 4 and K <= 512, and the
 * fused-heads mode is on (xtb_set_fuse_heads), the online forward of both streams, the combine, TD target, loss and
 * the streams' backward run as one kernel; the target and double-DQN forwards, and every other shape, go layer by layer. */
int xtb_dqn_train(xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                  const int32_t* idx, const int32_t* action, const float* reward, const uint8_t* done,
                  const float* disc, int n_sample, float gamma, float huber_delta, int q_tensor, float* qn_t,
                  float* qn_o, float* loss_out, int use_graph, void* stream);

/* IMPALA with the Keras learner (xt/algorithm/impala/impala.py, xt/model/impala/impala_mlp.py, impala_cnn.py).  The
 * policy head `logit_tensor` is the linear `output_actions` layer; its softmax is evaluated in the kernels.
 * ImpalaMlp/ImpalaCnn.train = one Keras fit epoch (batch_size fit_batch, shuffle): minibatch k holds rows
 * order[k*fit_batch ...] (device int32 [n], the host-drawn np.random.shuffle order) of obs / action_mat [n, A] (one-hot
 * y_true) / adv [n] / target_v [n]; per minibatch forward, the Keras loss (see xtb_impala_keras_loss_grad, value weight
 * 0.5), backward and the optimiser step.  *loss_out = the epoch loss: per-row loss summed over the n rows, over n.
 * Both calls return XTB_ERR_STATE, launching nothing, while a communicator is installed. */
int xtb_impala_keras_fit(xtb_net* net, xtb_adam* opt, const void* obs, const int32_t* order, const float* action_mat,
                         const float* adv, const float* target_v, int n, int fit_batch, int logit_tensor, int v_tensor,
                         float ent_coef, float* loss_out, int use_graph, void* stream);
/* IMPALA.train: n_traj trajectories of ep_len steps, stored trajectory by trajectory. */
typedef struct xtb_impala_traj {
  const void* obs;            /* [n_traj*(ep_len+1), ...] states, the last of each trajectory its bootstrap state */
  const float* behav_prob;    /* [n_traj*ep_len, A] behaviour policy probabilities */
  const float* action_mat;    /* [n_traj*ep_len, A] one-hot actions */
  const float* reward;        /* [n_traj*ep_len] */
  const uint8_t* done;        /* [n_traj*ep_len] */
} xtb_impala_traj;
/* 1. forward of every state with the current weights; 2. the V-trace variant of impala.py:124-184 into pg_adv and
 * target_v ([n_traj*ep_len] device scratch the caller may read); 3. for every `slice`-row slice of the training rows,
 * in order, one fit epoch as xtb_impala_keras_fit with adv = pg_adv.  order: [n_traj*ep_len] training rows, slice by
 * slice (each slice a permutation of its own rows); training row i reads state row i + i / ep_len (obs_idx: scratch of
 * the same size).  loss_per_slice[k] = the epoch loss of slice k.  n_traj*(ep_len+1) must not exceed max_batch. */
int xtb_impala_keras_train(xtb_net* net, xtb_adam* opt, const xtb_impala_traj* tr, int n_traj, int ep_len, int slice,
                           int fit_batch, const int32_t* order, int32_t* obs_idx, float gamma, float ent_coef,
                           int logit_tensor, int v_tensor, float* pg_adv, float* target_v, float* loss_per_slice,
                           int use_graph, void* stream);

/* Rollout inference: for t in [0,n_step): forward over n_env observations (row e of step t is
 * obs[step_idx[t*n_env+e]], NULL = rows t*n_env..), draw actions as xtb_categorical_sample / xtb_diag_gaussian_sample do
 * with Philox4x32-10(seed, offset = *offset_dev + t), and write action [n_step, n_env] int32 or [n_step, n_env, A] float
 * and logp / value [n_step, n_env] time-major; finally *offset_dev += n_step.  This is the batched replacement of the
 * per-explorer batch-1 PPO.predict calls (xt/agent/ppo/ppo.py:35-45, xt/algorithm/ppo/ppo.py:87-95). */
int xtb_ppo_rollout_infer(xtb_net* net, const void* obs, const int32_t* step_idx, int n_env, int n_step, int pi_tensor,
                          int v_tensor, int logstd_tensor, uint64_t seed, unsigned long long* offset_dev, void* action,
                          float* logp, float* value, int use_graph, void* stream);

/* PPO.predict (xt/model/ppo/ppo.py:104-109) on host buffers in one call: staged H2D of `obs_host` (pageable,
 * obs_bytes) into `obs_dev`, xtb_ppo_rollout_infer with n_step = 1 writing the packed block
 *   out_dev = [action | logp f32 x n_env | value f32 x n_env], action int32 x n_env or (DiagGaussian) f32 x n_env*A,
 * one D2H of it into `out_host` (pinned), one D2H of the [n_env, A] output of `pi_tensor` into `head_host` (pinned;
 * NULL = skip: for actors whose predict() also returns the logits, ImpalaCnnOpt.predict,
 * xt/model/impala/impala_cnn_opt.py:267-277) and a stream synchronise: when it returns, both hold the step's results. */
int xtb_ppo_predict_host(xtb_net* net, const void* obs_host, size_t obs_bytes, void* obs_dev, int n_env, int pi_tensor,
                         int v_tensor, int logstd_tensor, uint64_t seed, unsigned long long* offset_dev, float* out_dev,
                         float* out_host, float* head_host, int use_graph, void* stream);

/* ---- PPO with a diagonal Gaussian policy (action_type DiagGaussian): replaces DiagGaussianDist
 *      (xt/model/tf_dist.py:49-86) as PPO.build_graph wires it (xt/model/ppo/ppo.py:62-95) --------------
 * mean = the linear pi_latent head [B, A], log_std = the A floats of an XTB_LOGSTD layer, std = exp(log_std).
 *   neglog_prob(x) = 0.5 log(2 pi) A + 0.5 sum_i ((x_i - mean_i) / std_i)^2 + sum_i log_std_i,  logp = -neglog_prob
 *   entropy        = sum_i (log_std_i + 0.5 (log(2 pi) + 1))   (state independent)
 * Actions are unbounded floats: no clipping or squashing, as in the reference. */
/* DiagGaussianDist.sample + log_prob (tf_dist.py:85-86, ppo.py:82-83): action = mean + std * n, logp computed from
 * the action.  n from `normals` [batch, adim] if non-NULL, else standard normals drawn with Philox4x32-10(seed, offset)
 * and Box-Muller: sample b, dimension group g = i / 4 uses counter (b, g, offset_lo, offset_hi) and key (seed_lo,
 * seed_hi); its four words give uniforms u0..u3 = (x >> 8) 2^-24 + 2^-25 (never 0 or 1, as xtb_categorical_sample) and
 *   n_{4g}   = sqrt(-2 log u0) cos(2 pi u1),  n_{4g+1} = sqrt(-2 log u0) sin(2 pi u1),
 *   n_{4g+2} = sqrt(-2 log u2) cos(2 pi u3),  n_{4g+3} = sqrt(-2 log u2) sin(2 pi u3).
 * action [batch, adim] f32, logp [batch] f32.  adim <= 32. */
int xtb_diag_gaussian_sample(const float* mean, const float* log_std, int batch, int adim, const float* normals,
                             uint64_t seed, uint64_t offset, float* action, float* logp, void* stream);
/* actor_loss_with_entropy + critic_loss (xt/model/ppo/__init__.py:4-25, ppo.py:87-92) on the Gaussian head: as
 * xtb_ppo_loss_grad with logp = log_prob(action) of the float behaviour action [N, A] (indexed through gather_idx) and
 * the entropy above.  Writes dmean [B, A], dv [B] and dlog_std [A] (overwritten: the gradient of this minibatch's loss
 * summed over its samples in a fixed order), adds the loss to *loss_out.  One block: the step is reproducible. */
int xtb_ppo_gauss_loss_grad(const float* mean, const float* v, const float* log_std, const int32_t* gather_idx,
                            const float* action, const float* old_logp, const float* adv, const float* old_v,
                            const float* target_v, int batch, int adim, const xtb_ppo_hyper* hp, float inv_count,
                            float* dmean, float* dv, float* dlog_std, float* loss_out, void* stream);

/* ---- MuZero: replaces MuzeroModel's train / inference graphs (xt/model/muzero/muzero_model.py:74-239) ----------------
 * The model is three nets: representation (obs -> hidden h, H wide), dynamics (concat(h, one_hot(a)) -> next hidden and
 * reward logits) and prediction (h -> policy logits, value logits).  Their softmax outputs are evaluated by the kernels,
 * so the policy, value and reward heads are linear dense layers.  The three nets are bound to slices [rep | dyn | pred],
 * in this order, of one parameter buffer (MuzeroBase's Keras weight-list order; gaps between the slices are allowed, e.g.
 * to keep each slice 16-byte aligned as xtb_net_bind requires of a net with tensor-core layers), and to the slices at
 * the same offsets of one gradient buffer; the optimiser spans the buffer from the first slice to the last.  The
 * dynamics net is bound to its parameter slice and to a gradient buffer of its own OUTSIDE the shared one, which every
 * application of it fills before it is added to its slice in a fixed order.  The dynamics and prediction nets read float
 * observations (decode scale 1) with dense layers only.
 *   h(x) = sign(x)(sqrt(|x| + 1) - 1) + 0.001 x   (value_compression, muzero_utils.py:38-40)
 *   two-hot target of a scalar x (conver_value, muzero_model.py:200-216): v = h(clip(x, min, max) - min) in float64,
 *     1 - frac(v) at floor(v), frac(v) at floor(v) + 1
 *   scalar of a support (value_transform, :218-226): clip(h^-1(sum_j softmax_j j) + min, min, max), h^-1 in closed form
 * Supports and the action count are at most 1024 wide. */
typedef struct xtb_muzero xtb_muzero;
typedef struct xtb_muzero_desc {
  int32_t unroll;                 /* K (td_step) */
  int32_t rep_h;                  /* representation net: hidden-state tensor (relu / tanh / linear), H wide */
  int32_t dyn_h, dyn_r;           /* dynamics net: next hidden state (H wide, relu / tanh / linear) and reward logits */
  int32_t pred_p, pred_v;         /* prediction net: policy logits (A wide) and value logits */
  float value_min, value_max;     /* value support range */
  float reward_min, reward_max;   /* reward support range */
} xtb_muzero_desc;
/* Checks the nets and their binding and allocates the step's device scratch for up to max_batch samples (the prediction
 * net must hold (unroll + 1) * max_batch rows).  The nets must outlive the object and stay bound as they were. */
int xtb_muzero_create(xtb_net* rep, xtb_net* dyn, xtb_net* pred, const xtb_muzero_desc* desc, int max_batch, xtb_muzero** out);
void xtb_muzero_destroy(xtb_muzero* mz);
/* One training batch of B samples (device arrays). */
typedef struct xtb_muzero_batch {
  const void* obs;              /* [B, ...] observations of the representation net */
  const int32_t* action;        /* [B, unroll] */
  const float* target_value;    /* [B, unroll + 1] scalars */
  const float* target_reward;   /* [B, unroll + 1] scalars (column `unroll` is not used) */
  const float* target_policy;   /* [B, unroll + 1, A] */
  int32_t unroll;               /* must equal the model's */
} xtb_muzero_batch;
/* MuzeroModel.train (muzero_model.py:103-140, 154-169) as one step: h_0 = rep(obs); for k < K h_{k+1}, r_k =
 * dyn(concat(h_k, one_hot(a_k))); policy/value of h_0..h_K as one prediction pass over (K+1) B rows;
 *   loss = CE(p_0, pi_0) + CE(v_0, z_0) + sum_{k<K} [CE(r_k, u_k) + CE(p_{k+1}, pi_{k+1}) + CE(v_{k+1}, z_{k+1})]
 *   CE(p, t) = mean_b mean_j -t_j log(p_j + 1e-10)   (p = softmax of the logits)
 * the gradient of every term under the sum scaled by 1/K, the gradient reaching h_{k+1} (k+1 < K) from dynamics step k+1
 * scaled by 0.5 (h_0 unscaled); backward (dynamics recomputed step by step); one Adam step of `opt` (created over the
 * whole buffer, no clipping) and the weight refresh of the three nets.  *loss_out = loss_offset + loss, its terms summed
 * in a fixed order.  value_out != NULL: [B] the value of every observation after the update (value_inference).
 * XTB_ERR_STATE, launching nothing, while a communicator is installed. */
int xtb_muzero_train(xtb_muzero* mz, xtb_adam* opt, const xtb_muzero_batch* batch_in, int batch, float loss_offset,
                     float* loss_out, float* value_out, int use_graph, void* stream);
/* initial_inference / value_inference (muzero_model.py:74-82, 228-239) over `batch` observations: hidden [B, H],
 * value [B] scalars, policy [B, A] probabilities; any output may be NULL. */
int xtb_muzero_initial_inference(xtb_muzero* mz, const void* obs, int batch, float* hidden_out, float* value_out,
                                 float* policy_out, int use_graph, void* stream);
/* recurrent_inference (muzero_model.py:84-96) over `batch` hidden states [B, H] and actions [B]: next hidden [B, H],
 * reward [B] and value [B] scalars, policy [B, A] probabilities; any output may be NULL. */
int xtb_muzero_recurrent_inference(xtb_muzero* mz, const float* hidden, const int32_t* action, int batch, float* hidden_out,
                                   float* reward_out, float* value_out, float* policy_out, int use_graph, void* stream);
/* Device scratch of the tree search for up to max_envs trees of up to max_simulations simulations each, for the action
 * count and hidden width of `mz` (which it does not keep). */
typedef struct xtb_muzero_tree xtb_muzero_tree;
int xtb_muzero_tree_create(const xtb_muzero* mz, int max_envs, int max_simulations, xtb_muzero_tree** out);
void xtb_muzero_tree_destroy(xtb_muzero_tree* tree);
/* Mcts.run_mcts (xt/agent/muzero/mcts.py, util.py) over n_envs observations at once, one tree per observation, advanced
 * in lock step: xtb_muzero_initial_inference of the observations gives the roots; the root priors become
 * prior * (1 - exploration_frac) + noise * exploration_frac when noise [n_envs, A] (float64) is given; then each of
 * num_simulations simulations descends every tree by
 *   ucb = (log((N_p + pb_c_base + 1) / pb_c_base) + pb_c_init) * sqrt(N_p) / (N_c + 1) * prior
 *         + (N_c > 0 ? normalize(value_sum / N_c) : 0)
 * (ties to the higher action) to an unexpanded child, evaluates all leaves with one xtb_muzero_recurrent_inference
 * launch sequence, expands them and backs the leaf value up the path (v = reward + discount * v), with one MinMaxStats
 * per tree (normalize(x) = (x - min) / (max - min) once max > min, else x).  Tree statistics are float64, products
 * rounded before they are added.  Writes the root child visit counts visit_counts_out [n_envs, A] and the root values
 * root_value_out [n_envs] (float64).  n_envs in [1, min(tree max_envs, model max_batch)], num_simulations in
 * [1, tree max_simulations], pb_c_base finite and positive; XTB_ERR_STATE while a communicator is installed. */
int xtb_muzero_search(xtb_muzero* mz, xtb_muzero_tree* tree, const void* obs, int n_envs, int num_simulations,
                      const double* noise, double pb_c_base, double pb_c_init, double discount, double exploration_frac,
                      int32_t* visit_counts_out, double* root_value_out, int use_graph, void* stream);
/* xtb_net_backward that also writes d loss / d observation [batch, obs width] into dobs (overwritten): the data-gradient
 * GEMM of every dense layer that reads the observation, summed in layer order.  Float observations with scale 1 read
 * by dense layers only; otherwise XTB_ERR_ARG. */
int xtb_net_backward_input(xtb_net* net, const void* obs, const int32_t* gather_idx, int batch,
                           const int32_t* head_tensors, int n_heads, float* dobs, void* stream);

/* Data-parallel communicator owned by the library (SURVEY 8(e); precedent zeus/trainer/trainer_tf.py:187-203): NCCL is
 * resolved with dlopen (`nccl_path` NULL = "libnccl.so.2").  Rank 0 calls xtb_comm_unique_id and ships the 128 bytes to
 * the other ranks (engine.py uses torch.distributed); every rank then calls xtb_comm_create.  With a communicator
 * installed (xtb_set_grad_comm) the fused training loops all-reduce the flat gradient bucket themselves -- the large
 * dense weight gradient as soon as it is final, on a side stream under the rest of the backward pass -- and stay inside
 * the CUDA graph. */
typedef struct xtb_comm xtb_comm;
int xtb_comm_unique_id(const char* nccl_path, void* id128);
int xtb_comm_create(const char* nccl_path, const void* id128, int rank, int world, xtb_comm** out);
void xtb_comm_destroy(xtb_comm* comm);
int xtb_comm_world(const xtb_comm* comm);
int xtb_set_grad_comm(xtb_comm* comm);
int xtb_comm_allreduce(xtb_comm* comm, float* buf, long long count, void* stream);

/* Launch one kernel of one layer alone (which: 0 forward, 1 weight gradient) on the tensors
 * currently in the workspace -- measurement hook for bench.py's roofline object. */
int xtb_net_bench_layer(xtb_net* net, int layer, int which, const void* obs, const int32_t* gather_idx,
                        int batch, void* stream);

/* Kernel-path selection: 1 (default) = wgmma tensor-core kernels wherever the shape is covered,
 * 0 = fp32 CUDA-core kernels only (also XTB_TC=0 in the environment).  For A/B parity tests. */
int xtb_set_tc_mode(int mode);
/* 1 (default): xtb_ppo_train (and xtb_dqn_train on a dueling head) evaluates both heads, the loss and their backward
 * in one fused kernel; 0: layer-by-layer (also XTB_FUSE_HEADS=0).  Takes effect at the next call.  The same mode
 * selects the fused heads of the rollout-inference calls. */
int xtb_set_fuse_heads(int on);
int xtb_get_tc_mode(void);
/* Self-test of the wgmma GEMM core on plain fp32 matrices (sizes multiples of 8):
 * mode 0: C = A[M,K] B[K,N]; mode 1: C = A[M,K] Bt[N,K]^T; mode 2: C = At[K,M]^T B[K,N]. */
int xtb_tc_gemm_test(int mode, const float* a, const float* b, float* c, int M, int N, int K, int ksplit,
                     void* stream);

/* ---- host <-> device staging (SURVEY 8(f1): pinned ring replacing feed_dict copies) --- */
void* xtb_pinned_alloc(size_t bytes);
void xtb_pinned_free(void* p);
int xtb_copy_h2d(void* dst_dev, const void* src_host, size_t bytes, void* stream);
/* Pageable host memory -> device: worker threads memcpy 256 KiB chunks into a pinned ring while the caller
 * enqueues one async copy per staged chunk on `stream`.  On return `src_host` has been consumed (it may be
 * reused); the device side is ordered on `stream`.  Replaces the single-threaded feed_dict staging of
 * sess.run (xt/model/ppo/ppo.py:104-132).  XTB_STAGE_THREADS (default 4) sizes the pool. */
int xtb_copy_h2d_staged(void* dst_dev, const void* src_host, size_t bytes, void* stream);
int xtb_copy_d2h(void* dst_host, const void* src_dev, size_t bytes, void* stream);
int xtb_stream_sync(void* stream);

#ifdef __cplusplus
}
#endif
#endif /* XTB200_H_ */
