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
/* Number of CUDA graphs the library has captured (a replay of a cached graph does not count). */
long long xtb_graph_capture_count(void);

/* ---- network: replaces XTModel's TF graph (xt/model/model.py:30-127) ---------- */
/* Flat fp32 parameter layout: per layer, kernel [K,N] (HWIO flattened) then bias [N];
 * identical to iterating TFVariables' ordered dict (xt/model/tf_utils.py:84-102). */
/* xtb_net_create plans on the host and makes no CUDA call: it needs no device. */
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
/* argmax over the last axis (DQN greedy action, xt/algorithm/algorithm.py:124-135): as np.argmax, the first maximum
 * wins and the first NaN wins over any number */
int xtb_argmax(const float* q, int batch, int adim, int32_t* action, void* stream);

/* ---- GAE: replaces PPO.data_proc (xt/agent/ppo/ppo.py:77-106) ------------------- */
/* value [E,T+1], reward [E,T], done [E,T] (uint8) -> adv, old_value, target_value [E,T].
 * sign_clip != 0 applies np.sign to rewards (xt/agent/ppo/atari_ppo.py:46), which keeps a NaN reward NaN.
 * E = 0 or T = 0 is a no-op; a negative size is refused. */
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
 * return, 0 = the window hit a terminal step); huber_delta > 0 selects the Huber loss instead of the squared error.
 * wt != NULL scales sample b's loss and gradient by wt[b] (Keras sample_weight); td_abs != NULL receives |y_b - q[b, a_b]|.
 * dq is written in full: zero on every action not taken. */
int xtb_dqn_td_loss_grad(const float* q, const float* q_next_target, const float* q_next_online, const int32_t* idx,
                         const int32_t* action, const float* reward, const uint8_t* done, const float* disc, int batch,
                         int adim, float gamma, float huber_delta, float inv_count, const float* wt, float* dq,
                         float* y_out, float* td_abs, float* loss_out, void* stream);
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
/* Switch the optimiser handle to tf.train.RMSPropOptimizer(lr, decay, epsilon) with its defaults centered=False and
 * momentum 0: ms = decay ms + (1 - decay) g^2, theta -= lr g / sqrt(ms + epsilon).  The `m` buffer of xtb_adam_create
 * becomes the `rms` slot, set to ones here as TF initialises it; `v` is unused.  Clipping, chunking and the weight-blob
 * refresh are those of the Adam step. */
int xtb_opt_use_rmsprop_plain(xtb_adam* opt, float decay, float epsilon);

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
/* The fused-heads instantiation the PPO calls would launch for these heads under the current fused-heads mode: the
 * training kernel (infer == 0) or the rollout-inference kernel (infer != 0), as (*kpl, *amax): it covers K <= 32 * kpl
 * hidden units and A <= amax actions; (0, 0) when the heads run layer by layer.  Head tensors the PPO calls reject
 * return XTB_ERR_ARG, as there.  Launches nothing. */
int xtb_ppo_heads_plan(const xtb_net* net, int pi_tensor, int v_tensor, int infer, int* kpl, int* amax);
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
/* xtb_dqn_train with importance weights: sample b's loss and gradient are scaled by weights[b] (Keras train_on_batch with
 * sample_weight: loss = 1/(B A) sum_b weights[b] sum_a e_ba), and td_abs[b] = |y_b - Q(s_b, a_b)| from the online forward
 * before the update.  Either may be NULL; with both NULL the step is xtb_dqn_train's. */
int xtb_dqn_train_weighted(xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                           const int32_t* idx, const int32_t* action, const float* reward, const uint8_t* done,
                           const float* disc, int n_sample, float gamma, float huber_delta, int q_tensor, float* qn_t,
                           float* qn_o, const float* weights, float* td_abs, float* loss_out, int use_graph, void* stream);
/* The heads_kernel entry the DQN steps launch for q_tensor under the current fused-heads mode: (kpl, amax) covering K <=
 * 32 kpl hidden units and A <= amax actions; (0, 0) when the step runs layer by layer (q_tensor is not a fusable dueling
 * layer).  A q_tensor out of range returns XTB_ERR_ARG.  Launches nothing. */
int xtb_dqn_heads_plan(const xtb_net* net, int q_tensor, int* kpl, int* amax);

/* ---- prioritized experience replay (Schaul et al., proportional variant) over the slots of a device replay ring: the
 *      rules of PrioritizedReplayBuffer (xt/algorithm/prioritized_replay_buffer_muzero.py:77-200), leaf i = ring slot i ----
 * Insert: every slot written (wrapped slots included) gets max_priority ** alpha; max_priority starts at 1, is the
 *   largest raw priority an update wrote and is never lowered.
 * Sample B indices with replacement, stratified: mass_k = (u_k + k) total / B, u_k uniform in [0, 1); the draw descends
 *   to the first leaf whose running sum exceeds mass_k, and one past the stored slots is clamped to count - 1.  total
 *   is the sum over ALL stored leaves (the reference's sum(0, len - 1) has an exclusive end and never draws slot len - 1;
 *   the reference DQN has no prioritized replay, so nothing binds to that).
 * Importance weights, in float64, stored as float32: p_min = max(min_leaf / total, 1e-5),
 *   w_k = ((leaf[idx_k] / total) count) ** -beta / (p_min count) ** -beta.
 * Update: the reference's sequential loop over k: leaf[idx_k] = (|delta_k| + eps) ** alpha (an index named twice takes
 *   the later k) and max_priority = max(max_priority, |delta_k| + eps).  An entry whose priority is not finite is skipped
 *   and sets XTB_PER_NONFINITE.
 * The sum and min trees are float64 over capacity rounded up to a power of two (empty leaves: 0 and +inf); every
 * internal node is op(left, right) of its final children, so the trees are bitwise a function of their leaves.  The
 * trees, count, max_priority, the status bits and the Philox offset live in one device allocation of the object and
 * are read by the kernels, so one captured xtb_dqn_per_train graph serves every step while the ring fills.
 * xtb_per_add / _sample / _update / xtb_dqn_per_train return XTB_ERR_STATE while a communicator is installed. */
typedef struct xtb_per xtb_per;
#define XTB_PER_NONFINITE 1   /* status: an update met a priority that is not finite (and did not write it) */
#define XTB_PER_BAD_INDEX 2   /* status: an update named a slot outside [0, count) */
#define XTB_PER_EMPTY 4       /* status: a draw from a tree with no stored slot (it wrote idx 0, w 0) */
/* capacity >= 1 (the ring's), alpha >= 0, eps > 0 (finite), seed: the Philox key of the device draws. */
int xtb_per_create(int capacity, double alpha, double eps, uint64_t seed, xtb_per** out);
void xtb_per_destroy(xtb_per* per);
/* Insert: ring slots [first_slot, first_slot + n) were written (a wrapped write is two calls); count covers them. */
int xtb_per_add(xtb_per* per, int first_slot, int n, void* stream);
/* B = batch draws into idx [B] int32 and w [B] float32, beta > 0.  uniforms [B] float64 in [0, 1) when non-NULL;
 * otherwise u_k = 53 bits of Philox4x32-10 on counter (k, 0, offset) and the object's seed, ((x0 >> 5) 2^26 + (x1 >> 6))
 * 2^-53, and the device offset advances by one. */
int xtb_per_sample(xtb_per* per, int batch, double beta, const double* uniforms, int32_t* idx, float* w, void* stream);
/* Update leaves idx[0..n) from td_abs[0..n) (|TD error|, float32). */
int xtb_per_update(xtb_per* per, const int32_t* idx, const float* td_abs, int n, void* stream);
/* Read-only snapshot after a device synchronise; any output may be NULL.  sum_host / min_host: [2 leaves] float64 in
 * heap order (node 1 the root, node i's children 2i and 2i + 1, leaf j at node leaves + j). */
int xtb_per_state(const xtb_per* per, int* leaves, int* count, double* max_priority, int* status, unsigned long long* offset,
                  double* sum_host, double* min_host);
/* One prioritized DQN step as one captured graph: xtb_per_sample of n_sample rows (Philox) into idx / w,
 * xtb_dqn_train_weighted on them (weights w, |TD error| into td_abs), xtb_per_update(idx, td_abs), and a copy of the
 * status bits into *status_out (device int32).  beta > 0. */
int xtb_dqn_per_train(xtb_per* per, xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                      const int32_t* action, const float* reward, const uint8_t* done, const float* disc, int n_sample,
                      float gamma, float huber_delta, double beta, int q_tensor, float* qn_t, float* qn_o, int32_t* idx,
                      float* w, float* td_abs, float* loss_out, int32_t* status_out, int use_graph, void* stream);

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

/* ---- MuZero trajectory replay on the device: the Muzero learner's buffer (xt/algorithm/muzero/muzero.py over
 *      prioritized_replay_buffer_muzero.py) with its rules and float64 arithmetic, kept in HBM ----------------------------
 * Storage: a pool of pool_steps steps (observation rows of obs_bytes as the representation net reads them, actions
 *   int32, target values float64, rewards float32, child visits [A] float32) and `capacity` trajectory slots.  Slot s
 *   holds the trajectory at pool [off, off + len); the caller places trajectories (xtb_muzero_replay_add), evicting the
 *   oldest when a new one does not fit.  An evicted slot keeps its place in count, its leaf is 0 and stays 0.
 * Trees, float64, every internal node left + right of its final children:
 *   trajectory tree: leaf s = the weight of slot s's position tree (its root / (len - K)), capacity rounded up to a
 *     power of two; position tree of a slot: leaf i < len - K = |value_i - target_value_i|, capacity = len rounded up.
 * Draw of B samples from uniforms u [2B] (float64, the host's random.random() calls in its order):
 *   trajectory k: mass = u[k] step + k step, step = reduce(0, count - 1) / B, where reduce(0, n - 1) sums leaves
 *     0 .. n - 2 in the order of the host segment tree's midpoint recursion (its exclusive end); the descent takes the
 *     first leaf whose running sum exceeds the mass, with the host's subtractions.  A descent that ends on a slot
 *     without a live trajectory (evicted, or past count through rounding) takes the nearest live slot below it,
 *     wrapping from slot 0 to count - 1, and sets XTB_MZR_REMAPPED;
 *   its position: mass = u[B + k] total + 0 total in that slot's tree, total = reduce(0, len - K - 1), clamped to
 *     len - K - 1.
 * Update from post-step values v [B]: new_pri_k = max(|v_k - target_value[pos_k]|, 1e-5) (NaN stays NaN); in batch
 *   order k, position leaf pos_k of slot_k takes new_pri_k, then trajectory leaf k (the batch position, the reference's
 *   rule) takes slot_k's weight at that moment unless slot k holds no live trajectory.  The sequence stops before the
 *   first entry whose priority is not > 0 (XTB_MZR_BAD_PRIORITY) or that names no live slot, a position outside it or
 *   a batch position k >= count (XTB_MZR_BAD_INDEX).
 * The masses are formed as the host forms them: both products rounded, then the sum (no fused multiply-add).
 * Every value that changes from call to call (count, the slot table, both tree levels, the status) is on the device,
 * so one captured xtb_muzero_replay_train graph serves the run while the ring fills and wraps.
 * xtb_muzero_replay_add / _sample / _update / _train return XTB_ERR_STATE, launching nothing, while a communicator is
 * installed (create and the read-only state snapshot do not train and are allowed). */
typedef struct xtb_muzero_replay xtb_muzero_replay;
typedef struct xtb_muzero_replay_slot {
  int64_t off;      /* first pool step */
  int32_t len;      /* steps */
  int32_t live;     /* 1: holds its trajectory; 0: empty or evicted */
} xtb_muzero_replay_slot;
/* The minibatch a draw gathers (device arrays of B rows), laid out as xtb_muzero_batch reads it. */
typedef struct xtb_muzero_replay_batch {
  void* obs;                /* [B, obs_bytes] */
  int32_t* action;          /* [B, unroll] */
  float* target_value;      /* [B, unroll + 1] */
  float* target_reward;     /* [B, unroll + 1] */
  float* target_policy;     /* [B, unroll + 1, A] */
} xtb_muzero_replay_batch;
#define XTB_MZR_BAD_PRIORITY 1   /* status: an update met a priority that is not > 0; it and the entries after it were not applied */
#define XTB_MZR_REMAPPED 2       /* status: a draw's descent ended on a slot without a live trajectory */
#define XTB_MZR_BAD_INDEX 4      /* status: an update named no live slot, a position outside it or a batch position past
                                    count; not applied from there */
/* capacity (BUFFER_SIZE) >= 1, pool_steps >= 1, unroll K >= 1, obs_bytes >= 1, n_actions A in [1, 1024], max_batch >= 1:
 * the largest B of a draw. */
int xtb_muzero_replay_create(int capacity, long long pool_steps, int unroll, long long obs_bytes, int n_actions, int max_batch,
                             xtb_muzero_replay** out);
void xtb_muzero_replay_destroy(xtb_muzero_replay* r);
/* Store one trajectory of len steps (K + 1 < len <= pool_steps) from device arrays obs [len, obs_bytes], action [len],
 * target_value [len] (float64), reward [len], child_visits [len, A] at slot `slot` and pool [off, off + len), after
 * evicting slots [evict_first, evict_first + n_evict) mod capacity (which must not include `slot`).  values [len]
 * (float64) gives the values of the position priorities; NULL: xtb_muzero_initial_inference of mz on the stored pool
 * rows, max_batch rows per forward as the host's value_inference. */
int xtb_muzero_replay_add(xtb_muzero_replay* r, xtb_muzero* mz, int slot, long long off, int evict_first, int n_evict,
                          const void* obs, const int32_t* action, const double* target_value, const float* reward,
                          const float* child_visits, int len, const double* values, void* stream);
/* The draw of B in [1, max_batch] samples from uniforms [2B] into slot_out [B] / pos_out [B] (int32) and the gathered
 * batch.  Resets the status to this draw's bits.  XTB_ERR_STATE when nothing is stored. */
int xtb_muzero_replay_sample(xtb_muzero_replay* r, int batch, const double* uniforms, int32_t* slot_out, int32_t* pos_out,
                             const xtb_muzero_replay_batch* out, void* stream);
/* The update of B entries (slot [B], pos [B] from a draw) from values [B] float64.  B in [1, min(max_batch, count)]:
 * batch position B - 1 must be a stored slot, as the host's update requires (XTB_ERR_ARG otherwise). */
int xtb_muzero_replay_update(xtb_muzero_replay* r, int batch, const int32_t* slot, const int32_t* pos, const double* values,
                             void* stream);
/* One learner step: xtb_muzero_replay_sample, xtb_muzero_train of mz / opt on the gathered batch (loss_offset,
 * *loss_out) with the post-update values, xtb_muzero_replay_update from them, and a copy of the status into
 * *status_out (device int32).  B in [1, min(max_batch, count)], as for the update. */
int xtb_muzero_replay_train(xtb_muzero_replay* r, xtb_muzero* mz, xtb_adam* opt, int batch, const double* uniforms,
                            int32_t* slot_out, int32_t* pos_out, const xtb_muzero_replay_batch* out, float loss_offset,
                            float* loss_out, int32_t* status_out, int use_graph, void* stream);
/* Read-only snapshot after a device synchronise; any output may be NULL.  slots [capacity]; traj_tree [2 tree_leaves]
 * heap order; forest [4 pool_steps]: slot s's position tree is the 2 cap doubles at forest + 4 off. */
int xtb_muzero_replay_state(const xtb_muzero_replay* r, int* count, int* status, int* tree_leaves,
                            xtb_muzero_replay_slot* slots, double* traj_tree, double* forest);

/* ---- QMIX: replaces QMixModel's train and explore graphs (xt/model/qmix/qmix_tf.py:172-589) -------------------------
 * One weight set is a flat float buffer [fc1 | GRU | fc2 | mixer]: fc1 = dense(H, relu) on the agent inputs (net `fc1`,
 * obs_dim wide), the GRUCell's rnn/gru_cell/gates/kernel [2H, 2H], gates/bias [2H], candidate/kernel [2H, H] and
 * candidate/bias [H] back to back at float offset gru_off (kernel rows: x first, then h), fc2 = dense(A) on the GRU
 * outputs (net `fc2`, H wide, float input) and the mixer's hypernetworks, one net `hyper` on the state whose 7 dense layers
 * are, in order, hyper_w1 (hypernet_embed relu, then E n_agents linear), hyper_b1 (E linear, on the state),
 * hyper_w_final (hypernet_embed relu, then E linear) and val_for_bias (E relu, then 1 linear) -- the TF variable order
 * of the eval_agent and eval_mixer scopes.  The three nets are bound to their slices of the eval set (gaps between the
 * slices are allowed) and of a gradient buffer with the same layout; the optimiser spans the set (per-tensor clipping:
 * one segment per variable).  Target and explore sets are caller buffers with the same layout (an explore set needs
 * only the agent part).
 * Limits (XTB_ERR_ARG otherwise, at create): 1 <= H with the GRU kernels' shared-memory plan fitting (H <= 137),
 * n_agents <= 32, n_actions <= 255 (the reference casts actions to uint8), mixing embed E <= 128. */
typedef struct xtb_qmix xtb_qmix;
typedef struct xtb_qmix_desc {
  int32_t batch;          /* B episodes per training batch */
  int32_t episode_limit;  /* L: a batch holds L + 1 steps of agent inputs and L transitions */
  int32_t n_agents;
  int32_t use_double_q;
  float gamma;
  long long gru_off;      /* offset (floats) of gates/kernel in a weight set */
  int32_t act_envs;       /* most environments one xtb_qmix_act call steps (0: one); fc1 and fc2 must hold act_envs
                             n_agents rows */
} xtb_qmix_desc;
int xtb_qmix_create(xtb_net* fc1, xtb_net* fc2, xtb_net* hyper, const xtb_qmix_desc* desc, xtb_qmix** out);
void xtb_qmix_destroy(xtb_qmix* q);
/* One training batch (device arrays). */
typedef struct xtb_qmix_batch {
  const float* obs;         /* [B, L+1, n_agents, obs_dim] agent inputs */
  const int32_t* seq_len;   /* [B n_agents] GRU sequence lengths (train_obs_len, sequence b n_agents + a), read at run time,
                               clamped to [0, L+1] */
  const float* avail;       /* [B, L+1, n_agents, A] available actions (0 = unavailable) */
  const int32_t* actions;   /* [B, L, n_agents] taken actions in [0, A) */
  const float* state;       /* [B, L, state_dim] eval mixer input (batch["state"][:, :-1]) */
  const float* next_state;  /* [B, L, state_dim] target mixer input (batch["state"][:, 1:]) */
  const float* reward;      /* [B, L] */
  const float* terminated;  /* [B, L] */
  const float* mask;        /* [B, L] */
} xtb_qmix_batch;
/* QMixModel.train (qmix_tf.py:351-492, 546-589) as one step: the target and eval agents over all B (L+1) n_agents rows
 * (fc1 and fc2 on the engine, the GRU recurrence of dynamic_rnn as one persistent kernel: outputs at t >= seq_len are
 * zero), both hypernetworks over the B L state rows, the fused mixer / TD kernel (see qmix.cuh), the backward (the GRU's
 * in reverse time, its weight gradients as GEMMs over all rows) and one step of `opt`, which must be set to centred
 * RMSProp by the caller (xtb_opt_use_rmsprop, decay 0.95, epsilon 1.5e-7, per-tensor clip at grad_norm_clip), then the
 * weight refresh of the three nets.  *loss_out = sum (mask td)^2 / sum mask, summed in a fixed order.  target: the
 * target weight set.  XTB_ERR_STATE while a communicator is installed. */
int xtb_qmix_train(xtb_qmix* q, xtb_adam* opt, const float* target, const xtb_qmix_batch* batch, float* loss_out, int use_graph,
                   void* stream);
/* QMixModel.infer_actions (qmix_tf.py:242-251) for one environment: fc1 -> one GRU step -> fc2 with the weight set
 * `explore` on obs [n_agents, obs_dim]; hidden [n_agents, H] is read as the state and overwritten with the new one;
 * q_out [n_agents, A]. */
int xtb_qmix_infer(xtb_qmix* q, const float* explore, const float* obs, float* hidden, float* q_out, int use_graph, void* stream);
/* QMixAlg.predict_with_selector for n_envs environments at once (1 <= n_envs <= act_envs), as one launch sequence:
 *   - the agent inputs of build_inputs for one step: obs [n_envs, n_agents, o] (o = fc1's width less n_actions with
 *     obs_last_action, less n_agents with obs_agent_id), then the one-hot of last_action [n_envs, n_agents] (zeros for
 *     a value < 0), then the one-hot of the agent;
 *   - an environment whose reset [n_envs] flag is non-zero starts from zero hidden rows and no last action (its
 *     last_action rows become -1 before the inputs are read);
 *   - fc1 -> one GRU step -> fc2 of the weight set `explore` on the n_envs n_agents rows, hidden [n_envs, n_agents, H]
 *     read and overwritten; the Q values stay in fc2's output tensor (rows e n_agents + a);
 *   - EpsilonGreedyActionSelector.select_action per row: avail [n_envs, n_agents, A] int32 action weights (< 1e-6:
 *     unavailable), epsilon [n_envs] float64; the action is np.random.choice(A, p=avail/sum) for u1 if u0 < epsilon,
 *     else the first argmax of the masked Q (agent_act.cuh states the rule).  (u0, u1) = uniforms[e, 0, a] and
 *     uniforms[e, 1, a] (float64 [n_envs, 2, n_agents]); with uniforms NULL they are 53-bit uniforms of Philox4x32-10
 *     keyed by seed on counter (a, e, counter[e]), counter [n_envs] uint64 in device memory advancing by one per call.
 * actions [n_envs, n_agents] int32 and last_action get the chosen actions.  Every array is a device array.  A row
 * without a positive weight gets an action that means nothing.  XTB_ERR_ARG before any launch for a null pointer (counter
 * only when uniforms is NULL), n_envs outside [1, act_envs] or no room for the observation in fc1's inputs. */
int xtb_qmix_act(xtb_qmix* q, const float* explore, int n_envs, int obs_last_action, int obs_agent_id, const float* obs,
                 const int32_t* avail, const int32_t* reset, const double* epsilon, const double* uniforms, unsigned long long seed,
                 unsigned long long* counter, float* hidden, int32_t* last_action, int32_t* actions, int use_graph, void* stream);

/* ---- SCC: replaces SCCModel's train and explore graphs (xt/model/scc/scc_tf.py:195-707) -----------------------------
 * The agent network and its explore step are QMIX's (above): fc1 / GRU / fc2 in the same layout, with the same limits
 * on H, n_agents and n_actions.  A weight set is one flat float buffer [fc1 | GRU | fc2 | critic nets | head]:
 *   - multi-channel critic (enable_critic_multi_channel, scc_tf.py:290-313): one net per agent group, in group order,
 *     each dense(U, relu) -> dense(U, relu) on one agent's (obs, one-hot action) slice of D = o + A floats (o = obs_shape
 *     - n_actions - n_agents, the raw observation width); the head kernel is [n_agents U, 1] (concat) or [U, 1] (add);
 *   - single-channel critic (scc_tf.py:283-289): one net dense(U, relu) -> dense(U, relu) on the n_agents D row and a
 *     [U, 1] head kernel;
 *   then the head bias [1], at float offset head_off (a multiple of 4).  The nets are bound to their slices (in this order,
 *   each starting at a multiple of 4 floats) of the eval set and of a gradient buffer with the same layout.  The target
 *   set has the same layout (only its critic part is read: the reference has no target agent); an explore set needs only
 *   the agent part.
 * Limits (XTB_ERR_ARG at create, before any launch): those of QMIX's agent (H <= 137, n_agents <= 32, n_actions <= 255);
 * 1 <= U <= 512 (dense_unit_number); 0 <= n_groups <= 8 with every group non-empty and the groups summing to n_agents
 * (the reference's reshape would not fit otherwise); channel_merge 0 (concat) or 1 (add); mc_sample_times >= 1 when
 * n_agents > 2; critic nets holding B L group-size rows (multi-channel) or B L V rows (single-channel, V below). */
typedef struct xtb_scc xtb_scc;
#define XTB_SCC_MAX_GROUPS 8
typedef struct xtb_scc_desc {
  int32_t batch;            /* B episodes per training batch */
  int32_t episode_limit;    /* L */
  int32_t n_agents;
  int32_t n_groups;         /* 0: single-channel critic; else the multi-channel critic's group count */
  int32_t group[XTB_SCC_MAX_GROUPS];   /* agents per group (agent_group_dict, scc_tf.py:56-60) */
  int32_t channel_merge;    /* 0 concat, 1 add */
  int32_t mc_sample_times;
  float gamma;
  long long gru_off;        /* offset (floats) of gates/kernel in a weight set */
  long long head_off;       /* offset (floats) of the critic head's kernel */
  int32_t act_envs;         /* as xtb_qmix_desc's */
} xtb_scc_desc;
/* critic: n_groups nets (1 when n_groups = 0) */
int xtb_scc_create(xtb_net* fc1, xtb_net* fc2, xtb_net* const* critic, const xtb_scc_desc* desc, xtb_scc** out);
void xtb_scc_destroy(xtb_scc* q);
typedef struct xtb_scc_batch {
  const float* obs;         /* [B, L+1, n_agents, obs_dim] agent inputs */
  const float* raw_obs;     /* [B, L+1, n_agents, o] batch["obs"]; steps t < L build the critic states */
  const int32_t* seq_len;   /* [B n_agents] GRU sequence lengths, read at run time, clamped to [0, L+1] */
  const int32_t* actions;   /* [B, L, n_agents] taken actions in [0, A) */
  const float* reward;      /* [B, L] */
  const float* terminated;  /* [B, L] */
  const float* mask;        /* [B, L] */
  const uint32_t* subsets;  /* [n_agents, mc_sample_times] agent bitmasks of the Monte-Carlo subsets (scc_tf.py:665-668);
                               read by the single-channel critic with n_agents > 2 only (else may be NULL) */
} xtb_scc_batch;
/* SCCModel.train (scc_tf.py:535-564 with the graph of 321-448) as one step:
 *   - critic states s[b, t] = concat_a [raw_obs[b, t, a], one_hot(actions[b, t, a])], t < L, read shifted as the
 *     reference's alias leaves them: s'[b, t] = s[b, min(t + 1, L - 1)] for every critic evaluation;
 *   - the eval agent over all B (L+1) n_agents rows; the eval and target critics on s';
 *   - credits from the eval critic before the update: n_agents <= 2, V(s') - V(s' with agent i's slice zeroed);
 *     n_agents > 2, the mean over the subsets S of V(s' with the actions of S zeroed) - V(... of S and i zeroed).  In
 *     multi-channel mode only agent i's channel differs, so this is u_i(s') - u_i(masked), independent of S;
 *   - mixer loss sum (mask (V - (r + gamma (1 - term) V_target)))^2 / sum mask; actor loss
 *     sum (mask Q_chosen - mask credit)^2 / (n_agents sum mask);
 *   - one step of critic_opt (Adam, over [critic nets | head]) and of actor_opt (xtb_opt_use_rmsprop_plain, over
 *     [fc1 | GRU | fc2]), each clipping every variable by norm or neither (the reference clips both only when
 *     actor_grad_norm_clip > 0), then the nets' weight refresh.
 * loss_out[0] = mixer loss, loss_out[1] = actor loss, summed in a fixed order.  XTB_ERR_STATE while a communicator is
 * installed.  Single-channel critics with n_agents > 2 evaluate 2 n_agents mc_sample_times credit variants per row. */
int xtb_scc_train(xtb_scc* q, xtb_adam* critic_opt, xtb_adam* actor_opt, const float* target, const xtb_scc_batch* batch,
                  float* loss_out, int use_graph, void* stream);
/* SCCModel.infer_actions: as xtb_qmix_infer. */
int xtb_scc_infer(xtb_scc* q, const float* explore, const float* obs, float* hidden, float* q_out, int use_graph, void* stream);
/* SCC's acting: as xtb_qmix_act. */
int xtb_scc_act(xtb_scc* q, const float* explore, int n_envs, int obs_last_action, int obs_agent_id, const float* obs,
                const int32_t* avail, const int32_t* reset, const double* epsilon, const double* uniforms, unsigned long long seed,
                unsigned long long* counter, float* hidden, int32_t* last_action, int32_t* actions, int use_graph, void* stream);
/* SCCModel.get_mixer_output (scc_tf.py:500-503): v_out[r] = V_eval(states[r]) for states [rows, n_agents D], rows <= B L. */
int xtb_scc_critic(xtb_scc* q, const float* states, int rows, float* v_out, int use_graph, void* stream);

/* ---- QMIX / SCC episode replay in HBM: QMixAlg's ReplayBuffer (xt/algorithm/qmix/episode_buffer_np.py) and the batch
 * assembly of QMixAlg.train (qmix_alg.py: build_inputs, the mask, max_t_filled) ------------------------------------------
 * One device allocation holds `capacity` episode rows of T = episode_limit + 1 steps.  A row is, in this order, each field
 * starting at a multiple of 16 bytes:
 *   state f32 [T, state_dim] | obs f32 [T, n_agents, obs_dim] | actions i32 [T, n_agents] |
 *   actions_onehot f32 [T, n_agents, A] | avail_actions i32 [T, n_agents, A] | reward f32 [T] | terminated u8 [T] |
 *   filled i64 [T]
 * The caller packs a row on the host and stores it with xtb_episode_replay_add; the ring bookkeeping (which slot,
 * how many are stored) is the caller's, as in ReplayBuffer.insert_episode_batch, and the library mirrors the stored count
 * (the highest slot written + 1).  The draws are the caller's too: each call below takes B host episode ids, each in
 * [0, stored count), with 1 <= B <= stored count.  It copies them into the replay's id buffer with one staged upload and
 * then reads them on the device, so one captured graph serves every draw, every episode length and the whole fill and
 * wrap of the ring.
 * Limits (XTB_ERR_ARG at create): capacity >= 1, episode_limit >= 1, 1 <= n_agents <= 32, 1 <= n_actions <= 255,
 * obs_dim >= 0, state_dim >= 1.  Add, gather and the train calls return XTB_ERR_STATE, launching nothing, while a
 * communicator is installed, and XTB_ERR_ARG, launching nothing, for a bad slot, row size, batch or id. */
typedef struct xtb_episode_replay xtb_episode_replay;
/* A drawn batch (device arrays; any may be NULL, and is then not written). */
typedef struct xtb_episode_batch {
  float* obs;           /* [B, L+1, n_agents, obs_dim (+ A) (+ n_agents)] agent inputs: obs | one-hot of the previous step's
                           action (zeros at t = 0), with obs_last_action | one-hot of the agent id, with obs_agent_id */
  float* raw_obs;       /* [B, L+1, n_agents, obs_dim] the stored observations */
  int32_t* seq_len;     /* [B n_agents] max_t_filled(): the largest per-episode sum of filled, for every sequence */
  float* avail;         /* [B, L+1, n_agents, A] */
  int32_t* actions;     /* [B, L, n_agents] */
  float* state;         /* [B, L, state_dim] state[:, :-1] */
  float* next_state;    /* [B, L, state_dim] state[:, 1:] */
  float* reward;        /* [B, L] */
  float* terminated;    /* [B, L] */
  float* mask;          /* [B, L] filled[:, :-1] with mask[:, 1:] *= 1 - terminated[:, :-1], in float32 */
} xtb_episode_batch;
/* obs_last_action / obs_agent_id: build_inputs' switches (0 or 1). */
int xtb_episode_replay_create(int capacity, int episode_limit, int n_agents, int n_actions, int obs_dim, int state_dim,
                              int obs_last_action, int obs_agent_id, xtb_episode_replay** out);
void xtb_episode_replay_destroy(xtb_episode_replay* r);
/* Bytes of one packed episode row. */
long long xtb_episode_replay_row_bytes(const xtb_episode_replay* r);
/* Store the packed row at host `row` (`bytes` must be the row size) in slot `slot` with one staged upload.  Every action
 * of the first episode_limit steps must be in [0, A) and the sum of filled in [0, L+1] (XTB_ERR_ARG otherwise): the
 * batch reads them as indices and sequence lengths. */
int xtb_episode_replay_add(xtb_episode_replay* r, int slot, const void* row, long long bytes, void* stream);
/* The batch of the B episodes `ids` (host) into *out; *max_t_out (device, may be NULL) = max_t_filled(). */
int xtb_episode_replay_gather(xtb_episode_replay* r, int batch, const int32_t* ids, const xtb_episode_batch* out, int32_t* max_t_out,
                              void* stream);
/* QMixAlg.train on the device: the gather into *batch, then xtb_qmix_train of q / opt / target on it, as one call (one
 * graph when use_graph).  B must be q's batch and the replay's shapes q's (agent input width, n_agents, A, L, state_dim).
 * *loss_out as xtb_qmix_train; *max_t_out (device) = max_t_filled(). */
int xtb_qmix_replay_train(xtb_episode_replay* r, xtb_qmix* q, xtb_adam* opt, const float* target, int batch, const int32_t* ids,
                          const xtb_qmix_batch* bufs, float* loss_out, int32_t* max_t_out, int use_graph, void* stream);
/* SCCAlg.train on the device: as xtb_qmix_replay_train with xtb_scc_train; the raw obs comes from the ring (obs_dim must
 * be q's o).  bufs->subsets is the caller's, as for xtb_scc_train. */
int xtb_scc_replay_train(xtb_episode_replay* r, xtb_scc* q, xtb_adam* critic_opt, xtb_adam* actor_opt, const float* target, int batch,
                         const int32_t* ids, const xtb_scc_batch* bufs, float* loss_out, int32_t* max_t_out, int use_graph,
                         void* stream);

/* ---- InfoFlow recommender DQN: replaces DqnInfoFlowModel's Keras graph (xt/model/dqn/dqn_rec_model.py:63-169) and the
 * target computation of DQNInfoFlowAlg.train (xt/algorithm/dqn/dqn_infoflw_alg.py:76-174) --------------------------------
 * Inputs are int32 ids in [0, vocab) (Keras Embedding's cast; not checked on the device): user [user_dim], history_click
 * and history_no_click [5 item_dim], item [item_dim].  With E = emb_dim and U = item_dim E, a weight set is one flat
 * float buffer [gru | gru_1 | head]: each GRU is Keras GRU v1 (hard_sigmoid gates, reset_after=False, last output only)
 * with kernel [U, 3U], recurrent_kernel [U, 3U] and bias [3U] back to back (gate columns [z | r | h]), gru at offset 0
 * on the clicked history and gru_1 at gru1_off on the viewed one; the head is one net of three dense layers, dense
 * (relu) on rows of D = user_dim E + 3U floats [Flatten(emb(user)) | h_click | h_noclick | Flatten(emb(item))], dense_1
 * (relu) and q_value (1 wide, activation last_act), bound at head_off of the set and of a gradient buffer with the same
 * layout.  The embedding table [vocab, E] is frozen and lives outside the set.
 * Limits (XTB_ERR_ARG at create): every size positive, U <= 137 (the GRU kernels' shared-memory plan), gru1_off and
 * head_off multiples of 64 with the slices in order and not overlapping. */
typedef struct xtb_infoflow xtb_infoflow;
typedef struct xtb_infoflow_desc {
  int32_t user_dim, item_dim, emb_dim, vocab;
  int32_t batch;            /* B transitions per training step */
  int32_t last_act;         /* xtb_act of q_value */
  double gamma;
  long long gru_off;        /* 0 */
  long long gru1_off;       /* offset (floats) of gru_1/kernel */
  long long head_off;       /* offset (floats) of dense/kernel */
  const float* table;       /* [vocab, emb_dim] Emb/embeddings (device) */
} xtb_infoflow_desc;
int xtb_infoflow_create(const xtb_infoflow_desc* desc, xtb_infoflow** out);
void xtb_infoflow_destroy(xtb_infoflow* f);
/* One minibatch of B transitions (device arrays).  The candidates of the next states are ragged: transition b's are
 * rows cand_off[b] .. cand_off[b+1] of cand_item, and cand_off[B] must equal n_cand. */
typedef struct xtb_infoflow_batch {
  const int32_t* user;          /* [B, user_dim] */
  const int32_t* click;         /* [B, 5 item_dim] */
  const int32_t* noclick;       /* [B, 5 item_dim] */
  const int32_t* item;          /* [B, item_dim] the action taken */
  const int32_t* next_user;     /* [B, user_dim] */
  const int32_t* next_click;    /* [B, 5 item_dim] */
  const int32_t* next_noclick;  /* [B, 5 item_dim] */
  const int32_t* cand_off;      /* [B + 1], read on the device */
  const int32_t* cand_item;     /* [cand_cap, item_dim], rows past n_cand unread */
  const double* reward;         /* [B] */
  const int32_t* done;          /* [B] nonzero: done */
  const float* label;           /* NULL: the target pass computes the targets; else the targets [B] of a plain fit step
                                   (DqnInfoFlowModel.train), and the next_* / cand_* / reward / done fields may be NULL */
  int32_t n_cand;               /* candidate rows of the batch */
  int32_t cand_cap;             /* rows the target pass runs: >= max(n_cand, B), <= the head's max batch; callers keep it
                                   to a few values (a power of two that only grows) so that few graphs are captured */
} xtb_infoflow_batch;
/* DQNInfoFlowAlg.train's target and DqnInfoFlowModel.train (one Keras fit step) as one graph:
 *   1. target pass with the online weights: both GRUs once per transition on the next histories, the head on cand_cap
 *      rows [next user | h_click | h_noclick | candidate item] (rows past n_cand zeroed), then
 *      target[b] = reward[b] if done[b] else (float)(max_c q_c * gamma + reward[b]) in float64 (NaN propagates);
 *   2. the training forward on the B transitions, the mse loss (*loss_out, before the update, summed in a fixed order),
 *      the head's backward with d loss / d input, the GRUs' backward from the h_click / h_noclick slices (no gradient
 *      into the frozen table) and their weight gradients as GEMMs over all step rows;
 *   3. one step of `opt` (Keras Adam, epsilon 1e-7, no clipping) over [gru | gru_1 | head], then the head's weight refresh.
 * With batch->label the target pass is skipped and the labels are the targets.  target_out [B] (may be NULL) receives
 * the targets.  XTB_ERR_STATE while a communicator is installed: the GRUs'
 * gradients are not summed over ranks. */
int xtb_infoflow_train(xtb_infoflow* f, xtb_net* head, xtb_adam* opt, const xtb_infoflow_batch* batch, float* loss_out,
                       float* target_out, int use_graph, void* stream);
/* DqnInfoFlowModel.predict (dqn_rec_model.py:156-169): q_out[r] for n rows in the tiled dict form (user [n, user_dim],
 * click / noclick [n, 5 item_dim], item [n, item_dim]), each row its own GRU sequences; n <= the head's max batch. */
int xtb_infoflow_predict(xtb_infoflow* f, xtb_net* head, const int32_t* user, const int32_t* click, const int32_t* noclick,
                         const int32_t* item, int n, float* q_out, int use_graph, void* stream);

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
