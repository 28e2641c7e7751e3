// learners.cu -- the RL learners on the layer engine and rl_kernels.cuh: the single-kernel losses, sampling and returns,
// PPO (train and rollout inference), IMPALA and IMPALA-Keras, MuZero (model, tree search and replay), DQN with the
// dueling TD step, and prioritized replay.
#include "engine.cuh"

#include <cmath>

#include "rl_kernels.cuh"
#include "per.cuh"
#include "muzero_replay.cuh"
#include "stager.cuh"


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
// opt-in of the fused heads kernels to the large dynamic shared-memory carve-out, once per process: the learner entry
// points that may launch them call it before any stream capture
static int heads_kernel_attrs() {
  static bool done = false;
  if (done) return XTB_OK;
  cudaError_t e = cudaSuccess;
  auto opt_in = [&](const void* k) { if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem); };
  for (const auto& h : kHeadsKernels<PpoLoss>) opt_in((const void*)h.kern);
  for (const auto& h : kHeadsKernels<DuelingTdLoss>) opt_in((const void*)h.kern);
  for (const auto& h : kHeadsKernels<PpoGaussLoss>) opt_in((const void*)h.kern);
  if (e != cudaSuccess) return fail(XTB_ERR_CUDA, "kernel attributes: %s", cudaGetErrorString(e));
  done = true;
  return XTB_OK;
}

// ------------------------------------------------------------------------------------------
// heads, GAE, losses
// ------------------------------------------------------------------------------------------
extern "C" int xtb_categorical_sample(const float* logits, int batch, int adim, const float* uniforms,
                                      uint64_t seed, uint64_t offset, int32_t* action, float* logp, void* stream) {
  if (!logits || !action || !logp || batch <= 0 || adim <= 0) return fail(XTB_ERR_ARG, "xtb_categorical_sample: bad argument");
  XLAUNCH(sample_kernel<Categorical>, (batch + 127) / 128, 128, 0, S(stream), logits, (const float*)nullptr, batch, batch, adim,
          uniforms, seed, offset, (const unsigned long long*)nullptr, 0, action, logp, (const float*)nullptr, (float*)nullptr);
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
  if (n_env < 0 || n_step < 0) return fail(XTB_ERR_ARG, "xtb_gae: negative size");
  if (n_env == 0 || n_step == 0) return XTB_OK;   // empty rollout: nothing to do
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
  XLAUNCH(sample_kernel<DiagGaussian>, (batch + 127) / 128, 128, 0, S(stream), mean, log_std, batch, batch, adim, normals, seed,
          offset, (const unsigned long long*)nullptr, 0, action, logp, (const float*)nullptr, (float*)nullptr);
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

// dqn_loss_kernel with its optional per-sample weights `wt` and |TD error| output `td_abs` (NULL: the plain step)
static int dqn_td_loss(const float* q, const float* q_next_target, const float* q_next_online, const int32_t* idx,
                       const int32_t* action, const float* reward, const uint8_t* done, const float* disc, int batch, int adim,
                       float gamma, float huber_delta, float inv_count, const float* wt, float* dq, float* y_out, float* td_abs,
                       float* loss_out, void* stream) {
  XLAUNCH(dqn_loss_kernel, (batch + 127) / 128, 128, 0, S(stream), q, q_next_target, q_next_online, idx, action, reward, done, disc,
          batch, adim, gamma, huber_delta, inv_count, wt, dq, y_out, td_abs, loss_out);
  LAUNCH_CHECK();
  return XTB_OK;
}
extern "C" int xtb_dqn_td_loss_grad(const float* q, const float* q_next_target, const float* q_next_online, const int32_t* idx,
                                    const int32_t* action, const float* reward, const uint8_t* done, const float* disc, int batch,
                                    int adim, float gamma, float huber_delta, float inv_count, const float* wt, float* dq,
                                    float* y_out, float* td_abs, float* loss_out, void* stream) {
  if (!q || !q_next_target || !action || !reward || !done || !dq || !loss_out) return fail(XTB_ERR_ARG, "xtb_dqn_td_loss_grad: null pointer");
  if (batch <= 0 || adim <= 0) return fail(XTB_ERR_ARG, "xtb_dqn_td_loss_grad: bad sizes");
  return dqn_td_loss(q, q_next_target, q_next_online, idx, action, reward, done, disc, batch, adim, gamma, huber_delta, inv_count,
                     wt, dq, y_out, td_abs, loss_out, stream);
}
extern "C" int xtb_dqn_loss_grad(const float* q, const float* q_next_target, const float* q_next_online,
                                 const int32_t* action, const float* reward, const uint8_t* done, int batch,
                                 int adim, float gamma, float inv_count, float* dq, float* y_out,
                                 float* loss_out, void* stream) {
  return xtb_dqn_td_loss_grad(q, q_next_target, q_next_online, nullptr, action, reward, done, nullptr, batch, adim, gamma, 0.f,
                              inv_count, nullptr, dq, y_out, nullptr, loss_out, stream);
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
  int blocks = std::max(1, std::min(kSMs, (mb + 7) / 8));      // one sample per warp up to 8 * kSMs = 1056 samples
  const int HK = lpi.K, nacc = HK * adim + 3 * HK + adim + 2 + (LOSS::kLogStd ? adim : 0);
  a.part = (float*)(net->ws + net->heads_part_off); a.slab = (nacc + 3) & ~3;
  size_t shb = (size_t)8 * nacc * sizeof(float);
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

// the heads_kernel (infer: infer_heads_kernel) entry the PPO calls launch for these heads, (0, 0) when layer by layer
extern "C" int xtb_ppo_heads_plan(const xtb_net* net, int pi_t, int v_t, int infer, int* kpl, int* amax) {
  const char* fn = "xtb_ppo_heads_plan";
  if (!net || !kpl || !amax) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (int rc = ppo_heads_check(fn, net, pi_t, v_t, 0)) return rc;
  *kpl = *amax = 0;
  if (!ppo_heads_fusable(net, pi_t, v_t, infer != 0)) return XTB_OK;
  const int K = net->L[pi_t - 1].K, A = net->tsize[pi_t];
  if (infer) {
    const auto* e = heads_pick(kInferHeadsKernels<Categorical>, K, A);
    *kpl = e->kpl; *amax = e->amax;
  } else {
    const auto* e = heads_pick(kHeadsKernels<PpoLoss>, K, A);
    *kpl = e->kpl; *amax = e->amax;
  }
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
  if (int rc = heads_kernel_attrs()) return rc;
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
  void* buf = nullptr;
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
  if (int rc = carve_scratch("xtb_muzero_create", &m->buf, {{&m->hbuf, R1 * H}, {&m->xbuf, RK * (H + A)}, {&m->rlog, RK * Sr},
                                                            {&m->dr, RK * Sr}, {&m->tv, R1 * Sv}, {&m->tr, RK * Sr}, {&m->dh, R1 * H},
                                                            {&m->dx, Bm * (H + A)}, {&m->part, m->n_part}})) {
    delete m;
    return rc;
  }
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
  auto* tr = new xtb_muzero_tree();
  MctsTrees& t = tr->t;
  if (int rc = carve_scratch("xtb_muzero_tree_create", &tr->buf,
                             {{&t.hid, NN * E * H}, {&t.reward, E * NN}, {&t.prior, E * NN * A}, {&t.vsum, E * NN * A},
                              {&t.visits, E * NN * A}, {&t.child, E * NN * A}, {&t.root_vsum, E}, {&t.root_visits, E},
                              {&t.minmax, E * 2}, {&t.path_node, E * NN}, {&t.path_act, E * NN}, {&t.depth, E},
                              {&tr->reward, E}, {&tr->value, E}, {&tr->policy, E * A}})) {
    delete tr;
    return rc;
  }
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

// ---- MuZero trajectory replay (muzero_replay.cuh) ---------------------------------------------------------------------
// The pool, the slot table, both tree levels and the state are one device allocation; `count` mirrors the device's so
// that a draw from an empty buffer is refused before a launch.
struct xtb_muzero_replay {
  MzrDev d{};
  int capacity = 0, max_batch = 0, count = 0;
  long long pool = 0;
  void* buf = nullptr;
  float* vbuf = nullptr;       // [max(pool, max_batch)] float values: value inference of an add, post-step values of a train
};

extern "C" int xtb_muzero_replay_create(int capacity, long long pool_steps, int unroll, long long obs_bytes, int n_actions,
                                        int max_batch, xtb_muzero_replay** out) {
  const char* fn = "xtb_muzero_replay_create";
  if (!out) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (capacity < 1 || capacity > (1 << 30) || pool_steps < 1 || pool_steps > (1LL << 36) || unroll < 1 || obs_bytes < 1 ||
      n_actions < 1 || n_actions > MZ_MAX_SUPPORT || max_batch < 1)
    return fail(XTB_ERR_ARG, "%s: capacity %d / pool_steps %lld / unroll %d / obs_bytes %lld / actions %d / max_batch %d out of range",
                fn, capacity, pool_steps, unroll, obs_bytes, n_actions, max_batch);
  auto* r = new xtb_muzero_replay();
  MzrDev& d = r->d;
  d.tleaves = 1;
  while (d.tleaves < capacity) d.tleaves *= 2;
  d.row_bytes = obs_bytes; d.K = unroll; d.A = n_actions;
  const long long P = pool_steps;
  if (int rc = carve_scratch(fn, &r->buf, {{&d.obs, P * obs_bytes}, {&d.action, P}, {&d.tv, P}, {&d.reward, P},
                                           {&d.child, P * n_actions}, {&d.traj, 2LL * d.tleaves}, {&d.forest, 4 * P},
                                           {&d.slot, (long long)capacity}, {&d.st, 1}, {&d.wt, (long long)max_batch},
                                           {&r->vbuf, std::max<long long>(P, max_batch)}})) {
    delete r;
    return rc;
  }
  r->capacity = capacity; r->pool = P; r->max_batch = max_batch;
  *out = r;
  return XTB_OK;
}

extern "C" void xtb_muzero_replay_destroy(xtb_muzero_replay* r) {
  if (!r) return;
  drop_graphs_of(r);
  cudaDeviceSynchronize();
  cudaFree(r->buf);
  delete r;
}

static int mzr_check(const char* fn, const xtb_muzero_replay* r, bool missing) {
  if (!r || missing) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (g_comm) return fail(XTB_ERR_STATE, "%s: data-parallel training (communicator) is not supported", fn);
  return XTB_OK;
}
// the model reads the replay's observation rows, actions and unroll
static int mzr_model_check(const char* fn, const xtb_muzero_replay* r, const xtb_muzero* m) {
  const long long row = (long long)m->rep->tsize[0] * (m->rep->desc.input_u8 ? 1 : (long long)sizeof(float));
  if (m->K != r->d.K || m->A != r->d.A || row != r->d.row_bytes)
    return fail(XTB_ERR_ARG, "%s: model (unroll %d, %d actions, %lld-byte observations) does not match the replay (%d, %d, %lld)", fn,
                m->K, m->A, row, r->d.K, r->d.A, r->d.row_bytes);
  return XTB_OK;
}
static int mzr_batch_check(const char* fn, const xtb_muzero_replay* r, int batch, const xtb_muzero_replay_batch* out) {
  if (!out || !out->obs || !out->action || !out->target_value || !out->target_reward || !out->target_policy)
    return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (batch < 1 || batch > r->max_batch) return fail(XTB_ERR_ARG, "%s: batch %d not in [1, %d]", fn, batch, r->max_batch);
  if (r->count < 1) return fail(XTB_ERR_STATE, "%s: no trajectory stored", fn);
  return XTB_OK;
}
// an update writes trajectory leaf k for every batch position k: each must be a stored slot, as the host's
// update_priorities requires
static int mzr_update_batch_check(const char* fn, const xtb_muzero_replay* r, int batch) {
  if (batch < 1 || batch > r->max_batch) return fail(XTB_ERR_ARG, "%s: batch %d not in [1, %d]", fn, batch, r->max_batch);
  if (batch > r->count) return fail(XTB_ERR_ARG, "%s: batch %d exceeds the %d stored slots", fn, batch, r->count);
  return XTB_OK;
}

static int mzr_sample_launch(xtb_muzero_replay* r, int B, const double* u, int32_t* slot, int32_t* pos, const xtb_muzero_replay_batch& o,
                             cudaStream_t st) {
  XLAUNCH(mzr_draw_kernel, 1, std::min(kMzrThreads, (B + 31) / 32 * 32), 0, st, r->d, B, u, slot, pos);
  LAUNCH_CHECK();
  XLAUNCH(mzr_gather_kernel, B, 256, 0, st, r->d, (const int32_t*)slot, (const int32_t*)pos, (uint8_t*)o.obs, o.action, o.target_value,
          o.target_reward, o.target_policy);
  LAUNCH_CHECK();
  return XTB_OK;
}
static int mzr_update_launch(xtb_muzero_replay* r, int B, const int32_t* slot, const int32_t* pos, const float* vf, const double* vd,
                             cudaStream_t st) {
  XLAUNCH(mzr_update_kernel, 1, kMzrThreads, 0, st, r->d, B, slot, pos, vf, vd);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_muzero_replay_add(xtb_muzero_replay* r, xtb_muzero* m, int slot, long long off, int evict_first, int n_evict,
                                     const void* obs, const int32_t* action, const double* target_value, const float* reward,
                                     const float* child_visits, int len, const double* values, void* stream) {
  const char* fn = "xtb_muzero_replay_add";
  if (int rc = mzr_check(fn, r, !obs || !action || !target_value || !reward || !child_visits || (!values && !m))) return rc;
  const MzrDev& d = r->d;
  if (len <= d.K + 1 || len > r->pool) return fail(XTB_ERR_ARG, "%s: length %d not in [%d, %lld]", fn, len, d.K + 2, r->pool);
  if (slot < 0 || slot >= r->capacity || off < 0 || off + len > r->pool)
    return fail(XTB_ERR_ARG, "%s: slot %d / pool range [%lld, %lld) outside the replay", fn, slot, off, off + len);
  if (evict_first < 0 || evict_first >= r->capacity || n_evict < 0 || n_evict >= r->capacity ||
      (slot - evict_first + r->capacity) % r->capacity < n_evict)
    return fail(XTB_ERR_ARG, "%s: eviction range %d + %d is not a set of other slots", fn, evict_first, n_evict);
  if (!values) {
    if (int rc = mz_check(fn, m, false, nullptr, 1)) return rc;
    if (int rc = mzr_model_check(fn, r, m)) return rc;
  }
  cudaStream_t st = S(stream);
  CUDA_TRY(cudaMemcpyAsync(d.obs + off * d.row_bytes, obs, (size_t)len * d.row_bytes, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d.action + off, action, (size_t)len * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d.tv + off, target_value, (size_t)len * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d.reward + off, reward, (size_t)len * sizeof(float), cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d.child + off * d.A, child_visits, (size_t)len * d.A * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (!values) {
    for (int s0 = 0; s0 < len; s0 += m->max_batch) {
      const int n = std::min(m->max_batch, len - s0);
      int rc = mz_initial_launch(m, d.obs + (off + s0) * d.row_bytes, n, nullptr, r->vbuf + s0, nullptr, st);
      if (rc) return rc;
    }
  }
  XLAUNCH(mzr_add_kernel, 1, kMzrThreads, 0, st, r->d, slot, off, len, evict_first, n_evict, r->capacity,
          values ? (const float*)nullptr : (const float*)r->vbuf, values);
  LAUNCH_CHECK();
  r->count = std::max(r->count, slot + 1);
  return XTB_OK;
}

extern "C" int xtb_muzero_replay_sample(xtb_muzero_replay* r, int batch, const double* uniforms, int32_t* slot_out, int32_t* pos_out,
                                        const xtb_muzero_replay_batch* out, void* stream) {
  const char* fn = "xtb_muzero_replay_sample";
  if (int rc = mzr_check(fn, r, !uniforms || !slot_out || !pos_out)) return rc;
  if (int rc = mzr_batch_check(fn, r, batch, out)) return rc;
  return mzr_sample_launch(r, batch, uniforms, slot_out, pos_out, *out, S(stream));
}

extern "C" int xtb_muzero_replay_update(xtb_muzero_replay* r, int batch, const int32_t* slot, const int32_t* pos, const double* values,
                                        void* stream) {
  const char* fn = "xtb_muzero_replay_update";
  if (int rc = mzr_check(fn, r, !slot || !pos || !values)) return rc;
  if (int rc = mzr_update_batch_check(fn, r, batch)) return rc;
  return mzr_update_launch(r, batch, slot, pos, nullptr, values, S(stream));
}

extern "C" int xtb_muzero_replay_train(xtb_muzero_replay* r, xtb_muzero* m, xtb_adam* opt, int batch, const double* uniforms,
                                       int32_t* slot_out, int32_t* pos_out, const xtb_muzero_replay_batch* out, float loss_offset,
                                       float* loss_out, int32_t* status_out, int use_graph, void* stream) {
  const char* fn = "xtb_muzero_replay_train";
  if (int rc = mzr_check(fn, r, !uniforms || !slot_out || !pos_out || !loss_out || !status_out)) return rc;
  if (int rc = mz_check(fn, m, !opt, opt, batch)) return rc;
  if (int rc = mzr_batch_check(fn, r, batch, out)) return rc;
  if (int rc = mzr_update_batch_check(fn, r, batch)) return rc;
  if (int rc = mzr_model_check(fn, r, m)) return rc;
  const xtb_muzero_replay_batch o = *out;
  return run_graph(capture_key(kMuzeroReplayTrain, {m->rep, m->dyn, m->pred, m, opt, r}, r, m, batch, uniforms, slot_out, pos_out,
                               o.obs, o.action, o.target_value, o.target_reward, o.target_policy, loss_offset, loss_out, status_out),
                   use_graph, stream, [&](void* sv) -> int {
    cudaStream_t st = S(sv);
    int rc = mzr_sample_launch(r, batch, uniforms, slot_out, pos_out, o, st);
    if (rc) return rc;
    xtb_muzero_batch bt{o.obs, o.action, o.target_value, o.target_reward, o.target_policy, m->K};
    rc = mz_train_launch(m, opt, bt, batch, loss_offset, loss_out, r->vbuf, st);
    if (rc) return rc;
    rc = mzr_update_launch(r, batch, slot_out, pos_out, r->vbuf, nullptr, st);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(status_out, &r->d.st->status, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    return XTB_OK;
  });
}

extern "C" int xtb_muzero_replay_state(const xtb_muzero_replay* r, int* count, int* status, int* tree_leaves,
                                       xtb_muzero_replay_slot* slots, double* traj_tree, double* forest) {
  if (!r) return fail(XTB_ERR_ARG, "xtb_muzero_replay_state: null pointer");
  CUDA_TRY(cudaDeviceSynchronize());
  MzrState s;
  CUDA_TRY(cudaMemcpy(&s, r->d.st, sizeof s, cudaMemcpyDeviceToHost));
  if (slots) CUDA_TRY(cudaMemcpy(slots, r->d.slot, sizeof(xtb_muzero_replay_slot) * r->capacity, cudaMemcpyDeviceToHost));
  if (traj_tree) CUDA_TRY(cudaMemcpy(traj_tree, r->d.traj, sizeof(double) * 2 * r->d.tleaves, cudaMemcpyDeviceToHost));
  if (forest) CUDA_TRY(cudaMemcpy(forest, r->d.forest, sizeof(double) * 4 * r->pool, cudaMemcpyDeviceToHost));
  if (count) *count = s.count;
  if (status) *status = s.status;
  if (tree_leaves) *tree_leaves = r->d.tleaves;
  return XTB_OK;
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

// the heads_kernel<DuelingTdLoss> entry the DQN steps launch for q_tensor, (0, 0) when they run layer by layer
extern "C" int xtb_dqn_heads_plan(const xtb_net* net, int q_tensor, int* kpl, int* amax) {
  const char* fn = "xtb_dqn_heads_plan";
  if (!net || !kpl || !amax) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (q_tensor < 1 || q_tensor > (int)net->L.size()) return fail(XTB_ERR_ARG, "%s: bad head tensor", fn);
  *kpl = *amax = 0;
  if (!dueling_fusable(net, q_tensor)) return XTB_OK;
  const LayerPlan& lq = net->L[q_tensor - 1];
  const auto* e = heads_pick(kHeadsKernels<DuelingTdLoss>, net->L[lq.d.src - 1].K, net->tsize[lq.d.src]);
  *kpl = e->kpl; *amax = e->amax;
  return XTB_OK;
}

// The online half of the dueling TD step in one heads_kernel launch (heads_fused with the value stream as the pi head
// and the adv stream as the value head): both streams' forward, the combine, TD target and loss, the streams' backward
// and the gradient wrt the hidden tensor; then the backward pass of the layers below.
static int dueling_td_fused(xtb_net* net, const void* obs, const int32_t* idx, const int32_t* action, const float* reward,
                            const uint8_t* done, const float* disc, int n, float gamma, float huber, int q_tensor,
                            const float* qn_t, const float* qn_o, float inv_count, const float* wt, float* td_abs, float* loss_out,
                            cudaStream_t st) {
  const LayerPlan& lq = net->L[q_tensor - 1];
  const int h = net->L[lq.d.src - 1].d.src;
  const unsigned skip = (1u << (q_tensor - 1)) | (1u << (lq.d.src - 1)) | (1u << (lq.d.k - 1));
  int rc = net_forward_impl(net, nullptr, obs, idx, n, st, skip, 1u << h);
  if (rc) return rc;
  PpoHeadsArgs a;
  memset(&a, 0, sizeof a);
  a.idx = idx; a.action = action; a.reward = reward; a.done = done; a.disc = disc; a.qn_t = qn_t; a.qn_o = qn_o; a.loss_in = loss_out;
  a.gamma = gamma; a.huber = huber; a.inv_count = inv_count; a.wt = wt; a.td_abs = td_abs;
  return heads_fused<DuelingTdLoss>(net, obs, a, n, lq.d.src, lq.d.k, skip, -1, loss_out, st);
}

// DQN.train (xt/algorithm/dqn/dqn.py:61-103) on a device replay ring: rows idx[0..n) of (obs, next_obs, action, reward,
// done[, disc]); target-network forward on s', optional double-DQN online forward on s', online forward on s, TD target +
// loss gradient, backward, clip + Adam.  qn_t / qn_o: scratch [n, adim] (qn_o NULL = plain DQN).  Reference mode:
// disc = NULL, huber_delta = 0.  With a communicator every rank holds n of world*n samples: inv_count = 1/(world*n*adim).
// wt / td_abs (both may be NULL): per-sample loss weights and the |TD error| output of the loss kernels.
static int dqn_check(const char* fn, bool missing, xtb_net* net, xtb_net* target, xtb_adam* opt, int n_sample, int q_tensor) {
  if (int rc = learner_check(fn, missing, net, opt, n_sample, true)) return rc;
  if (!target->ws) return fail(XTB_ERR_STATE, "%s: target net not bound", fn);
  const int nl = (int)net->L.size();
  if (q_tensor < 1 || q_tensor > nl || (int)target->L.size() != nl) return fail(XTB_ERR_ARG, "%s: bad head tensor", fn);
  if (n_sample > target->max_batch) return fail(XTB_ERR_ARG, "%s: batch exceeds the target net's max_batch", fn);
  return XTB_OK;
}
static int dqn_train_launch(xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                            const int32_t* idx, const int32_t* action, const float* reward, const uint8_t* done,
                            const float* disc, int n_sample, float gamma, float huber_delta, int q_tensor, float* qn_t,
                            float* qn_o, const float* wt, float* td_abs, float* loss_out, void* st) {
  const int adim = net->tsize[q_tensor];
  const size_t qbytes = (size_t)n_sample * adim * sizeof(float);
  int rc = net_forward_impl(target, nullptr, next_obs, idx, n_sample, st, 0u, 1u << q_tensor);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(qn_t, xtb_net_tensor(target, q_tensor), qbytes, cudaMemcpyDeviceToDevice, S(st)));
  if (qn_o) {
    rc = net_forward_impl(net, nullptr, next_obs, idx, n_sample, st, 0u, 1u << q_tensor);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(qn_o, xtb_net_tensor(net, q_tensor), qbytes, cudaMemcpyDeviceToDevice, S(st)));
  }
  const float inv_count = dp_inv_world() / ((float)n_sample * adim);
  if (dueling_fusable(net, q_tensor)) {
    rc = dueling_td_fused(net, obs, idx, action, reward, done, disc, n_sample, gamma, huber_delta, q_tensor, qn_t, qn_o,
                          inv_count, wt, td_abs, loss_out, S(st));
    if (rc) return rc;
  } else {
    rc = net_forward_impl(net, nullptr, obs, idx, n_sample, st, 0u, 1u << q_tensor);
    if (rc) return rc;
    rc = dqn_td_loss(xtb_net_tensor(net, q_tensor), qn_t, qn_o, idx, action, reward, done, disc, n_sample, adim, gamma,
                     huber_delta, inv_count, wt, xtb_net_tensor_grad(net, q_tensor), nullptr, td_abs, loss_out, st);
    if (rc) return rc;
    const int32_t heads[1] = {q_tensor};
    BackwardOpts o(heads, 1); o.all_reduce = true;
    rc = net_backward_impl(net, obs, idx, n_sample, st, o);
    if (rc) return rc;
  }
  return xtb_adam_step_net(opt, net, 1.f, st);
}
extern "C" int xtb_dqn_train(xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                             const int32_t* idx, const int32_t* action, const float* reward, const uint8_t* done,
                             const float* disc, int n_sample, float gamma, float huber_delta, int q_tensor, float* qn_t,
                             float* qn_o, float* loss_out, int use_graph, void* stream) {
  const bool missing = !net || !target || !opt || !obs || !next_obs || !action || !reward || !done || !qn_t || !loss_out;
  if (int rc = dqn_check("xtb_dqn_train", missing, net, target, opt, n_sample, q_tensor)) return rc;
  if (int rc = heads_kernel_attrs()) return rc;
  return run_graph(capture_key(kDqnTrain, {net, target, opt}, obs, next_obs, idx, action, reward, done, disc, qn_t, qn_o, loss_out,
                               n_sample, gamma, huber_delta, q_tensor),
                   use_graph, stream, [&](void* st) -> int {
    return dqn_train_launch(net, target, opt, obs, next_obs, idx, action, reward, done, disc, n_sample, gamma, huber_delta, q_tensor,
                            qn_t, qn_o, nullptr, nullptr, loss_out, st);
  });
}
extern "C" int xtb_dqn_train_weighted(xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                                      const int32_t* idx, const int32_t* action, const float* reward, const uint8_t* done,
                                      const float* disc, int n_sample, float gamma, float huber_delta, int q_tensor, float* qn_t,
                                      float* qn_o, const float* weights, float* td_abs, float* loss_out, int use_graph, void* stream) {
  const bool missing = !net || !target || !opt || !obs || !next_obs || !action || !reward || !done || !qn_t || !loss_out;
  if (int rc = dqn_check("xtb_dqn_train_weighted", missing, net, target, opt, n_sample, q_tensor)) return rc;
  if (int rc = heads_kernel_attrs()) return rc;
  return run_graph(capture_key(kDqnTrainWeighted, {net, target, opt}, obs, next_obs, idx, action, reward, done, disc, qn_t, qn_o,
                               weights, td_abs, loss_out, n_sample, gamma, huber_delta, q_tensor),
                   use_graph, stream, [&](void* st) -> int {
    return dqn_train_launch(net, target, opt, obs, next_obs, idx, action, reward, done, disc, n_sample, gamma, huber_delta, q_tensor,
                            qn_t, qn_o, weights, td_abs, loss_out, st);
  });
}

// ---- prioritized replay (per.cuh) -------------------------------------------------------------------------------------
struct xtb_per {
  PerTree t{};
  int capacity = 0;
  double alpha = 0, eps = 0;
  uint64_t seed = 0;
  void* buf = nullptr;         // the one device allocation: both trees, the update scratch and the PerState
};

extern "C" int xtb_per_create(int capacity, double alpha, double eps, uint64_t seed, xtb_per** out) {
  if (!out) return fail(XTB_ERR_ARG, "xtb_per_create: null pointer");
  if (capacity < 1 || capacity > (1 << 30)) return fail(XTB_ERR_ARG, "xtb_per_create: capacity %d not in [1, 2^30]", capacity);
  if (!std::isfinite(alpha) || alpha < 0) return fail(XTB_ERR_ARG, "xtb_per_create: alpha %g is not finite and >= 0", alpha);
  if (!std::isfinite(eps) || !(eps > 0)) return fail(XTB_ERR_ARG, "xtb_per_create: eps %g is not finite and > 0", eps);
  auto* p = new xtb_per();
  PerTree& t = p->t;
  t.leaves = 1; t.depth = 0;
  while (t.leaves < capacity) { t.leaves *= 2; t.depth++; }
  const std::vector<double> inf((size_t)2 * t.leaves, INFINITY);
  const std::vector<int32_t> none((size_t)t.leaves, -1);
  PerState st0{};
  st0.max_priority = 1.0;
  if (int rc = carve_scratch("xtb_per_create", &p->buf, {{&t.sum, 2LL * t.leaves}, {&t.mn, 2LL * t.leaves, inf.data()},
                                                        {&t.last, (long long)t.leaves, none.data()}, {&t.st, 1, &st0}})) {
    delete p;
    return rc;
  }
  p->capacity = capacity; p->alpha = alpha; p->eps = eps; p->seed = seed;
  *out = p;
  return XTB_OK;
}

extern "C" void xtb_per_destroy(xtb_per* p) {
  if (!p) return;
  drop_graphs_of(p);
  cudaDeviceSynchronize();
  cudaFree(p->buf);
  delete p;
}

static int per_check(const char* fn, const xtb_per* p, bool missing) {
  if (!p || missing) return fail(XTB_ERR_ARG, "%s: null pointer", fn);
  if (g_comm) return fail(XTB_ERR_STATE, "%s: data-parallel training (communicator) is not supported", fn);
  return XTB_OK;
}
static int per_sample_launch(xtb_per* p, int batch, double beta, const double* uniforms, int32_t* idx, float* w, void* stream) {
  XLAUNCH(per_sample_kernel, 1, std::min(kPerThreads, (batch + 31) / 32 * 32), 0, S(stream), p->t, batch, beta, uniforms, p->seed,
          idx, w);
  LAUNCH_CHECK();
  return XTB_OK;
}
static int per_update_launch(xtb_per* p, const int32_t* idx, const float* td_abs, int n, void* stream) {
  XLAUNCH(per_update_kernel, 1, std::min(kPerThreads, (n + 31) / 32 * 32), 0, S(stream), p->t, idx, td_abs, n, p->alpha, p->eps);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_per_add(xtb_per* p, int first_slot, int n, void* stream) {
  if (int rc = per_check("xtb_per_add", p, false)) return rc;
  if (first_slot < 0 || n < 1 || (long long)first_slot + n > p->capacity)
    return fail(XTB_ERR_ARG, "xtb_per_add: slots [%d, %d + %d) not inside [0, %d)", first_slot, first_slot, n, p->capacity);
  XLAUNCH(per_insert_kernel, 1, kPerThreads, 0, S(stream), p->t, first_slot, n, p->alpha);
  LAUNCH_CHECK();
  return XTB_OK;
}

extern "C" int xtb_per_sample(xtb_per* p, int batch, double beta, const double* uniforms, int32_t* idx, float* w, void* stream) {
  if (int rc = per_check("xtb_per_sample", p, !idx || !w)) return rc;
  if (batch < 1) return fail(XTB_ERR_ARG, "xtb_per_sample: batch %d is not positive", batch);
  if (!std::isfinite(beta) || !(beta > 0)) return fail(XTB_ERR_ARG, "xtb_per_sample: beta %g is not finite and > 0", beta);
  return per_sample_launch(p, batch, beta, uniforms, idx, w, stream);
}

extern "C" int xtb_per_update(xtb_per* p, const int32_t* idx, const float* td_abs, int n, void* stream) {
  if (int rc = per_check("xtb_per_update", p, !idx || !td_abs)) return rc;
  if (n < 1) return fail(XTB_ERR_ARG, "xtb_per_update: batch %d is not positive", n);
  return per_update_launch(p, idx, td_abs, n, stream);
}

extern "C" int xtb_per_state(const xtb_per* p, int* leaves, int* count, double* max_priority, int* status,
                             unsigned long long* offset, double* sum_host, double* min_host) {
  if (!p) return fail(XTB_ERR_ARG, "xtb_per_state: null pointer");
  CUDA_TRY(cudaDeviceSynchronize());
  PerState st;
  CUDA_TRY(cudaMemcpy(&st, p->t.st, sizeof st, cudaMemcpyDeviceToHost));
  if (sum_host) CUDA_TRY(cudaMemcpy(sum_host, p->t.sum, sizeof(double) * 2 * p->t.leaves, cudaMemcpyDeviceToHost));
  if (min_host) CUDA_TRY(cudaMemcpy(min_host, p->t.mn, sizeof(double) * 2 * p->t.leaves, cudaMemcpyDeviceToHost));
  if (leaves) *leaves = p->t.leaves;
  if (count) *count = st.count;
  if (max_priority) *max_priority = st.max_priority;
  if (status) *status = st.status;
  if (offset) *offset = st.offset;
  return XTB_OK;
}

extern "C" int xtb_dqn_per_train(xtb_per* p, xtb_net* net, xtb_net* target, xtb_adam* opt, const void* obs, const void* next_obs,
                                 const int32_t* action, const float* reward, const uint8_t* done, const float* disc, int n_sample,
                                 float gamma, float huber_delta, double beta, int q_tensor, float* qn_t, float* qn_o, int32_t* idx,
                                 float* w, float* td_abs, float* loss_out, int32_t* status_out, int use_graph, void* stream) {
  const char* fn = "xtb_dqn_per_train";
  const bool missing = !net || !target || !opt || !obs || !next_obs || !action || !reward || !done || !qn_t || !loss_out || !idx ||
                       !w || !td_abs || !status_out;
  if (int rc = per_check(fn, p, missing)) return rc;
  if (int rc = dqn_check(fn, missing, net, target, opt, n_sample, q_tensor)) return rc;
  if (!std::isfinite(beta) || !(beta > 0)) return fail(XTB_ERR_ARG, "%s: beta %g is not finite and > 0", fn, beta);
  if (int rc = heads_kernel_attrs()) return rc;
  return run_graph(capture_key(kDqnPerTrain, {net, target, opt, p}, obs, next_obs, action, reward, done, disc, n_sample, gamma,
                               huber_delta, beta, q_tensor, qn_t, qn_o, idx, w, td_abs, loss_out, status_out),
                   use_graph, stream, [&](void* st) -> int {
    int rc = per_sample_launch(p, n_sample, beta, nullptr, idx, w, st);
    if (rc) return rc;
    rc = dqn_train_launch(net, target, opt, obs, next_obs, idx, action, reward, done, disc, n_sample, gamma, huber_delta, q_tensor,
                          qn_t, qn_o, w, td_abs, loss_out, st);
    if (rc) return rc;
    rc = per_update_launch(p, idx, td_abs, n_sample, st);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(status_out, &p->t.st->status, sizeof(int32_t), cudaMemcpyDeviceToDevice, S(st)));
    return XTB_OK;
  });
}

// ------------------------------------------------------------------------------------------
// rollout inference: T batched policy evaluations over the E stacked observations
// ------------------------------------------------------------------------------------------
// T policy evaluations of the action distribution DIST, infer_chunk_steps(max_batch, E) steps per forward (the last
// chunk ragged): per chunk the forward of the layers below the heads and infer_heads_kernel (both heads and the draw)
// within the fused-inference limits, otherwise every layer and then the sampling kernel; the draws are the same either
// way.  The steps are independent (fixed weights, draws keyed on (env, step)), and every kernel of a chunk computes a
// row as it would in a one-step forward: the dense split-K is chosen for E rows, whatever the chunk holds.  So the
// results do not depend on the chunking.  step_idx NULL: step t reads observation rows t*E .. (t+1)*E - 1.
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
  const int c = infer_chunk_steps(net->max_batch, E);
  int n = 0;   // steps in the chunk
  for (int t0 = 0; t0 < T; t0 += c) {
    n = std::min(c, T - t0);
    const int rows = n * E;
    const long long r0 = (long long)t0 * E;
    const void* obs_t = step_idx ? obs : (const void*)((const char*)obs + (size_t)r0 * row_bytes);
    int rc = net_forward_impl(net, nullptr, obs_t, step_idx ? step_idx + r0 : nullptr, rows, stream, skip, want, E);
    if (rc) return rc;
    typename DIST::Action* a_t = action + r0 * DIST::action_width(adim);
    float* lp_t = logp + r0; float* v_o = value + r0;
    if (fuse) {
      XLAUNCH(heads_pick(kInferHeadsKernels<DIST>, lpi.K, adim)->kern, std::max(1, std::min(kSMs, (rows + 7) / 8)), 256, 0,
              S(stream), (const float*)out_f32(net, lpi.d.src), (const float*)out_f32(net, lv.d.src), net->params + lpi.w_off,
              net->params + lpi.b_off, net->params + lv.w_off, net->params + lv.b_off, log_std, rows, E, lpi.K, adim, seed,
              offset_dev, t0, a_t, lp_t, v_o, pi_out);
    } else {
      XLAUNCH(sample_kernel<DIST>, (rows + 127) / 128, 128, 0, S(stream), pi_out, log_std, rows, E, adim, (const float*)nullptr,
              seed, (uint64_t)0, offset_dev, t0, a_t, lp_t, v_in, v_o);
    }
    LAUNCH_CHECK();
  }
  // the pi head of the last step goes to rows [0, E) of its tensor, where a one-step call leaves it
  if (n > 1)
    CUDA_TRY(cudaMemcpyAsync(pi_out, pi_out + (size_t)(n - 1) * E * adim, sizeof(float) * (size_t)E * adim,
                             cudaMemcpyDeviceToDevice, S(stream)));
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
