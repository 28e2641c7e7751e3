"""Algorithm/Model plugin parity: the reference-facing API (prepare_data / train / predict /
get_weights / save / restore) driven like TrainWorker does (xt/framework/learner.py:298-380),
compared with the oracle learners step for step."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import xt_oracle as orc  # noqa: E402

REL = 1e-3


def rel_err(a, b, floor=1e-6):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(float(np.max(np.abs(b))), floor))


def l2_rel(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-12))


def ppo_cnn_info(batch=24, iters=2):
    return {"actor": {"model_name": "PpoCnn", "state_dim": [84, 84, 4], "action_dim": 4, "input_dtype": "uint8",
                      "model_config": {"BATCH_SIZE": batch, "CRITIC_LOSS_COEF": 1.0, "ENTROPY_LOSS": 0.003,
                                       "LOSS_CLIPPING": 0.1, "LR": 0.00025, "MAX_GRAD_NORM": 5.0, "NUM_SGD_ITER": iters,
                                       "SUMMARY": False, "VF_SHARE_LAYERS": True, "activation": "relu",
                                       "hidden_sizes": [256], "action_type": "Categorical", "init_seed": 7}}}


def alg_cfg(**kw):
    cfg = {"instance_num": 4, "agent_num": 1}
    cfg.update(kw)
    return cfg


def make_trajs(E, T, seed, state_dim=(84, 84, 4), A=4, dtype=np.uint8):
    ro = orc.synth_ppo_rollout(seed, E, T, state_dim=state_dim, action_dim=A, dtype=dtype)
    trajs = []
    for e in range(E):
        sl = slice(e * T, (e + 1) * T)
        adv, ov, tv = orc.gae(ro["value"][e], ro["reward"][sl], ro["done"][sl])
        trajs.append(dict(cur_state=ro["obs"][sl], action=ro["action"][sl], logp=ro["logp"][sl],
                          adv=adv, old_value=ov, target_value=tv, value=ro["value"][e],
                          reward=ro["reward"][sl], done=ro["done"][sl]))
    return trajs


@pytest.mark.parametrize("raw", [False, True, "mixed"])
def test_ppo_cnn_train_matches_oracle(raw):
    """a8-a11 end to end: E trajectories -> prepare_data xE -> train(): per-step loss trace and final
    weights vs the oracle PpoLearner under the same np.random shuffle stream (ragged last minibatch).  "mixed" sends
    every second trajectory raw, so device GAE runs per trajectory and its buffers grow past rows they never held."""
    import xingtian_b200 as xb
    E, T = 4, 16
    info = ppo_cnn_info(batch=24, iters=2)
    alg = xb.alg_builder("PPO", info, alg_cfg())
    assert alg.async_flag is False and alg.prepare_data_times == 4 and alg.alg_name == "ppo"
    w0 = alg.get_weights()
    assert sum(v.size for v in w0.values()) == 847493
    arch = orc.ppo_cnn_arch()
    assert list(w0.keys()) == list(orc.param_shapes(arch).keys())
    ref = orc.PpoLearner(arch, w0, lr=0.00025, batch_size=24, critic_coef=1.0, ent_coef=0.003, clip_ratio=0.1,
                         max_grad_norm=5.0, num_sgd_iter=2, vf_clip=5.0)
    trajs = make_trajs(E, T, seed=3)
    for i, tr in enumerate(trajs):
        if raw is True or (raw == "mixed" and i % 2):   # learner-side GAE on the device
            alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "value", "reward", "done")})
        else:     # reference message format (host GAE)
            alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
    np.random.seed(123)
    loss = alg.train()
    np.random.seed(123)
    cat = lambda k: np.concatenate([t[k] for t in trajs])
    ro = alg.actor.rollout
    for key, ref_key in (("adv", "adv"), ("old_v", "old_value"), ("target_v", "target_value")):
        assert rel_err(getattr(ro, key)[:E * T].cpu().numpy(), cat(ref_key).reshape(-1)) < 1e-4, key
    ref_loss, ref_trace = ref.train([cat("cur_state")], [cat("action"), cat("logp"), cat("adv").astype(np.float32),
                                                          cat("old_value"), cat("target_value").astype(np.float32)])
    trace = alg.actor.last_losses
    assert len(trace) == len(ref_trace) == 2 * 3
    assert rel_err(trace, ref_trace) < 5e-3, (trace, ref_trace)
    assert abs(loss - ref_loss) < 5e-3 * max(1.0, abs(ref_loss))
    w1, r1 = alg.get_weights(), ref.weights()
    upd = np.concatenate([(w1[k] - w0[k]).ravel() for k in w0])
    rupd = np.concatenate([(r1[k] - w0[k]).ravel() for k in w0])
    # Six Adam steps: m/sqrt(v) turns ulp-level differences of near-zero gradients (dead ReLU units) into +-lr steps,
    # so the multi-step update is compared by direction and in L2; the single-step test below carries the tight bound.
    cos = float(np.dot(upd, rupd) / (np.linalg.norm(upd) * np.linalg.norm(rupd)))
    assert cos > 0.995 and l2_rel(upd, rupd) < 1e-1, (cos, l2_rel(upd, rupd))
    # second iteration keeps working (buffers were reset)
    for tr in trajs:
        alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
    assert np.isfinite(alg.train())


def test_ppo_single_sgd_step_weights():
    """One SGD step (no shuffle ambiguity): gradient norm and weight update vs oracle."""
    import xingtian_b200 as xb
    info = ppo_cnn_info(batch=64, iters=1)
    alg = xb.alg_builder("PPO", info, alg_cfg())
    w0 = alg.get_weights()
    ref = orc.PpoLearner(orc.ppo_cnn_arch(), w0, lr=0.00025, batch_size=64, ent_coef=0.003, clip_ratio=0.1, num_sgd_iter=1)
    trajs = make_trajs(4, 16, seed=5)
    for tr in trajs:
        alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
    np.random.seed(1); loss = alg.train()
    np.random.seed(1)
    cat = lambda k: np.concatenate([t[k] for t in trajs])
    ref_loss, _ = ref.train([cat("cur_state")], [cat("action"), cat("logp"), cat("adv").astype(np.float32), cat("old_value"), cat("target_value").astype(np.float32)])
    assert abs(loss - ref_loss) < REL * max(1.0, abs(ref_loss))
    assert abs(alg.actor.opt.grad_norm() - ref.last_grad_norm) < REL * ref.last_grad_norm
    g = alg.actor.net.get_weights(alg.actor.net.grads)
    # gradients of the same minibatch
    np.random.seed(1); inds = np.arange(64); np.random.shuffle(inds)
    ref2 = orc.PpoLearner(orc.ppo_cnn_arch(), w0, batch_size=64, ent_coef=0.003, clip_ratio=0.1)
    _, grads = ref2.loss_and_grads(cat("cur_state")[inds], cat("action")[inds], cat("logp")[inds], cat("adv").astype(np.float32)[inds],
                                   cat("old_value")[inds], cat("target_value").astype(np.float32)[inds])
    for k, gr in zip(w0.keys(), grads):
        assert rel_err(g[k], gr.numpy()) < REL, k


def test_ppo_predict_contract_and_noise():
    import xingtian_b200 as xb
    alg = xb.alg_builder("PPO", ppo_cnn_info(), alg_cfg())
    rng = np.random.default_rng(0)
    state = rng.integers(0, 256, (84, 84, 4), dtype=np.uint8)
    a, lp, v = alg.predict(state)          # batch-1 reshape of xt/algorithm/ppo/ppo.py:87-95
    assert a.shape == (1,) and a.dtype == np.int32 and lp.shape == (1, 1) and v.shape == (1, 1)
    a2, _, _ = alg.predict([state, state])
    assert a2.shape == (2,)
    obs = rng.integers(0, 256, (33, 84, 84, 4), dtype=np.uint8)
    u = rng.random((33, 4)).astype(np.float32) * 0.998 + 0.001
    act, logp, val = alg.actor.predict(obs, uniforms=u)
    ract, rlogp, rval = orc.ppo_predict(orc.ppo_cnn_arch(), alg.get_weights(), obs, u)
    assert rel_err(val, rval) < REL and rel_err(logp, rlogp) < REL
    assert (act == ract).mean() >= 0.97      # mismatches only on fp near-ties
    with torch.no_grad():
        logits = orc.forward(orc.ppo_cnn_arch(), alg.get_weights(), obs)[0].numpy()
    s = np.sort(logits - np.log(-np.log(u)), 1)
    assert not ((act != ract) & (s[:, -1] - s[:, -2] > 1e-3)).any()


def test_cartpole_ppo_mlp_plumbing(tmp_path):
    """BASELINE config 1: examples/cartpole_ppo.yaml shapes (PpoMlp tanh [64,64], separate towers,
    variable-length episodes, save/restore)."""
    import xingtian_b200 as xb
    info = {"actor": {"model_name": "PpoMlp", "state_dim": [4], "action_dim": 2, "input_dtype": "float32",
                      "model_config": {"BATCH_SIZE": 200, "CRITIC_LOSS_COEF": 1.0, "ENTROPY_LOSS": 0.01, "LR": 0.0003,
                                       "LOSS_CLIPPING": 0.2, "MAX_GRAD_NORM": 5.0, "NUM_SGD_ITER": 8, "SUMMARY": False,
                                       "VF_SHARE_LAYERS": False, "activation": "tanh", "hidden_sizes": [64, 64],
                                       "action_type": "Categorical", "init_seed": 1}}}
    alg = xb.alg_builder("PPO", info, alg_cfg(instance_num=10, save_model=True, save_interval=100))
    w0 = alg.get_weights()
    arch = orc.ppo_mlp_arch()
    assert list(w0.keys()) == list(orc.param_shapes(arch).keys())
    ref = orc.PpoLearner(arch, w0, lr=0.0003, batch_size=200, ent_coef=0.01, clip_ratio=0.2, num_sgd_iter=8)
    rng = np.random.default_rng(4)
    trajs = []
    for e in range(10):
        T = int(rng.integers(9, 200))
        tr = make_trajs(1, T, seed=100 + e, state_dim=(4,), A=2, dtype=np.float32)[0]
        tr["done"][-1] = True
        trajs.append(tr)
        alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "value", "reward", "done")})
    np.random.seed(9); loss = alg.train()
    np.random.seed(9)
    cat = lambda k: np.concatenate([t[k] for t in trajs])
    adv = np.concatenate([orc.gae(t["value"], t["reward"], t["done"])[0] for t in trajs]).astype(np.float32)
    tv = np.concatenate([orc.gae(t["value"], t["reward"], t["done"])[2] for t in trajs]).astype(np.float32)
    ov = np.concatenate([t["value"][:-1] for t in trajs])
    ref_loss, ref_trace = ref.train([cat("cur_state")], [cat("action"), cat("logp"), adv, ov, tv])
    assert rel_err(alg.actor.last_losses, ref_trace) < 5e-3
    assert abs(loss - ref_loss) < 5e-3 * max(1.0, abs(ref_loss))
    # checkpoint cadence + npz format (algorithm.py:80-87,180-194; tf_utils.py:130-144)
    assert alg.if_save(100) and not alg.if_save(101)
    names = alg.save(str(tmp_path), 100)
    assert names == [os.path.join(str(tmp_path), "actor_00100.npz")]
    z = np.load(names[0])
    assert sorted(z.files) == sorted(w0.keys())
    w1 = alg.get_weights()
    alg2 = xb.alg_builder("PPO", info, alg_cfg(instance_num=10))
    alg2.restore(model_name=names[0])
    for k in w1:
        np.testing.assert_array_equal(alg2.get_weights()[k], w1[k])
    alg2.restore(model_weights=w0)
    np.testing.assert_array_equal(alg2.get_weights()["pi_latent/kernel"], w0["pi_latent/kernel"])
    with pytest.raises(KeyError):
        alg2.set_weights({"nope": np.zeros(3)})


def test_impala_opt_train_matches_oracle():
    """a12-a15: IMPALAOpt prepare_data/train with BATCH_SIZE slicing vs oracle ImpalaLearner."""
    import xingtian_b200 as xb
    S, k = 16, 6
    info = {"actor": {"model_name": "ImpalaCnnOpt", "state_dim": [84, 84, 4], "input_dtype": "uint8", "state_mean": 0.0,
                      "state_std": 255.0, "action_dim": 4,
                      "model_config": {"LR": 0.0005, "sample_batch_step": S, "grad_norm_clip": 40.0, "init_seed": 3}}}
    alg = xb.alg_builder("IMPALAOpt", info, alg_cfg(instance_num=2, prepare_times_per_train=1, train_per_checkpoint=1, BATCH_SIZE=4 * S))
    w0 = alg.get_weights()
    arch = orc.impala_cnn_arch()
    assert list(w0.keys()) == list(orc.param_shapes(arch).keys()) and sum(v.size for v in w0.values()) == 1005109
    ref = orc.ImpalaLearner(arch, w0, lr=0.0005, grad_norm_clip=40.0, sample_batch_step=S)
    ro = orc.synth_ppo_rollout(8, k, S)
    ro["reward"] = ro["reward"] * 3.0     # exercise the [-1,1] clip
    for i in range(0, k, 2):    # messages of vector_env_size=2 trajectories
        sl = slice(i * S, (i + 2) * S)
        alg.prepare_data(dict(cur_state=ro["obs"][sl], logit=ro["logits"][sl], action=ro["action"][sl], reward=ro["reward"][sl], done=ro["done"][sl]))
    loss = alg.train()
    ref_losses = []
    for s in range(0, k * S, 4 * S):
        sl = slice(s, min(k * S, s + 4 * S))
        ref_losses.append(ref.train(ro["obs"][sl], [ro["logits"][sl], ro["action"][sl], ro["done"][sl], ro["reward"][sl]]))
    assert abs(loss - np.mean(ref_losses)) < 5e-3 * max(1.0, abs(np.mean(ref_losses)))
    w1, r1 = alg.get_weights(), ref.weights()
    upd = np.concatenate([(w1[k_] - w0[k_]).ravel() for k_ in w0]); rupd = np.concatenate([(r1[k_] - w0[k_]).ravel() for k_ in w0])
    assert l2_rel(upd, rupd) < 5e-2
    logits, base, act = alg.predict(ro["obs"][:5])
    rl, rb = orc.forward(arch, w1, ro["obs"][:5])
    assert logits.shape == (5, 4) and base.shape == (5,) and act.shape == (5,) and act.dtype == np.int32
    assert rel_err(logits, rl.numpy()) < REL and rel_err(base, rb.numpy()[:, 0]) < REL
    assert ((act >= 0) & (act < 4)).all()
    # graph-captured rollout inference (T steps, one graph) = the per-step host predict on the same frames
    m = alg.actor
    E, T = 3, 4
    obs_d = torch.from_numpy(ro["obs"][:E * T]).cuda()
    step_idx = torch.arange(E * T, dtype=torch.int32, device="cuda").reshape(T, E).contiguous()      # time-major rows
    a_t = torch.empty(T, E, dtype=torch.int32, device="cuda"); lp_t = torch.empty(T, E, device="cuda"); v_t = torch.empty(T, E, device="cuda")
    m.rollout_infer_device(obs_d, step_idx, E, T, a_t, lp_t, v_t)
    rl2, rb2 = orc.forward(arch, w1, ro["obs"][:E * T])
    assert rel_err(v_t.cpu().numpy().reshape(-1), rb2.numpy()[:, 0]) < REL
    lsm = torch.log_softmax(rl2, 1).numpy()
    picked = lsm[np.arange(E * T), a_t.cpu().numpy().reshape(-1)]
    assert np.abs(lp_t.cpu().numpy().reshape(-1) - picked).max() < 2e-3
    assert alg.dist_model_policy.get_dist_info(-1) == {"broker_id": -1, "explorer_id": -1}


@pytest.mark.parametrize("variant", ["rmsprop", "lr_schedule"])
def test_impala_optimiser_options_match_oracle(variant):
    """a14: ImpalaCnnOpt with opt_type rmsprop (centred, decay .99, eps .1) and with the Adam linear_cosine_decay schedule:
    three train steps through the plugin vs the oracle learner with the same option (impala_cnn_opt.py:198-217,234-249)."""
    import xingtian_b200 as xb
    S, k = 16, 4
    cfg = {"LR": 0.0005, "sample_batch_step": S, "grad_norm_clip": 40.0, "init_seed": 5}
    sched = [[0, 0.001], [20000, 0.000002]]
    if variant == "rmsprop":
        cfg["opt_type"] = "rmsprop"
    else:
        cfg["lr_schedule"] = sched
    info = {"actor": {"model_name": "ImpalaCnnOpt", "state_dim": [84, 84, 4], "input_dtype": "uint8", "state_mean": 0.0,
                      "state_std": 255.0, "action_dim": 4, "model_config": cfg}}
    alg = xb.alg_builder("IMPALAOpt", info, alg_cfg(instance_num=k, prepare_times_per_train=1, BATCH_SIZE=k * S))
    w0 = alg.get_weights()
    arch = orc.impala_cnn_arch()
    ref = orc.ImpalaLearner(arch, w0, lr=0.0005, grad_norm_clip=40.0, sample_batch_step=S,
                            opt_type="rmsprop" if variant == "rmsprop" else "adam", lr_schedule=sched if variant == "lr_schedule" else None)
    if variant == "lr_schedule":
        alg.actor._global_step = 14000; ref.global_step = 14000    # late in the schedule: lr = 0.2 x LR, so a schedule that is
                                                                     # ignored fails the update comparison below
    losses, ref_losses = [], []
    for it in range(3):
        ro = orc.synth_ppo_rollout(20 + it, k, S)
        alg.prepare_data(dict(cur_state=ro["obs"], logit=ro["logits"], action=ro["action"], reward=ro["reward"], done=ro["done"]))
        losses.append(alg.train())
        ref_losses.append(ref.train(ro["obs"], [ro["logits"], ro["action"], ro["done"], ro["reward"]]))
    assert rel_err(losses, ref_losses) < 5e-3, (losses, ref_losses)
    w1, r1 = alg.get_weights(), ref.weights()
    upd = np.concatenate([(w1[n] - w0[n]).ravel() for n in w0]); rupd = np.concatenate([(r1[n] - w0[n]).ravel() for n in w0])
    # RMSProp(eps 0.1) is smooth in the gradient; three Adam steps carry the m/sqrt(v) sign noise of near-zero gradients
    assert l2_rel(upd, rupd) < (5e-2 if variant == "rmsprop" else 1e-1), l2_rel(upd, rupd)
    if variant == "lr_schedule":
        assert abs(alg.actor.scheduled_lr(14000) - orc.linear_cosine_decay(0.001, 14000, 20000.0, beta=0.000002 / 20000.0)) < 1e-12


def test_dqn_train_matches_oracle():
    """a16-a19: replay -> TD target -> mse -> Adam(clipnorm) -> hard target sync."""
    import random
    import xingtian_b200 as xb
    from xingtian_b200.algorithm import dqn as dqn_mod
    info = {"actor": {"model_name": "DqnCnn", "state_dim": [84, 84, 4], "action_dim": 4, "model_config": {"LR": 0.00015, "init_seed": 5}}}
    alg = xb.alg_builder("DQN", info, alg_cfg(instance_num=2, prepare_times_per_train=4, learning_starts=40, BUFFER_SIZE=64,
                                              BATCH_SIZE=32, TARGET_UPDATE_FREQ=2))
    assert dqn_mod.BUFFER_SIZE == 64 and dqn_mod.TARGET_UPDATE_FREQ == 2
    w0 = alg.get_weights()
    arch = orc.dqn_cnn_arch()
    assert sum(v.size for v in w0.values()) == 882084
    ref = orc.DqnLearner(arch, w0, lr=0.00015, clipnorm=10.0, target_update_freq=2)
    rng = np.random.default_rng(0)
    n = 48
    s = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8); s2 = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)
    a = rng.integers(0, 4, n); r = np.sign(rng.standard_normal(n)); d = rng.random(n) < 0.1
    assert not alg.train_ready(0)
    for i in range(n):   # one transition per message (cartpole_dqn.py:80-83)
        alg.prepare_data(dict(cur_state=[s[i]], action=[a[i]], reward=[r[i]], next_state=[s2[i]], done=[d[i]]))
    assert alg.train_ready(0) and alg.buff.size() == 48
    for step in range(3):
        random.seed(step)
        loss = alg.train()
        random.seed(step)
        picks = random.sample(range(n), 32)
        ref_loss = ref.train(s[picks], a[picks], r[picks], s2[picks], d[picks])
        assert abs(loss - ref_loss) < 5e-3 * max(1.0, abs(ref_loss)), step
    w1, r1 = alg.get_weights(), ref.weights()
    upd = np.concatenate([(w1[k] - w0[k]).ravel() for k in w0]); rupd = np.concatenate([(r1[k] - w0[k]).ravel() for k in w0])
    assert l2_rel(upd, rupd) < 5e-2
    # Algorithm.predict: greedy action of one state (algorithm.py:124-135)
    act = alg.predict(s[0])
    assert act == int(np.argmax(ref.predict(s[:1])[0]))
    # keras-style train(state, y) entry point
    y = ref.predict(s[:8]); y[:, 1] += 1.0
    l1 = alg.actor.train(s[:8], y)
    assert abs(l1 - 0.25) < 0.05


def test_impala_c3_config_size_step_matches_oracle():
    """C3 shapes through the plugin: E=64 envs deliver T=128-step trajectories, BATCH_SIZE=512 = 4 trajectories per SGD
    step (T' = 127 after drop_last inside the V-trace); two captured steps vs the oracle learner."""
    import xingtian_b200 as xb
    S, k = 128, 8
    info = {"actor": {"model_name": "ImpalaCnnOpt", "state_dim": [84, 84, 4], "input_dtype": "uint8", "state_mean": 0.0,
                      "state_std": 255.0, "action_dim": 4, "max_batch": 512,
                      "model_config": {"LR": 0.0005, "sample_batch_step": S, "grad_norm_clip": 40.0, "init_seed": 3}}}
    alg = xb.alg_builder("IMPALAOpt", info, alg_cfg(instance_num=64, prepare_times_per_train=1, train_per_checkpoint=1, BATCH_SIZE=512))
    w0 = alg.get_weights()
    arch = orc.impala_cnn_arch()
    ref = orc.ImpalaLearner(arch, w0, lr=0.0005, grad_norm_clip=40.0, sample_batch_step=S)
    ro = orc.synth_ppo_rollout(21, k, S)
    for i in range(k):
        sl = slice(i * S, (i + 1) * S)
        alg.prepare_data(dict(cur_state=ro["obs"][sl], logit=ro["logits"][sl], action=ro["action"][sl], reward=ro["reward"][sl], done=ro["done"][sl]))
    loss = alg.train()
    ref_losses = []
    for s0 in range(0, k * S, 512):
        sl = slice(s0, s0 + 512)
        ref_losses.append(ref.train(ro["obs"][sl], [ro["logits"][sl], ro["action"][sl], ro["done"][sl], ro["reward"][sl]]))
    print("impala C3 loss", loss, np.mean(ref_losses))
    assert abs(loss - np.mean(ref_losses)) < 5e-3 * max(1.0, abs(np.mean(ref_losses)))
    w1, r1 = alg.get_weights(), ref.weights()
    upd = np.concatenate([(w1[k_] - w0[k_]).ravel() for k_ in w0]); rupd = np.concatenate([(r1[k_] - w0[k_]).ravel() for k_ in w0])
    print("impala C3 update l2 rel", l2_rel(upd, rupd))
    assert l2_rel(upd, rupd) < 5e-2


def test_dqn_c4_config_size_step_matches_oracle():
    """C4 shapes through the plugin: batch 512 out of a device replay ring, two captured steps vs the oracle learner."""
    import random
    import xingtian_b200 as xb
    info = {"actor": {"model_name": "DqnCnn", "state_dim": [84, 84, 4], "action_dim": 4, "max_batch": 512,
                      "model_config": {"LR": 0.00015, "init_seed": 5}}}
    alg = xb.alg_builder("DQN", info, alg_cfg(instance_num=2, prepare_times_per_train=4, learning_starts=40, BUFFER_SIZE=1024,
                                              BATCH_SIZE=512, TARGET_UPDATE_FREQ=1000))
    w0 = alg.get_weights()
    arch = orc.dqn_cnn_arch()
    ref = orc.DqnLearner(arch, w0, lr=0.00015, clipnorm=10.0, target_update_freq=1000)
    rng = np.random.default_rng(0)
    n = 768
    s = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8); s2 = rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)
    a = rng.integers(0, 4, n); r = np.sign(rng.standard_normal(n)); d = rng.random(n) < 0.1
    alg.prepare_data(dict(cur_state=s, action=a, reward=r, next_state=s2, done=d))
    for step in range(2):
        random.seed(step)
        loss = alg.train()
        random.seed(step)
        picks = random.sample(range(n), 512)
        ref_loss = ref.train(s[picks], a[picks], r[picks], s2[picks], d[picks])
        print("dqn C4 step", step, loss, ref_loss)
        assert abs(loss - ref_loss) < 5e-3 * max(1.0, abs(ref_loss)), step
    w1, r1 = alg.get_weights(), ref.weights()
    upd = np.concatenate([(w1[k] - w0[k]).ravel() for k in w0]); rupd = np.concatenate([(r1[k] - w0[k]).ravel() for k in w0])
    print("dqn C4 update l2 rel", l2_rel(upd, rupd))
    assert l2_rel(upd, rupd) < 5e-2


@pytest.mark.parametrize("E,T,n", [(1, 64, 3), (5, 33, 1), (3, 40, 5)])
def test_nstep_returns_kernel(E, T, n):
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    rng = np.random.default_rng(E * 100 + T + n)
    rew = rng.normal(0, 1, (E, T)).astype(np.float32); done = rng.random((E, T)) < 0.1
    rd, dd = torch.from_numpy(rew).cuda(), torch.from_numpy(done.view(np.uint8)).cuda()
    ret = torch.empty(E, T, device="cuda"); disc = torch.empty(E, T, device="cuda")
    last = torch.empty(E, T, dtype=torch.int32, device="cuda"); dn = torch.empty(E, T, dtype=torch.uint8, device="cuda")
    capi.check(capi.lib().xtb_nstep_returns(_ptr(rd), _ptr(dd), E, T, n, 0.99, _ptr(ret), _ptr(disc), _ptr(last), _ptr(dn), stream_ptr()))
    for e in range(E):
        r_ret, r_disc, r_last, r_dn = orc.nstep_returns(rew[e], done[e], n, 0.99)
        assert rel_err(ret[e].cpu().numpy(), r_ret) < 1e-5 and rel_err(disc[e].cpu().numpy(), r_disc, floor=1.0) < 1e-6
        np.testing.assert_array_equal(last[e].cpu().numpy() - e * T, r_last)
        np.testing.assert_array_equal(dn[e].cpu().numpy().astype(bool), r_dn)


def test_dqn_nstep_huber_step_matches_numpy():
    """north_star extension (ns1): N_STEP=3 replay + Huber loss, one SGD step vs a torch-CPU restatement built on the
    oracle's network; the default configuration (1-step, mse) is covered by test_dqn_train_matches_oracle."""
    import random
    import xingtian_b200 as xb
    info = {"actor": {"model_name": "DqnCnn", "state_dim": [84, 84, 4], "action_dim": 4, "model_config": {"LR": 0.00015, "init_seed": 5}}}
    alg = xb.alg_builder("DQN", info, alg_cfg(instance_num=1, prepare_times_per_train=4, learning_starts=8, BUFFER_SIZE=256,
                                              BATCH_SIZE=32, TARGET_UPDATE_FREQ=1000, N_STEP=3, HUBER_DELTA=1.0))
    assert alg.n_step == 3 and alg.huber_delta == 1.0
    w0 = alg.get_weights()
    arch = orc.dqn_cnn_arch()
    rng = np.random.default_rng(1)
    T = 64
    s = rng.integers(0, 256, (T, 84, 84, 4), dtype=np.uint8); s2 = rng.integers(0, 256, (T, 84, 84, 4), dtype=np.uint8)
    a = rng.integers(0, 4, T); r = rng.normal(0, 2, T).astype(np.float32); d = rng.random(T) < 0.1
    alg.prepare_data(dict(cur_state=s, action=a, reward=r, next_state=s2, done=d))
    ret, disc, last, dn = orc.nstep_returns(r, d, 3, 0.99)
    random.seed(0)
    loss = alg.train()
    random.seed(0)
    picks = random.sample(range(T), 32)
    params = {k: torch.from_numpy(v.copy()).requires_grad_(True) for k, v in w0.items()}
    with torch.no_grad():
        tq = orc.forward(arch, {k: torch.from_numpy(v) for k, v in w0.items()}, s2[last[picks]])[0].numpy()
    y = np.where(dn[picks], ret[picks], ret[picks] + disc[picks] * tq.max(1)).astype(np.float32)
    q = orc.forward(arch, params, s[picks])[0]
    qa = q[torch.arange(32), torch.from_numpy(a[picks])]
    diff = qa - torch.from_numpy(y)
    hub = torch.where(diff.abs() <= 1.0, 0.5 * diff * diff, diff.abs() - 0.5)
    ref_loss = hub.sum() / (32 * 4)
    assert abs(loss - float(ref_loss)) < 5e-3 * max(1.0, abs(float(ref_loss))), (loss, float(ref_loss))
    ref_loss.backward()
    ref_p = [p.detach().clone() for p in params.values()]
    opt = orc.TFAdam(ref_p, 0.00015, eps=1e-7)
    grads = []
    for p in params.values():
        g = p.grad; nn = float(g.norm())
        grads.append(g * (10.0 / nn) if nn > 10.0 else g)
    opt.step(grads)
    w1 = alg.get_weights()
    upd = np.concatenate([(w1[k] - w0[k]).ravel() for k in w0])
    rupd = np.concatenate([(rp.numpy() - w0[k]).ravel() for rp, k in zip(ref_p, w0)])
    assert l2_rel(upd, rupd) < 5e-2, l2_rel(upd, rupd)


def test_rollout_infer_graph_matches_per_step_predict():
    """The T-step graph-captured rollout inference equals T separate predict calls under the same Philox
    stream, and replays draw fresh noise (device-side offset counter)."""
    import xingtian_b200 as xb
    alg = xb.alg_builder("PPO", ppo_cnn_info(), alg_cfg())
    m = alg.actor
    E, T = 8, 5
    rng = np.random.default_rng(0)
    obs = torch.from_numpy(rng.integers(0, 256, (E * T, 84, 84, 4), dtype=np.uint8)).cuda()
    step_idx = (torch.arange(E, dtype=torch.int32, device="cuda")[None, :] * T + torch.arange(T, dtype=torch.int32, device="cuda")[:, None]).contiguous()
    act = torch.empty(T, E, dtype=torch.int32, device="cuda"); lp = torch.empty(T, E, device="cuda"); val = torch.empty(T + 1, E, device="cuda")
    m.rollout_infer_device(obs, step_idx, E, T, act, lp, val)
    a1 = act.cpu().numpy().copy()
    arch = orc.ppo_cnn_arch(); w = alg.get_weights()
    for t in range(T):
        rows = (np.arange(E) * T + t)
        u = orc.philox_uniforms(m._sample_seed, t, E, 4)
        ract, rlogp, rval = orc.ppo_predict(arch, w, obs.cpu().numpy()[rows], u)
        assert rel_err(val[t].cpu().numpy(), rval[:, 0]) < REL and rel_err(lp[t].cpu().numpy(), rlogp[:, 0]) < REL
        assert (a1[t] == ract).mean() >= 0.85
    m.rollout_infer_device(obs, step_idx, E, T, act, lp, val)     # graph replay: offset advanced by T
    assert int(m._offset_dev.cpu()[0]) == 2 * T
    u = orc.philox_uniforms(m._sample_seed, T, E, 4)
    ract, _, _ = orc.ppo_predict(arch, w, obs.cpu().numpy()[np.arange(E) * T], u)
    assert (act[0].cpu().numpy() == ract).mean() >= 0.85


def test_cuda_graph_path_is_taken_and_equals_eager():
    """The fused training loop and the rollout inference are replayed as CUDA graphs when the host passes the default
    (NULL) stream -- the library moves them onto its fenced private stream -- and give the eager path's results."""
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    lib = capi.lib()
    outs = []
    for graph in (True, False):
        info = ppo_cnn_info(batch=24, iters=2)
        info["actor"]["model_config"]["use_cuda_graph"] = graph
        alg = xb.alg_builder("PPO", info, alg_cfg())
        r0 = lib.xtb_graph_replay_count()
        losses = []
        for it in range(2):                 # second iteration replays the instantiated graph
            for tr in make_trajs(4, 16, seed=3 + it):
                alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
            np.random.seed(5 + it)
            losses.append(alg.train())
        replays = lib.xtb_graph_replay_count() - r0
        assert replays == (2 if graph else 0), replays
        w = alg.get_weights()
        outs.append((np.array(losses), np.concatenate([v.ravel() for v in w.values()])))
    assert rel_err(outs[0][0], outs[1][0]) < 1e-3
    assert l2_rel(outs[0][1], outs[1][1]) < 1e-3
    # Adam's learning rate lives in device memory: a captured graph must see xtb_adam_set_lr
    alg = xb.alg_builder("PPO", ppo_cnn_info(batch=24, iters=1), alg_cfg())
    w0 = np.concatenate([v.ravel() for v in alg.get_weights().values()])
    steps = []
    for lr in (2.5e-4, 0.0):
        capi.check(lib.xtb_adam_set_lr(alg.actor.opt.handle, lr))
        for tr in make_trajs(4, 16, seed=9):
            alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
        alg.train()
        w1 = np.concatenate([v.ravel() for v in alg.get_weights().values()])
        steps.append(float(np.abs(w1 - w0).max()))
        w0 = w1
    assert steps[0] > 0 and steps[1] == 0.0, steps


def test_fused_heads_equals_unfused():
    """The fused heads+loss kernel and the layer-by-layer path give the same loss trace and weights."""
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    lib = capi.lib()
    outs = []
    try:
        for fuse in (1, 0):
            lib.xtb_set_fuse_heads(fuse)
            alg = xb.alg_builder("PPO", ppo_cnn_info(batch=24, iters=2), alg_cfg())
            for tr in make_trajs(4, 16, seed=3):
                alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
            np.random.seed(5)
            loss = alg.train()
            w = alg.get_weights()
            outs.append((loss, np.array(alg.actor.last_losses), np.concatenate([v.ravel() for v in w.values()])))
    finally:
        lib.xtb_set_fuse_heads(1)
    # The two paths sum in different orders (~1e-7 per step).  Six Adam steps from zero moments amplify that by about
    # an order of magnitude per step (lr*m/sqrt(v) ~ lr*sign(g) for near-zero gradients), so the first steps carry the
    # tight bound and the whole trace / the weights a bound that still catches any real disagreement.
    print("fused vs unfused loss trace:", np.abs(outs[0][1] - outs[1][1]) / np.abs(outs[1][1]))
    assert rel_err(outs[0][1][:3], outs[1][1][:3]) < 1e-5
    assert rel_err(outs[0][1], outs[1][1]) < 2e-3
    assert l2_rel(outs[0][2], outs[1][2]) < 1e-3


def test_rollout_infer_graph_follows_fuse_heads_mode():
    """The fused-heads mode is part of a rollout-inference graph's key: after xtb_set_fuse_heads(0) a graphed call on
    the same buffers launches what an eager layer-by-layer call launches, not the fused graph captured before."""
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    lib = capi.lib()
    m = xb.alg_builder("PPO", ppo_cnn_info(), alg_cfg()).actor
    E, T = 8, 2
    obs = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (E * T, 84, 84, 4), dtype=np.uint8)).cuda()
    act = torch.empty(T, E, dtype=torch.int32, device="cuda"); lp = torch.empty(T, E, device="cuda"); val = torch.empty(T, E, device="cuda")

    def launches(use_graph):
        m.use_graph = use_graph
        n0, r0 = lib.xtb_launch_count(), lib.xtb_graph_replay_count()
        m.rollout_infer_device(obs, None, E, T, act, lp, val)
        torch.cuda.synchronize()
        assert lib.xtb_graph_replay_count() - r0 == int(use_graph)
        return lib.xtb_launch_count() - n0

    try:
        lib.xtb_set_fuse_heads(1)
        fused = launches(True)
        lib.xtb_set_fuse_heads(0)
        graphed = launches(True)
        eager = launches(False)
    finally:
        lib.xtb_set_fuse_heads(1)
    assert fused != eager, (fused, eager)
    assert graphed == eager, (graphed, eager)


def test_dqn_graph_is_keyed_on_scratch_and_discount_buffers():
    """A graphed xtb_dqn_train call that differs from a captured one only in its qn_t or disc buffer uses the new
    buffer: the old scratch keeps what the host wrote into it, and the loss is that of an eager call."""
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    info = {"actor": {"model_name": "DqnCnn", "state_dim": [84, 84, 4], "action_dim": 4, "model_config": {"LR": 0.00015, "init_seed": 5}}}
    alg = xb.alg_builder("DQN", info, alg_cfg(instance_num=1, learning_starts=8, BUFFER_SIZE=64, BATCH_SIZE=32))
    m, tgt = alg.actor, alg.target_actor
    m.opt.set_lr(0.0)        # the weights stay put: every call below sees the same network
    lib = m.net.lib
    n, A = 32, 4
    rng = np.random.default_rng(2)
    obs = torch.from_numpy(rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)).cuda()
    next_obs = torch.from_numpy(rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8)).cuda()
    action = torch.from_numpy(rng.integers(0, A, n).astype(np.int32)).cuda()
    reward = torch.zeros(n, device="cuda"); done = torch.zeros(n, dtype=torch.uint8, device="cuda")
    disc_gamma = torch.full((n,), 0.99, device="cuda"); disc_zero = torch.zeros(n, device="cuda")
    qn_t1 = torch.empty(n, A, device="cuda"); qn_t2 = torch.empty(n, A, device="cuda")
    loss = torch.zeros(1, device="cuda")

    def step(qn_t, disc, use_graph):
        loss.zero_()
        capi.check(lib.xtb_dqn_train(m.net.handle, tgt.net.handle, m.opt.handle, _ptr(obs), _ptr(next_obs), None, _ptr(action),
                                     _ptr(reward), _ptr(done), _ptr(disc), n, 0.99, 0.0, m.net.tid[m.q_name], _ptr(qn_t), None,
                                     _ptr(loss), use_graph, stream_ptr()))
        return float(loss.cpu()[0])

    step(qn_t1, disc_gamma, 1)                       # captured on qn_t1 and disc_gamma
    ref_gamma, ref_zero = step(qn_t2, disc_gamma, 0), step(qn_t2, disc_zero, 0)
    assert abs(ref_gamma - ref_zero) > 0.1 * max(abs(ref_gamma), abs(ref_zero)), (ref_gamma, ref_zero)
    disc_gamma.fill_(12345.0)
    got = step(qn_t1, disc_zero, 1)                  # another disc buffer
    assert abs(got - ref_zero) < 5e-3 * abs(ref_zero), (got, ref_zero)
    qn_t1.fill_(12345.0)
    got = step(qn_t2, disc_zero, 1)                  # another qn_t buffer
    assert bool((qn_t1 == 12345.0).all())
    assert abs(got - ref_zero) < 5e-3 * abs(ref_zero), (got, ref_zero)


def test_rebinding_a_net_drops_its_graphs():
    """xtb_net_bind_stream on a live handle drops the graphs captured with the old buffers: the next graphed training
    call updates the new parameter buffer and leaves the old one alone."""
    import ctypes as C
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    from xingtian_b200.engine import _ptr, stream_ptr
    alg = xb.alg_builder("PPO", ppo_cnn_info(batch=24, iters=1), alg_cfg())
    net = alg.actor.net
    lib = net.lib
    trajs = make_trajs(4, 16, seed=3)

    def train():
        for tr in trajs:
            alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
        np.random.seed(5)
        alg.train()

    r0 = lib.xtb_graph_replay_count()
    train()
    old_p, old_g = net.params, net.grads
    new_p, new_g = old_p.clone(), torch.zeros_like(old_g)
    capi.check(lib.xtb_net_bind_stream(net.handle, _ptr(new_p), _ptr(new_g), C.c_void_p(net._ws_base),
                                       lib.xtb_net_workspace_bytes(net.handle), stream_ptr()))
    net.params, net.grads = new_p, new_g
    old_snap, new_snap = old_p.clone(), new_p.clone()
    train()
    assert lib.xtb_graph_replay_count() - r0 == 2
    assert torch.equal(old_p, old_snap)
    assert not torch.equal(new_p, new_snap)


def test_staged_h2d_copy_is_exact():
    """xtb_copy_h2d_staged (threaded pinned-ring staging of pageable arrays) is a byte-exact copy for empty,
    sub-chunk, chunk-boundary and larger-than-ring sizes, back to back on one stream and across two streams."""
    from xingtian_b200 import capi
    from xingtian_b200.engine import stream_ptr
    lib = capi.lib()
    rng = np.random.default_rng(5)
    chunk, ring = 256 << 10, 48 * (256 << 10)
    sizes = [0, 1, 4097, chunk - 1, chunk, chunk + 1, 3 * chunk + 17, 32 * 28224, ring - 5, ring + chunk + 3, 3 * ring + 11]
    side = torch.cuda.Stream()
    for rep in range(2):
        srcs, dsts = [], []
        for i, n in enumerate(sizes):
            a = rng.integers(0, 256, size=n, dtype=np.uint8)
            d = torch.zeros(max(n, 1) + 64, dtype=torch.uint8, device="cuda")
            with torch.cuda.stream(side if (i & 1) else torch.cuda.current_stream()):
                capi.check(lib.xtb_copy_h2d_staged(d.data_ptr() + 32, a.ctypes.data, n, stream_ptr()))
            srcs.append(a.copy())
            a[:] = 0                      # the source may be reused as soon as the call returns
            dsts.append(d)
        torch.cuda.synchronize()
        for n, a, d in zip(sizes, srcs, dsts):
            h = d.cpu().numpy()
            assert not h[:32].any() and not h[32 + n:].any()
            assert np.array_equal(h[32:32 + n], a)
    assert lib.xtb_copy_h2d_staged(None, srcs[1].ctypes.data, 1, None) == -1


@pytest.mark.parametrize("tc", [1, 0])
def test_ppo_c2_full_iteration_matches_oracle(tc):
    """SURVEY 8(c) golden item 7 at BASELINE config C2 size: E=32 trajectories of T=128 (N=4096), BATCH_SIZE 320, 4 epochs
    = 52 SGD steps through prepare_data / train, against the oracle learner on the same shuffle stream: the whole
    per-step loss trace, the mean loss and the final weights.

    Observed distances (to the float64 learner, for the CUDA path and for the torch-CPU fp32 learner) are recorded
    through tests/parity_record.py."""
    import xingtian_b200 as xb
    from xingtian_b200 import capi
    E, T = 32, 128
    info = ppo_cnn_info(batch=320, iters=4)
    old_mode = capi.lib().xtb_get_tc_mode()
    capi.lib().xtb_set_tc_mode(tc)        # 1: tcgen05 bf16x3 kernels, 0: fp32 CUDA-core kernels (same engine)
    try:
        alg = xb.alg_builder("PPO", info, alg_cfg(instance_num=E))
        _c2_iteration_vs_oracle(alg, E, T, tc)
    finally:
        capi.lib().xtb_set_tc_mode(old_mode)


def _c2_iteration_vs_oracle(alg, E, T, tc):
    """Three learners on the same shuffle stream: the CUDA path, the torch-CPU fp32 oracle (the reference's arithmetic) and
    the float64 oracle (the yardstick).  The GPU trajectory may sit at most twice as far from float64 as the reference's
    own fp32 arithmetic does (plus the per-step 1e-3 contract as a floor)."""
    from parity_record import record as _record
    w0 = alg.get_weights()
    kw = dict(lr=0.00025, batch_size=320, critic_coef=1.0, ent_coef=0.003, clip_ratio=0.1, max_grad_norm=5.0, num_sgd_iter=4,
              vf_clip=5.0)
    ref = orc.PpoLearner(orc.ppo_cnn_arch(), w0, **kw)
    with orc.precision("f64"):
        ref64 = orc.PpoLearner(orc.ppo_cnn_arch(), w0, **kw)
    trajs = make_trajs(E, T, seed=11)
    for tr in trajs:
        alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
    np.random.seed(5)
    loss = alg.train()
    cat = lambda k: np.concatenate([t[k] for t in trajs])
    label = [cat("action"), cat("logp"), cat("adv").astype(np.float32), cat("old_value"), cat("target_value").astype(np.float32)]
    np.random.seed(5)
    ref_loss, ref_trace = ref.train([cat("cur_state")], label)
    np.random.seed(5)
    with orc.precision("f64"):
        loss64, trace64 = ref64.train([cat("cur_state")], label)
    trace = alg.actor.last_losses
    assert len(trace) == len(ref_trace) == len(trace64) == 52
    w1, r1, r64 = alg.get_weights(), ref.weights(), ref64.weights()
    flat = lambda w: np.concatenate([np.asarray(w[k], np.float64).ravel() for k in w0])
    upd, rupd, upd64 = flat(w1) - flat(w0), flat(r1) - flat(w0), flat(r64) - flat(w0)
    cos = lambda a, b: float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)))
    obs = {"trace_rel(gpu,f64)": rel_err(trace, trace64), "trace_rel(cpu32,f64)": rel_err(ref_trace, trace64),
           "trace_rel(gpu,cpu32)": rel_err(trace, ref_trace),
           "first3_rel(gpu,f64)": rel_err(trace[:3], trace64[:3]), "first3_rel(cpu32,f64)": rel_err(ref_trace[:3], trace64[:3]),
           "weights_l2(gpu,f64)": l2_rel(flat(w1), flat(r64)), "weights_l2(cpu32,f64)": l2_rel(flat(r1), flat(r64)),
           "update_l2(gpu,f64)": l2_rel(upd, upd64), "update_l2(cpu32,f64)": l2_rel(rupd, upd64),
           "update_cos(gpu,f64)": cos(upd, upd64), "update_cos(cpu32,f64)": cos(rupd, upd64),
           "mean_loss": [loss, ref_loss, loss64]}
    _record("c2_iteration/%s" % ("tcgen05" if tc else "fp32"), {k: (["%.6f" % x for x in v] if isinstance(v, list) else "%.3e" % v) for k, v in obs.items()})
    # the first steps carry no amplification yet: the per-step contract
    assert obs["first3_rel(gpu,f64)"] < REL
    # 52 Adam steps on noise-dominated gradients amplify any rounding difference (ReLU mask flips, m/sqrt(v) on near-zero
    # gradients): the reference's own fp32 run drifts from float64 too, and the CUDA path may drift at most twice as far
    assert obs["trace_rel(gpu,f64)"] <= max(2 * obs["trace_rel(cpu32,f64)"], C2_TRACE_FLOOR), obs
    assert abs(loss - loss64) <= max(2 * abs(ref_loss - loss64), C2_TRACE_FLOOR * max(1.0, abs(loss64))), obs
    assert obs["weights_l2(gpu,f64)"] <= max(2 * obs["weights_l2(cpu32,f64)"], C2_WEIGHT_FLOOR), obs


# floors of the trajectory-level bounds: the verdict's targets for a reduction-order-deterministic step
C2_TRACE_FLOOR = 1e-2
C2_WEIGHT_FLOOR = 5e-2


def test_ppo_training_is_bitwise_reproducible():
    """No atomics on the PPO step (ordered split-K finish, per-CTA weight-gradient slabs, per-block head slabs reduced in
    block order): two runs from the same weights and shuffle stream give identical loss traces and identical weights."""
    import xingtian_b200 as xb
    E, T = 16, 64
    trajs = make_trajs(E, T, seed=13)
    runs = []
    w_init = None
    for _ in range(2):
        alg = xb.alg_builder("PPO", ppo_cnn_info(batch=320, iters=2), alg_cfg(instance_num=E))
        if w_init is None:
            w_init = alg.get_weights()
        alg.set_weights(w_init)
        for tr in trajs:
            alg.prepare_data({k: tr[k] for k in ("cur_state", "action", "logp", "adv", "old_value", "target_value")})
        np.random.seed(21)
        alg.train()
        runs.append((np.asarray(alg.actor.last_losses, np.float32), alg.get_weights()))
    assert len(runs[0][0]) == 2 * 4                     # 1024 samples / 320 -> 4 minibatches (ragged last one) x 2 epochs
    assert np.array_equal(runs[0][0], runs[1][0]), (runs[0][0], runs[1][0])
    for k in runs[0][1]:
        assert np.array_equal(runs[0][1][k], runs[1][1][k]), k


def test_batched_predictor_serves_real_ppo_cnn():
    """f2 on the device: E explorers' single-frame requests -> ONE xtb_ppo_predict_host call of batch E on a real PpoCnn;
    each reply carries that explorer's row; values/log-probs equal a direct batched predict (same frames, same batch)."""
    import queue
    import xingtian_b200 as xb
    from xingtian_b200.service.predictor import BatchedPredictor, make_msg
    from xingtian_b200.ipc import UniComm
    E = 24
    alg = xb.alg_builder("PPO", ppo_cnn_info(), alg_cfg())
    calls = []
    real_predict = alg.actor.predict

    def counted(batch):
        calls.append(batch.shape[0])
        return real_predict(batch)

    req, rep = UniComm("ShareByShm"), queue.Queue()
    pred = BatchedPredictor(0, alg, req, rep, predict_fn=counted, max_batch=E, max_wait_s=0.2)
    rng = np.random.default_rng(11)
    frames = rng.integers(0, 256, (E, 84, 84, 4), dtype=np.uint8)
    for i in range(E):
        req.send(make_msg(frames[i].copy(), cmd="predict", sub_cmd="predict", explorer_id=i, broker_id=3))
    replays0 = alg.actor.net.lib.xtb_graph_replay_count()
    assert pred.process_once(timeout=2.0) == E and calls == [E]
    got = {}
    while not rep.empty():
        m = rep.get()
        if m["ctr_info"]["cmd"] == "predict_reply":
            got[m["ctr_info"]["explorer_id"]] = m["data"]
    assert sorted(got) == list(range(E))
    u = None
    ract, rlogp, rval = orc.ppo_predict(orc.ppo_cnn_arch(), alg.get_weights(), frames,
                                        np.full((E, 4), 0.5, np.float32))
    with torch.no_grad():
        logits = orc.forward(orc.ppo_cnn_arch(), alg.get_weights(), frames)[0].numpy()
    lsm = logits - np.log(np.exp(logits - logits.max(1, keepdims=True)).sum(1, keepdims=True)) - logits.max(1, keepdims=True)
    for i in range(E):
        a, lp, v = got[i]
        assert np.ndim(a) == 0 and 0 <= int(a) < 4
        assert abs(float(v[0]) - float(rval[i, 0])) < REL * max(1.0, float(np.abs(rval).max()))
        assert abs(float(lp[0]) - float(lsm[i, int(a)])) < 2e-3          # log-prob of the action it sampled
    # weight sync is a barrier message through the same queue
    w = alg.get_weights()
    w2 = {k: v * 0.5 for k, v in w.items()}
    req.send(make_msg(w2, cmd="predict", sub_cmd="sync_weights"))
    assert pred.process_once(timeout=2.0) == 0
    np.testing.assert_allclose(alg.get_weights()["pi_latent/kernel"], w2["pi_latent/kernel"], rtol=0, atol=0)
    assert alg.actor.net.lib.xtb_graph_replay_count() >= replays0
    req.close()


def test_predict_obs_ring_equals_second_upload():
    """Row 5 of the round-1 verdict: frames uploaded by the learner-side batched predict() stay on the device; a
    prepare_data(ring_rows=...) rollout trains bit-identically to the reference message format carrying cur_state."""
    import xingtian_b200 as xb
    E, T = 4, 16
    trajs = make_trajs(E, T, seed=5)
    keys = ("action", "logp", "adv", "old_value", "target_value")
    out = []
    for use_ring in (False, True):
        alg = xb.alg_builder("PPO", ppo_cnn_info(batch=24, iters=2), alg_cfg())
        if use_ring:
            alg.actor.keep_predict_obs(E, T)
            for t in range(T):                      # the rollout's inference calls, time-major, batch E
                alg.actor.predict(np.stack([trajs[e]["cur_state"][t] for e in range(E)]))
            for e, tr in enumerate(trajs):
                d = {k: tr[k] for k in keys}
                d["ring_rows"] = (e, 0, T)
                alg.prepare_data(d)
        else:
            for tr in trajs:
                alg.prepare_data({k: tr[k] for k in ("cur_state",) + keys})
        np.random.seed(9)
        alg.train()
        out.append((list(alg.actor.last_losses), alg.get_weights()))
    # same frames, same kernels: equal up to the order of the loss-term atomics
    assert rel_err(out[1][0], out[0][0]) < 1e-5
    for k in out[0][1]:
        np.testing.assert_allclose(out[1][1][k], out[0][1][k], rtol=0, atol=2e-6)
