"""CPU tier: the oracle (and the host-side mirror) against fixtures produced by executing the
reference's own source files (tests/golden/make_golden.py)."""
import os
import random

import numpy as np
import pytest

from oracle import xt_oracle as orc

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_gae_bit_exact_vs_reference_data_proc():
    z = np.load(os.path.join(G, "gae.npz"))
    for c in range(6):
        adv, ov, tv = orc.gae(z["c%d_value" % c], z["c%d_reward" % c], z["c%d_done" % c])
        assert adv.dtype == np.float64 and z["c%d_adv" % c].dtype == np.float64   # the reference computes GAE in f64
        np.testing.assert_array_equal(adv, z["c%d_adv" % c])
        np.testing.assert_array_equal(ov, z["c%d_old_value" % c])
        np.testing.assert_array_equal(tv, z["c%d_target_value" % c])


def test_agent_mirror_host_gae_matches_reference():
    from xingtian_b200.agent.ppo import PPO as AgentPPO
    z = np.load(os.path.join(G, "gae.npz"))
    for c in range(6):
        value, reward, done = z["c%d_value" % c], z["c%d_reward" % c], z["c%d_done" % c]
        T = len(reward)
        ag = AgentPPO(agent_config={"device_gae": False})
        for t in range(T):
            ag.add_to_trajectory({"cur_state": np.zeros(4, np.float32), "action": 0, "logp": np.zeros(1, np.float32),
                                  "value": value[t], "reward": float(reward[t]), "done": bool(done[t])})
        traj = ag.get_trajectory(last_pred=(None, None, [value[T]]))
        np.testing.assert_array_equal(traj["adv"], z["c%d_adv" % c])
        np.testing.assert_array_equal(traj["target_value"], z["c%d_target_value" % c])
        assert "value" not in traj
        # raw (device-GAE) form keeps value[T+1]/reward/done for the learner
        ag2 = AgentPPO(agent_config={})
        for t in range(T):
            ag2.add_to_trajectory({"cur_state": np.zeros(4, np.float32), "action": 0, "logp": np.zeros(1, np.float32),
                                   "value": value[t], "reward": float(reward[t]), "done": bool(done[t])})
        raw = ag2.get_trajectory(last_pred=(None, None, [value[T]]))
        assert raw["value"].shape[0] == T + 1 and "adv" not in raw


def test_ppo_minibatch_order_vs_reference_train_loop():
    from xingtian_b200.model.ppo import minibatch_order
    z = np.load(os.path.join(G, "ppo_minibatch.npz"))
    for c in range(4):
        n, bs, iters, seed = [int(x) for x in z["c%d_cfg" % c]]
        np.random.seed(seed)
        perm = minibatch_order(n, iters)
        np.testing.assert_array_equal(perm.reshape(-1), z["c%d_order" % c])
        sizes = [min(bs, n - s) for _ in range(iters) for s in range(0, n, bs)]
        np.testing.assert_array_equal(sizes, z["c%d_sizes" % c])
        # the oracle's train loop visits the same slices and averages per-step losses the same way
        L = object.__new__(orc.PpoLearner)
        L.iters, L.bs = iters, bs
        seen = []

        def fake_step(obs, *rest, _seen=seen):
            _seen.append(np.asarray(obs).astype(np.int64).copy())
            return float(len(_seen))
        L.sgd_step = fake_step
        np.random.seed(seed)
        ids = np.arange(n, dtype=np.float64)
        mean_loss, _ = L.train([ids], [ids, ids, ids, ids, ids])
        np.testing.assert_array_equal(np.concatenate(seen), z["c%d_order" % c])
        assert mean_loss == float(z["c%d_mean_loss" % c])


def test_dqn_targets_vs_reference_train():
    from xingtian_b200.algorithm.replay_buffer import DeviceReplayBuffer, ReplayBuffer
    z = np.load(os.path.join(G, "dqn_target.npz"))
    for c in range(3):
        A, B, n, double, seed = [int(x) for x in z["c%d_cfg" % c]]
        ids = z["c%d_batch_ids" % c]
        # same draw as ReplayBuffer.get_batch (random.sample over the live entries)
        random.seed(seed)
        picks = random.sample(range(n), B)
        np.testing.assert_array_equal(picks, ids)
        rb = ReplayBuffer(1000)
        for i in range(n):
            rb.add(i)
        random.seed(seed)
        np.testing.assert_array_equal(rb.get_batch(B), ids)
        dev = object.__new__(DeviceReplayBuffer)
        dev.count, dev.capacity, dev.head = n, 1000, n
        random.seed(seed)
        np.testing.assert_array_equal(dev.sample_indices(B), ids)
        y = orc.dqn_targets(z["c%d_q" % c][ids], z["c%d_qn_target" % c][ids], z["c%d_action" % c][ids], z["c%d_reward" % c][ids],
                            z["c%d_done" % c][ids], 0.99, z["c%d_qn_online" % c][ids] if double else None)
        np.testing.assert_array_equal(y, z["c%d_y" % c])


def test_impala_slicing_vs_reference():
    z = np.load(os.path.join(G, "impala_proc.npz"))
    bs = int(z["batch_size"]); n = len(z["state_order"])
    count = (n + bs - 1) // bs
    assert count == int(z["n_slices"])
    np.testing.assert_array_equal(z["slice_sizes"], [min(bs, n - i * bs) for i in range(count)])
    np.testing.assert_array_equal(z["state_order"], np.arange(n))
    assert bool(z["done_dtype_is_bool"])
    assert float(z["mean_loss"]) == np.mean(np.arange(1, count + 1))


def test_philox_known_answers():
    z = orc.philox4x32_10(np.zeros((1, 4), np.uint32), np.zeros(2, np.uint32))[0]
    assert [hex(int(v)) for v in z] == ["0x6627e8d5", "0xe169c58d", "0xbc57ac4c", "0x9b00dbd8"]
    p = orc.philox4x32_10(np.array([[0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344]], np.uint32), np.array([0xa4093822, 0x299f31d0], np.uint32))[0]
    assert [hex(int(v)) for v in p] == ["0xd16cfe09", "0x94fdcceb", "0x5001e420", "0x24126ea1"]
    u = orc.philox_uniforms(7, 3, 64, 6)
    assert u.shape == (64, 6) and u.min() > 0 and u.max() < 1


def test_param_counts_and_names():
    assert sum(int(np.prod(s)) for s in orc.param_shapes(orc.ppo_cnn_arch()).values()) == 847493
    assert sum(int(np.prod(s)) for s in orc.param_shapes(orc.impala_cnn_arch()).values()) == 1005109
    assert sum(int(np.prod(s)) for s in orc.param_shapes(orc.dqn_cnn_arch()).values()) == 882084
    names = list(orc.param_shapes(orc.ppo_cnn_arch()).keys())
    assert names[0] == "shared_conv_layer_0/kernel" and names[-1] == "output_value/bias" and "pi_latent/kernel" in names
    assert orc.tensor_shapes(orc.impala_cnn_arch())["explore_agent/conv2d"] == (21, 21, 16)     # TF SAME, stride 4
    assert orc.tensor_shapes(orc.impala_cnn_arch())["explore_agent/conv2d_1"] == (11, 11, 32)
    assert orc._same_pad(84, 8, 4) == (21, 2, 2) and orc._same_pad(21, 4, 2) == (11, 1, 2)


def test_vtrace_matches_naive_recursion():
    rng = np.random.default_rng(0)
    T, B, A = 9, 3, 4
    tp = rng.standard_normal((T, B, A)).astype(np.float32); bp = rng.standard_normal((T, B, A)).astype(np.float32)
    act = rng.integers(0, A, (T, B)); disc = (rng.random((T, B)) > 0.2).astype(np.float32) * 0.99
    rew = rng.standard_normal((T, B)).astype(np.float32); val = rng.standard_normal((T, B)).astype(np.float32)
    boot = rng.standard_normal(B).astype(np.float32)
    vs, pg = orc.vtrace_from_logits(bp, tp, act, disc, rew, val, boot)
    lsm = lambda x: x - np.log(np.exp(x).sum(-1, keepdims=True))
    rho = np.exp(np.take_along_axis(lsm(tp.astype(np.float64)), act[..., None], -1)[..., 0] - np.take_along_axis(lsm(bp.astype(np.float64)), act[..., None], -1)[..., 0])
    c = np.minimum(1, rho)
    vs_ref = np.zeros((T + 1, B)); vs_ref[T] = boot
    nv = np.concatenate([val[1:], boot[None]], 0)
    for t in range(T - 1, -1, -1):   # v_s = V + delta + gamma*c*(v_{s+1} - V_{s+1})   (Espeholt et al. 2018, eq. 1)
        vs_ref[t] = val[t] + c[t] * (rew[t] + disc[t] * nv[t] - val[t]) + disc[t] * c[t] * (vs_ref[t + 1] - nv[t])
    np.testing.assert_allclose(vs, vs_ref[:T], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(pg, c * (rew + disc * vs_ref[1:] - val), rtol=2e-5, atol=2e-5)


def test_data_parallel_gradient_identity():
    """SURVEY 8(e): sum over ranks of gradients computed with the 1/B_global scale == gradient of the global
    minibatch (what xtb_ppo_train does with a communicator installed)."""
    import torch
    arch = orc.ppo_mlp_arch()
    w = orc.init_weights(arch, 3)
    ro = orc.synth_ppo_rollout(1, 1, 40, state_dim=(4,), action_dim=2, dtype=np.float32)
    adv = np.random.default_rng(0).standard_normal(40).astype(np.float32); z = np.zeros(40, np.float32)
    L = orc.PpoLearner(arch, w)
    _, g_full = L.loss_and_grads(ro["obs"], ro["action"], ro["logp"], adv, z, adv)
    parts = []
    for sl in (slice(0, 20), slice(20, 40)):
        _, g = L.loss_and_grads(ro["obs"][sl], ro["action"][sl], ro["logp"][sl], adv[sl], z[sl], adv[sl])
        parts.append([x * 0.5 for x in g])     # local mean over 20 -> global mean over 40
    for a, b, c in zip(g_full, *parts):
        torch.testing.assert_close(a, b + c, rtol=1e-4, atol=1e-6)


def _tf_losses():
    return np.load(os.path.join(G, "tf_losses.npz"))


def test_categorical_and_ppo_losses_vs_reference_code():
    """tf_losses.npz holds what xt/model/tf_dist.py:89-113 and xt/model/ppo/__init__.py:4-25 THEMSELVES return when
    executed over the numpy stand-in for their TensorFlow ops (tests/golden/make_golden.py): the oracle's categorical
    log-prob / entropy and the PPO loss (actor + c_v * critic, xt/model/ppo/ppo.py:89-92) must reproduce them."""
    import torch
    g = _tf_losses()
    for case in range(4):
        p = "ppo%d_" % case
        t = lambda k: torch.from_numpy(g[p + k])
        logits, act = t("logits"), torch.from_numpy(g[p + "action"].astype(np.int64))
        assert np.allclose(-orc.categorical_logp(logits, act).numpy(), g[p + "neglogp"], rtol=1e-5, atol=2e-5)
        assert np.allclose(orc.categorical_entropy(logits).numpy(), g[p + "entropy"], rtol=1e-5, atol=1e-6)
        for (clip, ent), vclip, cc in (((0.1, 0.003), 5.0, 1.0), ((0.2, 0.01), 0.5, 0.5)):
            want = float(g[p + "actor_loss_%g_%g" % (clip, ent)]) + cc * float(g[p + "critic_loss_%g" % vclip])
            got = float(orc.ppo_loss(logits, t("out_v"), act, t("old_logp"), t("adv"), t("old_v"), t("target_v"),
                                     clip, ent, vclip, cc))
            assert abs(got - want) <= 2e-5 * max(1.0, abs(want)), (case, got, want)


def test_vtrace_and_impala_loss_vs_reference_code():
    """vtrace.from_logic_outputs (xt/model/impala/vtrace.py:39-115) and vtrace_loss with its three terms
    (impala_cnn_opt.py:299-351) executed over the numpy TF stand-in: vs / pg_advantages of the oracle's V-trace and the
    total of the oracle's impala_loss (fed the env-major flat layout the learner sees, one dropped step appended)."""
    import torch
    g = _tf_losses()
    for case in range(3):
        p = "vt%d_" % case
        bp, tp, act = g[p + "bp"], g[p + "tp"], g[p + "action"]
        disc, rew, val, boot = g[p + "discount"], g[p + "reward"], g[p + "value"], g[p + "bootstrap"]
        vs, pg = orc.vtrace_from_logits(bp, tp, act, disc, rew, val, boot)
        assert np.allclose(vs, g[p + "vs"], rtol=2e-5, atol=2e-5) and np.allclose(pg, g[p + "pg_adv"], rtol=2e-5, atol=2e-5)
        # env-major flat inputs [B*(T+1), ...]: step T carries the bootstrap value, its other entries are dropped
        T, B, A = tp.shape
        pad = lambda x, fill: np.concatenate([x, np.full((1,) + x.shape[1:], fill, x.dtype)], 0)
        flat = lambda x: np.ascontiguousarray(np.swapaxes(x, 0, 1)).reshape((B * (T + 1),) + x.shape[2:])
        tp_f = torch.from_numpy(flat(pad(tp, 0.25)))
        base_f = torch.from_numpy(flat(np.concatenate([val, boot[None]], 0)))
        total = orc.impala_loss(tp_f, base_f, flat(pad(bp, 0.5)), flat(pad(act, 0)), flat(pad(disc == 0, False)),
                                flat(pad(rew, 0.0)), T + 1, gamma=0.99)
        want = float(g[p + "total_loss"])
        parts = float(g[p + "pi_loss"]) + 0.5 * float(g[p + "baseline_loss"]) + 0.01 * float(g[p + "entropy_loss"])
        assert abs(parts - want) <= 1e-5 * abs(want)
        assert abs(float(total) - want) <= 5e-5 * max(1.0, abs(want)), (case, float(total), want)
