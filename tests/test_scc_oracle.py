"""CPU tier: the SCC restatement (tests/scc_oracle.py) on its own terms: the reference's shifted critic states, the
credit identities of the multi-channel critic, the subset draws of Python's `random`, uncentred RMSProp and the losses'
gradients by finite differences."""
import random

import numpy as np
import torch

from oracle import xt_oracle as orc
import scc_oracle as so


def test_critic_states_are_shifted_through_the_alias():
    raw = np.arange(2 * 5 * 1 * 1, dtype=np.float32).reshape(2, 5, 1, 1) * 3
    act = np.zeros((2, 4, 1), np.int64)
    s = so.critic_states(raw, act, 2)
    assert s[0, :, 0].tolist() == [3, 6, 9, 9]      # rows [0, 3, 6, 9] shifted: s'[t] = s[min(t + 1, L - 1)]
    assert s[0, :, 1].tolist() == [1, 1, 1, 1]      # action 0 one-hot, float64
    assert s.dtype == np.float64


def _weights(rng, n, D, U, groups, merge):
    w = {}
    for j in range(len(groups)):
        for name, shape in (("dense/kernel", (D, U)), ("dense/bias", (U,)), ("dense_1/kernel", (U, U)), ("dense_1/bias", (U,))):
            w["channel_%d/%s" % (j, name)] = rng.normal(size=shape) * 0.5
    K = n * U if merge == "concat" else U
    w["v/kernel"], w["v/bias"] = rng.normal(size=(K, 1)), rng.normal(size=(1,))
    return w


def test_multi_channel_credits_do_not_depend_on_the_subsets():
    rng = np.random.default_rng(0)
    n, A, o, U = 5, 3, 2, 6
    cfg = dict(n_agents=n, n_actions=A, multi=True, groups=[2, 3], merge="concat")
    w = {k: torch.as_tensor(v) for k, v in _weights(rng, n, o + A, U, [2, 3], "concat").items()}
    s = rng.normal(size=(2, 3, n * (o + A)))
    with orc.precision("f64"):
        full = (1 << n) - 1
        one = np.array([[1 << ((i + 1) % n)] * 2 for i in range(n)], np.uint32)       # S = {the next agent}
        rest = np.array([[full & ~(1 << i)] * 2 for i in range(n)], np.uint32)       # S = every other agent
        a = so.credits(w, s, cfg, one)
        b = so.credits(w, s, cfg, rest)
    np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-12, atol=1e-12)


def test_subset_draws_follow_the_reference_order():
    from xingtian_b200.model.scc import SCCModel
    m = SCCModel.__new__(SCCModel)
    m.n_agents, m.model_config = 4, dict(mc_sample_times=3)
    random.seed(11)
    got = m.draw_subsets()
    random.seed(11)
    for i in range(4):
        for j in range(3):
            agents = [x for x in range(4)]
            agents.remove(i)
            k = random.randint(1, 3)
            assert got[i, j] == sum(1 << a for a in random.sample(agents, k))


def test_uncentred_rmsprop():
    p = torch.tensor([1.0], dtype=torch.float64)
    opt = so.TFRMSPropPlain([p], 0.1, decay=0.9, eps=1e-10)
    opt.step([torch.tensor([2.0], dtype=torch.float64)])
    ms = 0.9 + 0.1 * 4.0
    assert abs(p.item() - (1.0 - 0.1 * 2.0 / np.sqrt(ms + 1e-10))) < 1e-15


def test_losses_by_finite_differences():
    rng = np.random.default_rng(1)
    n, A, o, U, H, B, L = 3, 4, 2, 5, 6, 2, 4
    b = so.synth_batch(3, B, L, n, A, o, max_ep_t=L)
    cfg = dict(n_agents=n, n_actions=A, multi=True, groups=[n], merge="add", gamma=0.99)
    subsets = np.array([[1 << ((i + 1) % n), 7 & ~(1 << i)] for i in range(n)], np.uint32)
    wc = _weights(rng, n, o + A, U, [n], "add")
    obs = b["obs"].shape[-1]
    wa = {"dense/kernel": rng.normal(size=(obs, H)) * 0.3, "dense/bias": np.zeros(H),
          "rnn/gru_cell/gates/kernel": rng.normal(size=(2 * H, 2 * H)) * 0.3, "rnn/gru_cell/gates/bias": np.ones(2 * H),
          "rnn/gru_cell/candidate/kernel": rng.normal(size=(2 * H, H)) * 0.3, "rnn/gru_cell/candidate/bias": np.zeros(H),
          "dense_1/kernel": rng.normal(size=(H, A)) * 0.3, "dense_1/bias": np.zeros(A)}
    with orc.precision("f64"):
        ta = {k: torch.tensor(v, requires_grad=True) for k, v in wa.items()}
        tc = {k: torch.tensor(v, requires_grad=True) for k, v in wc.items()}
        tt = {k: torch.tensor(v) * 0.9 for k, v in wc.items()}
        mixer, actor, credit = so.step_losses(ta, tc, tt, b, cfg, subsets)
        gm = torch.autograd.grad(mixer, [tc["v/kernel"]])[0].numpy()
        ga = torch.autograd.grad(actor, [ta["dense_1/bias"]])[0].numpy()
        eps = 1e-6
        for (name, tab, g, which) in (("v/kernel", tc, gm, 0), ("dense_1/bias", ta, ga, 1)):
            flat = tab[name].detach().numpy().reshape(-1)
            for idx in range(min(3, flat.size)):
                def f(delta):
                    t2 = {k: v.detach().clone() for k, v in tab.items()}
                    t2[name].view(-1)[idx] += delta
                    args = (ta, t2, tt) if which == 0 else (t2, tc, tt)
                    out = so.step_losses(*[{k: v.detach() for k, v in d.items()} for d in args], b, cfg, subsets)
                    return out[which].item()
                num = (f(eps) - f(-eps)) / (2 * eps)
                assert abs(num - g.reshape(-1)[idx]) <= 1e-6 * max(1.0, abs(num)), (name, idx, num, g.reshape(-1)[idx])
