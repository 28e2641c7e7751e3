"""CPU tier: SCC's host side against tests/golden/scc.npz, which the reference's own SCCAlg and SCCModel.train produced
(tests/golden/make_golden_scc.py):
- SCCAlg's seeded session (tests/qmix_alg_scenario.py), bit for bit: every array handed to train, the raw observations
  second, the episode draws, epsilon values, selected actions and target syncs, and the train_ready message;
- the critic states SCCModel.train hands its critic (the reference's alias shift), bit for bit;
- the credits: SCCModel's credit methods and the float64 restatement (tests/scc_oracle.py) with the subsets
  SCCModel.draw_subsets takes from Python's `random`, against the reference's, and the state of `random` afterwards."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import xt_oracle as orc
import qmix_alg_scenario as sc
import scc_oracle as so

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scc.npz")
TRAIN_NAMES = ("trajectories", "obs", "obs_len", "avail", "actions", "cur_stats", "target_stats", "rewards", "terminated", "mask")
O, A = 3, 4


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


def test_alg_session_matches_the_reference_bit_for_bit(gold):
    from xingtian_b200.algorithm.qmix import EpisodeBatch
    from xingtian_b200.algorithm.scc import SCCAlg
    from xingtian_b200.registry import Registers

    class SccGoldenModel(sc.RecordingActor):
        pass

    Registers.model(SccGoldenModel)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "SccGoldenModel"
    alg = SCCAlg(model_info, alg_config)
    out = sc.drive(alg, lambda a: EpisodeBatch(a.scheme, a.groups, 1, sc.LIMIT + 1, preprocess=a.preprocess))
    out = {k: v for k, v in out.items() if not k.startswith("train")}
    for k, args in enumerate(alg.actor.trained):
        for name, a in zip(TRAIN_NAMES, args):
            out["train%d_%s" % (k, name)] = a
    out["alg_name"] = np.array(alg.alg_name)
    model_info, alg_config = sc.configs()
    model_info["actor"]["model_name"] = "SccGoldenModel"
    with pytest.raises(KeyError) as e:
        SCCAlg(model_info, alg_config).train_ready(0)
    out["train_ready_error"] = np.array(str(e.value.args[0]))
    want = {k[4:]: v for k, v in gold.items() if k.startswith("alg_")}
    assert sorted(out) == sorted(want)
    for k in sorted(want):
        assert out[k].dtype == want[k].dtype, (k, out[k].dtype, want[k].dtype)
        assert np.array_equal(out[k], want[k], equal_nan=out[k].dtype.kind == "f"), k


def _cases(gold):
    k = 0
    while "c%d_config" % k in gold:
        yield k
        k += 1


def _case(gold, k):
    cfg = gold["c%d_config" % k]
    n, multi, merge, mc = int(cfg[0]), bool(cfg[1]), {-1: None, 0: "concat", 1: "add"}[int(cfg[2])], int(cfg[3])
    groups = [int(x) for x in cfg[4:]]
    pre = "c%d_w_" % k
    w = {key[len(pre):]: v for key, v in gold.items() if key.startswith(pre)}
    return n, dict(n_agents=n, n_actions=A, multi=multi, groups=groups, merge=merge), mc, w


def test_critic_states_are_the_reference_shifted_states(gold):
    for k in _cases(gold):
        assert bool(gold["c%d_aliased" % k])       # the reference hands the same (shifted) array to both critics
        s = so.critic_states(gold["c%d_obs" % k], gold["c%d_actions" % k][..., 0], A)
        assert s.dtype == gold["c%d_mixer_state" % k].dtype
        assert np.array_equal(s, gold["c%d_mixer_state" % k]), k


def _model(n, mc, crit):
    from xingtian_b200.model.scc import SCCModel
    m = SCCModel.__new__(SCCModel)
    m.n_agents, m.model_config = n, {"mc_sample_times": mc}
    m.get_mixer_output = crit
    return m


def test_credits_and_random_stream_match_the_reference(gold):
    for k in _cases(gold):
        n, cfg, mc, w = _case(gold, k)
        s = gold["c%d_mixer_state" % k]
        want = gold["c%d_target_q_val" % k].reshape(s.shape[0], s.shape[1], n)
        with orc.precision("f64"):
            wt = {key: torch.as_tensor(v) for key, v in w.items()}
            m = _model(n, mc, lambda x: so.critic(wt, x, cfg).numpy())
            # the model's host credit methods, on a float64 critic
            random.seed(1000 + k)
            ex = (m.get_ex_according_to_mcshap_mask if n > 2 else m.get_ex_according_to_mask)(s, n, O, A)
            assert np.array_equal(np.array(random.getstate()[1], np.int64), gold["c%d_random_state" % k]), k
            np.testing.assert_allclose(ex.reshape(want.shape), want, rtol=1e-10, atol=1e-10)
            # the device step's inputs: the subsets as bitmasks, the restatement's literal masked forwards
            random.seed(1000 + k)
            subsets = m.draw_subsets() if n > 2 else None
            assert np.array_equal(np.array(random.getstate()[1], np.int64), gold["c%d_random_state" % k]), k
            np.testing.assert_allclose(so.credits(wt, s, cfg, subsets).numpy(), want, rtol=1e-10, atol=1e-10)
