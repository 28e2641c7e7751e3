#!/usr/bin/env python
"""Generate mcts.npz by EXECUTING the reference's own MuZero agent code:

* Mcts (xt/agent/muzero/mcts.py), MinMaxStats, Node and soft_max_sample (xt/agent/muzero/util.py) and the constants of
  xt/agent/muzero/default_config.py, driven by Muzero.infer_action (xt/agent/muzero/muzero.py:40-57) under np.random.seed,
  so the Dirichlet noise and the action sample come from the reference's own calls in its own order;
* the network is tests/mcts_oracle.StandIn, a small fixed float32 function of (hidden, action) whose NetworkOutput
  carries the value and reward as Python floats (np.asscalar in the reference model) and the policy widened to float64:
  under NumPy 1.x the reference's float32 prior times a Python float was a float64 product, which NumPy 2 (NEP 50) would
  keep in float32;
* Muzero.data_proc (muzero.py:74-91) over a few episodes.

Cases: A in {2, 6}, NUM_SIMULATIONS in {1, 2, 50}, with and without exploration noise, four steps each.  Recorded per
step: the root child visit counts, child_visits, root_value and the chosen action.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_mcts.py
It writes mcts.npz alone."""
import math
import os
import random
import sys
import types
from typing import Optional

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402
from make_golden_muzero import _exec  # noqa: E402
from mcts_oracle import StandIn  # noqa: E402

OBS_DIM, STEPS = 5, 4
CASES = [(A, S, explore) for A in (2, 6) for S in (1, 2, 50) for explore in (False, True)]


def case_key(A, S, explore):
    return "A%d_S%d_%s" % (A, S, "noise" if explore else "plain")


def case_seed(i):
    return 1000 + i


def case_obs(A, S, explore):
    return np.random.default_rng(A * 100 + S * 2 + int(explore)).normal(size=(STEPS, OBS_DIM)).astype(np.float32)


class _NetworkOutput(object):
    def __init__(self, value, reward, policy, hidden_state):
        self.value, self.reward, self.policy, self.hidden_state = value, reward, policy, hidden_state


class _Network(object):
    """The reference network interface (muzero_model.py:74-96) on the stand-in."""

    def __init__(self, net):
        self.net = net

    def initial_inference(self, input_data):
        policy, h = self.net.initial_one(input_data[0])
        return _NetworkOutput(0.0, 0, policy.astype(np.float64), h)

    def recurrent_inference(self, hidden_state, action):
        value, reward, policy, h = self.net.recurrent_one(hidden_state, action)
        return _NetworkOutput(value, reward, policy.astype(np.float64), h)


def main():
    cfg = {}
    exec(compile(open(os.path.join(mg.REF, "xt/agent/muzero/default_config.py")).read(), "default_config.py", "exec"), cfg)
    util = _exec("xt/agent/muzero/util.py", {"np": np, "Optional": Optional, "MAXIMUM_FLOAT_VALUE": float("inf")})
    ns = dict(math=math, np=np, random=random, MinMaxStats=util["MinMaxStats"], Node=util["Node"],
              soft_max_sample=util["soft_max_sample"])
    ns.update({k: v for k, v in cfg.items() if k.isupper()})
    mcts = _exec("xt/agent/muzero/mcts.py", ns, cls=None, names=("Mcts",))
    made = []

    class RecMcts(mcts["Mcts"]):
        def __init__(self, agent, root_state):
            super().__init__(agent, root_state)
            made.append(self)

    agent_fns = _exec("xt/agent/muzero/muzero.py", {"np": np, "Mcts": RecMcts, "GAMMA": cfg["GAMMA"], "TD_STEP": cfg["TD_STEP"]},
                      names=("infer_action", "data_proc"), cls="Muzero")
    out = {}
    for i, (A, S, explore) in enumerate(CASES):
        net = StandIn(OBS_DIM, A, seed=A)
        agent = types.SimpleNamespace(alg=types.SimpleNamespace(actor=_Network(net), action_dim=A), num_simulations=S,
                                      transition_data={})
        np.random.seed(case_seed(i))
        rec = dict(counts=[], child_visits=[], root_value=[], action=[])
        for obs in case_obs(A, S, explore):
            made.clear()
            action = agent_fns["infer_action"](agent, obs, explore)
            root = made[0].root
            rec["counts"].append([root.children[a].visit_count for a in range(A)])
            rec["child_visits"].append(agent.transition_data["child_visits"])
            rec["root_value"].append(agent.transition_data["root_value"])
            rec["action"].append(action)
        for k, v in rec.items():
            out[case_key(A, S, explore) + "_" + k] = np.asarray(v)
    rng = np.random.default_rng(5)
    episodes = [1, 2, 7, 12, 31]
    out["n_episodes"] = np.array(len(episodes))
    for e, L in enumerate(episodes):
        traj = dict(root_value=list(rng.normal(size=L) * 3), reward=list(rng.normal(size=L).round(2)),
                    done=list(rng.random(L) < 0.15))
        self = types.SimpleNamespace(trajectory=dict(traj))
        agent_fns["data_proc"](self)
        for k, v in traj.items():
            out["ep%d_%s" % (e, k)] = np.asarray(v)
        out["ep%d_target_value" % e] = np.asarray(self.trajectory["target_value"], np.float64)
    np.savez(os.path.join(HERE, "mcts.npz"), **out)


if __name__ == "__main__":
    main()
