"""The MuZero agents (xt/agent/muzero/muzero.py, muzero_atari.py, mcts.py) over MuzeroModel.search.

The reference builds one Python tree per environment step and calls the network 1 + NUM_SIMULATIONS times at batch 1.
Here the search runs on the device (xtb_muzero_search): every tree of a batch of observations advances in lock step,
with one batched recurrent inference per simulation.  What stays on the host are the two random draws, made with the
global np.random stream in the reference's order (the root's Dirichlet noise before the search, the visit-count sample
after it), so a seeded run draws the numbers the reference draws.  The env-step loop (run_one_episode, sync_model) stays
in the reference, as for the PPO agents."""
from collections import defaultdict

import numpy as np

from ..registry import Registers

# xt/agent/muzero/default_config.py
PB_C_BASE = 19652
PB_C_INIT = 1.25
NUM_SIMULATIONS = 50
ROOT_DIRICHLET_ALPHA = 0.25
ROOT_EXPLORATION_FRACTION = 0.25
GAMMA = 0.997
TD_STEP = 10


def soft_max_sample(visit_counts, t=1):
    """util.py:55-59: an action drawn with probability counts ** (1 / t) over their sum."""
    counts_exp = np.asarray(visit_counts) ** (1 / t)
    probs = counts_exp / np.sum(counts_exp, axis=0)
    return int(np.random.choice(len(probs), p=probs))


def search_actions(actor, states, num_simulations, use_explore):
    """One search over the observations states [N, ...]: the N root noises drawn first (add_exploration_noise, when
    exploring), then the N actions -> (action [N] int64, child_visits [N, A] float64, root_value [N] float64)."""
    states = np.asarray(states)
    A = actor.action_dim
    noise = None
    if use_explore:
        noise = np.stack([np.random.dirichlet([ROOT_DIRICHLET_ALPHA] * A) for _ in range(len(states))])
    counts, root_value = actor.search(states, num_simulations, noise=noise, pb_c_base=PB_C_BASE, pb_c_init=PB_C_INIT,
                                      discount=GAMMA, exploration_frac=ROOT_EXPLORATION_FRACTION)
    action = np.array([soft_max_sample(c) for c in counts], dtype=np.int64)
    child_visits = counts / counts.sum(axis=1, keepdims=True).astype(np.float64)
    return action, child_visits, np.asarray(root_value, dtype=np.float64)


def search_predict_fn(actor, num_simulations=NUM_SIMULATIONS, use_explore=True):
    """predict_fn of service.BatchedPredictor: the stacked observations of every waiting explorer in one search, answered
    with [action, child_visits, root_value] rows."""
    def predict(batch):
        return list(search_actions(actor, batch, num_simulations, use_explore))
    return predict


@Registers.agent
class Muzero(object):
    """muzero.py:31-91.  NUM_SIMULATIONS, GAMMA and TD_STEP come from agent_config when it sets them (import_config)."""

    def __init__(self, env=None, alg=None, agent_config=None, **kwargs):
        self.env, self.alg = env, alg
        self.agent_config = dict(agent_config or {})
        self.num_simulations = int(self.agent_config.get("NUM_SIMULATIONS", NUM_SIMULATIONS))
        self.gamma = float(self.agent_config.get("GAMMA", GAMMA))
        self.td_step = int(self.agent_config.get("TD_STEP", TD_STEP))
        self.keep_seq_len = False
        self.transition_data = defaultdict()
        self.trajectory = defaultdict(list)

    def infer_actions(self, states, use_explore):
        """N environments' steps from one search: (action [N], child_visits [N, A], root_value [N])."""
        return search_actions(self.alg.actor, states, self.num_simulations, use_explore)

    def infer_action(self, state, use_explore):
        """muzero.py:40-57: the search from one observation, the sampled action and the tree's train info."""
        action, child_visits, root_value = self.infer_actions(np.asarray(state)[None], use_explore)
        action = int(action[0])
        self.transition_data.update({"cur_state": state, "action": action})
        self.transition_data.update({"child_visits": child_visits[0].tolist(), "root_value": float(root_value[0])})
        return action

    def handle_env_feedback(self, next_raw_state, reward, done, info, use_explore):
        info.update({"eval_reward": reward})
        self.transition_data.update({"reward": reward, "done": done, "info": info})
        return self.transition_data

    def add_to_trajectory(self, transition_data):
        for k, val in transition_data.items():
            self.trajectory[k].append(val)

    def get_trajectory(self):
        self.data_proc()
        return dict(self.trajectory)

    def data_proc(self):
        """muzero.py:74-91: the TD_STEP-step bootstrapped target value of every step of the episode."""
        traj = self.trajectory
        value = traj["root_value"]
        reward = traj["reward"]
        dones = np.asarray(traj["done"])
        discounts = ~dones * self.gamma

        target_value = [reward[-1]] * len(reward)
        for i in range(len(reward) - 1):
            end_index = min(i + self.td_step, len(reward) - 1)
            sum_value = value[end_index]
            for j in range(i, end_index)[::-1]:
                sum_value = reward[j] + discounts[j] * sum_value
            target_value[i] = sum_value

        self.trajectory["target_value"] = target_value


@Registers.agent
class MuzeroAtari(Muzero):
    """muzero_atari.py:27-50: uint8 frames, and the trajectory keeps running past episode ends."""

    def __init__(self, env=None, alg=None, agent_config=None, **kwargs):
        super().__init__(env, alg, agent_config, **kwargs)
        self.keep_seq_len = True

    def infer_action(self, state, use_explore):
        return super().infer_action(np.asarray(state).astype("uint8"), use_explore)

    def infer_actions(self, states, use_explore):
        return super().infer_actions(np.asarray(states).astype("uint8"), use_explore)

    def handle_env_feedback(self, next_raw_state, reward, done, info, use_explore):
        next_raw_state = np.asarray(next_raw_state).astype("uint8")
        return super().handle_env_feedback(next_raw_state, reward, done, info, use_explore)
