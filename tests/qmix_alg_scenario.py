"""One seeded QMixAlg session shared by tests/golden/make_golden_qmix.py (run on the reference's QMixAlg and episode
buffer) and tests/test_qmix_alg_host.py (run on xingtian_b200's): episodes of random lengths are acted on through
predict_with_selector, stored with prepare_data and trained on with train(episode_num=...), with a stand-in actor that
records what it is handed.  The episode contents come from their own generators; the global np.random stream is left to
the algorithm, whose draws (episode sampling, epsilon-greedy) are what the comparison pins."""
import numpy as np

N_AGENTS, N_ACTIONS, OBS, STATE, LIMIT = 2, 5, 4, 6, 7
N_EPISODES, SEED = 12, 7


def configs():
    """(model_info, alg_config) of QMixAlg; model_name is filled in by the caller."""
    env_attr = dict(n_agents=N_AGENTS, n_actions=N_ACTIONS, state_shape=STATE, obs_shape=OBS, episode_limit=LIMIT)
    alg_config = dict(batch_size=4, buffer_size=6, epsilon_anneal_time=40, epsilon_finish=0.05, epsilon_start=1.0,
                      obs_agent_id=True, obs_last_action=True, target_update_interval=3, env_attr=env_attr, instance_num=1,
                      agent_num=1)
    model_info = {"actor": {"model_config": {"obs_shape": OBS}}}
    return model_info, alg_config


class RecordingActor(object):
    """Stands in for QMixModel: infer_actions is a fixed function of the inputs, train records its arguments."""

    def __init__(self, model_info=None):
        self.trained, self.synced, self.explore_syncs, self.resets = [], [], 0, 0
        self.proj = np.random.default_rng(0).normal(size=(64, N_ACTIONS)).astype(np.float32)

    def infer_actions(self, agent_inputs):
        x = np.asarray(agent_inputs, np.float32).reshape(N_AGENTS, -1)
        q = np.round(np.tanh(x @ self.proj[:x.shape[1]]), 1)     # rounded: ties between actions occur
        return q.reshape(1, N_AGENTS, N_ACTIONS)

    def reset_hidden_state(self):
        self.resets += 1

    def train(self, *args):
        self.trained.append([np.array(a) for a in args])
        return float(len(self.trained))

    def assign_explore_agent(self):
        self.explore_syncs += 1

    def assign_targets(self):
        self.synced.append(len(self.trained))


def episode(i):
    """Episode i as a [LIMIT + 1, ...] transition dict (zero padding past its length), and its length."""
    rng = np.random.default_rng(100 + i)
    T = LIMIT + 1
    m = int(rng.integers(2, T + 1))
    d = dict(state=np.zeros((T, STATE), np.float32), obs=np.zeros((T, N_AGENTS, OBS), np.float32),
             actions=np.zeros((T, N_AGENTS, 1), np.int64), avail_actions=np.zeros((T, N_AGENTS, N_ACTIONS), np.int32),
             reward=np.zeros((T, 1), np.float32), terminated=np.zeros((T, 1), np.uint8), filled=np.zeros((T, 1), np.int64))
    d["state"][:m] = rng.normal(size=(m, STATE)).round(3)
    d["obs"][:m] = rng.normal(size=(m, N_AGENTS, OBS)).round(3)
    av = (rng.random((m, N_AGENTS, N_ACTIONS)) < 0.5).astype(np.int32)
    av[..., int(rng.integers(0, N_ACTIONS))] = 1
    d["avail_actions"][:m] = av
    d["actions"][:m, :, 0] = rng.integers(0, N_ACTIONS, size=(m, N_AGENTS))
    d["reward"][:m, 0] = rng.normal(size=m).round(3)
    d["terminated"][m - 1, 0] = 1 if i % 3 else 0
    d["filled"][:m] = 1
    return d, m


def drive(alg, new_episode_batch):
    """Run the session on `alg` (its actor a RecordingActor).  new_episode_batch(alg) -> an empty one-episode batch of
    the algorithm's scheme with the actions preprocess.  Returns {name: array} of everything observable."""
    sampled, draw = [], np.random.choice

    def choice(*a, **k):      # records the buffer's episode draws (the only ones without replacement)
        r = draw(*a, **k)
        if k.get("replace", True) is False:
            sampled.append(np.array(r))
        return r

    np.random.choice = choice
    try:
        out = _session(alg, new_episode_batch)
    finally:
        np.random.choice = draw
    out["n_sampled"] = np.array(len(sampled))
    for k, ids in enumerate(sampled):
        out["sample%d_ids" % k] = ids
    return out


def _session(alg, new_episode_batch):
    np.random.seed(SEED)
    out, t_env, losses, ready, eps = {}, 0, [], [], []
    acted = []
    for i in range(N_EPISODES):
        d, m = episode(i)
        eb = new_episode_batch(alg)
        alg.reset_hidden_state()
        test_mode = i % 5 == 4
        for t in range(m):
            one = lambda x: x[t][None, None]     # [1, 1, ...]: the (episode, step) block the update writes
            eb.update({"state": one(d["state"]), "obs": one(d["obs"]), "avail_actions": one(d["avail_actions"])}, ts=t)
            act = alg.predict_with_selector(eb, t, t_env, test_mode)
            acted.append(np.asarray(act).reshape(-1))
            eps.append(alg.selector.epsilon)
            eb.update({"actions": np.asarray(act).reshape(1, 1, N_AGENTS, 1), "reward": one(d["reward"]),
                       "terminated": one(d["terminated"])}, ts=t, mark_filled=False)
            t_env += 1
        alg.prepare_data(d)
        ready.append(alg.buffer.can_sample(alg.alg_config["batch_size"]))
        losses.append(alg.train(episode_num=i + 1))
    out["acted"], out["epsilon"] = np.array(acted), np.array(eps, np.float64)
    out["losses"], out["ready"] = np.array(losses, np.float64), np.array(ready)
    out["synced_after_train"] = np.array(alg.actor.synced)
    out["explore_syncs"], out["resets"] = np.array(alg.actor.explore_syncs), np.array(alg.actor.resets)
    out["obs_shape"] = np.array(alg.obs_shape)
    out["n_trained"] = np.array(len(alg.actor.trained))
    names = ("trajectories", "obs_len", "avail", "actions", "cur_stats", "target_stats", "rewards", "terminated", "mask")
    for k, args in enumerate(alg.actor.trained):
        for name, a in zip(names, args):
            out["train%d_%s" % (k, name)] = a
    return out
