"""A seeded InfoFlow DQN session shared by tests/golden/make_golden_infoflow.py (which runs the reference's own
DQNInfoFlowAlg on it) and tests/test_infoflow_host.py (which runs this package's): transitions with ragged candidate
counts (1 to a few hundred), mixed done flags and float rewards, a replay buffer small enough to evict, and train calls
with target syncs.  The stand-in actors record what the algorithm hands them instead of computing."""
import random

import numpy as np

VOCAB, USER_DIM, ITEM_DIM = 50, 3, 2
BATCH, BUFFER, SYNC_FREQ, GAMMA = 8, 40, 3, 0.95
ROUNDS, PER_ROUND = 9, 6
SEED = 2024


def configs():
    model_info = {"actor": dict(model_name="RecordingInfoflowActor", state_dim=[1], action_dim=1, vocab_size=VOCAB, emb_dim=4,
                                user_dim=USER_DIM, item_dim=ITEM_DIM, input_type="int32", embeddings="", last_activate="linear")}
    alg_config = dict(instance_num=1, agent_num=1, buffer_size=BUFFER, batch_size=BATCH, target_update_freq=SYNC_FREQ, gamma=GAMMA,
                      item_dim=ITEM_DIM, user_dim=USER_DIM)
    return model_info, alg_config


def transitions(rng, first_id, n):
    """n transitions of the explorer's form; every state carries its transition id under "tid" (read by nothing)."""
    def state(tid):
        k = int(rng.integers(1, 300)) if rng.random() < 0.4 else int(rng.integers(1, 6))
        return dict(tid=tid, user=rng.integers(0, VOCAB, USER_DIM).tolist(), clicked_items=rng.integers(0, VOCAB, 5 * ITEM_DIM).tolist(),
                    viewed_items=rng.integers(0, VOCAB, 5 * ITEM_DIM).tolist(),
                    candidate_items=rng.integers(0, VOCAB, (k, ITEM_DIM)).tolist())
    ids = range(first_id, first_id + n)
    return dict(cur_state=[state(i) for i in ids], action=[rng.integers(0, VOCAB, ITEM_DIM).tolist() for _ in ids],
                reward=[float(rng.uniform(-1, 2)) for _ in ids], next_state=[state(i) for i in ids],
                done=[bool(rng.random() < 0.35) for _ in ids])


class Recorder(object):
    """The calls both stand-in actors record; q_values are float32 values (as the Keras model returns) carried as
    float64, so that NumPy 2's promotion computes the float64 target NumPy 1 computed from float32 Q values."""

    def __init__(self):
        self.rs = np.random.RandomState(7)     # its own stream: the global ones stay the algorithm's
        self.predicts, self.trains, self.syncs = [], [], []

    def q_values(self, n):
        return self.rs.standard_normal(n).astype(np.float32).astype(np.float64)


def stream_state():
    """(Python random's state, NumPy's MT19937 key and position) as arrays."""
    py = np.array(random.getstate()[1], np.int64)
    _, key, pos, _, _ = np.random.get_state()
    return py, np.asarray(key, np.int64), int(pos)


def drive(alg, recorder):
    """The session: ROUNDS prepare_data calls of PER_ROUND transitions, a train after each once a batch is stored
    (episode_num counting from 1).  -> dict of arrays for the golden."""
    random.seed(SEED)
    np.random.seed(SEED)
    rng = np.random.default_rng(SEED)
    out = dict(py_state=[], np_key=[], np_pos=[], synced_after_train=[])
    n_train = 0
    for r in range(ROUNDS):
        alg.prepare_data(transitions(rng, r * PER_ROUND, PER_ROUND))
        if alg.buff.size() < BATCH:
            continue
        n_syncs = len(recorder.syncs)
        alg.train(episode_num=n_train + 1)
        n_train += 1
        if len(recorder.syncs) > n_syncs:
            out["synced_after_train"].append(n_train)
        py, key, pos = stream_state()
        out["py_state"].append(py)
        out["np_key"].append(key)
        out["np_pos"].append(pos)
    out["n_trained"] = n_train
    return out
