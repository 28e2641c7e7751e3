"""DQNInfoFlowAlg on the CUDA engine (xt/algorithm/dqn/dqn_infoflw_alg.py): the host side of the InfoFlow recommender
DQN.  The replay buffer and its random.sample draw stay on the host, as in the reference; a train call packs the
minibatch into flat arrays (the next states once per transition, their candidates ragged behind offsets instead of
tiled) and DqnInfoFlowModel.train_transitions runs the target computation and the fit step as one device graph."""
import numpy as np

from ..model.dqn_infoflow import N_HISTORY, ids_int32
from ..model.impala_keras import fit_order
from ..registry import Registers
from .base import Algorithm
from .replay_buffer import ReplayBuffer

# xt/algorithm/dqn/default_config.py
BATCH_SIZE = 32
BUFFER_SIZE = 100000
TARGET_UPDATE_FREQ = 1000
GAMMA = 0.99


@Registers.algorithm
class DQNInfoFlowAlg(Algorithm):
    """DQNInfoFlowAlg (dqn_infoflw_alg.py:47-242)."""

    def __init__(self, model_info, alg_config, **kwargs):
        model_info = model_info["actor"]
        super().__init__(alg_name="info_flow_dqn", model_info=model_info, alg_config=alg_config)
        from ..registry import model_builder
        self.target_actor = model_builder(model_info)
        self.buff = ReplayBuffer(alg_config.get("buffer_size", BUFFER_SIZE))
        self.batch_size = alg_config.get("batch_size", BATCH_SIZE)
        self.target_update_freq = alg_config.get("target_update_freq", TARGET_UPDATE_FREQ)
        self.gamma = alg_config.get("gamma", GAMMA)
        self.item_dim = alg_config.get("item_dim")
        self.user_dim = alg_config.get("user_dim")
        self.async_flag = False

    # ---- data -------------------------------------------------------------------------------------------------------
    def _check_state(self, s, where):
        vocab = self.actor.vocab_size
        ids_int32(s["user"], vocab, where + " user")
        for k in ("clicked_items", "viewed_items"):
            a = ids_int32(s[k], vocab, where + " " + k)
            if a.size != N_HISTORY * self.item_dim:
                raise ValueError("{} {}: {} ids expected (5 items of item_dim {}), got {}".format(where, k, N_HISTORY * self.item_dim,
                                                                                              self.item_dim, a.size))

    def prepare_data(self, train_data, **kwargs):
        """dqn_infoflw_alg.py:197-219: every transition into the replay buffer, each checked first (ValueError): ids in
        [0, vocab_size) after the int32 cast, histories of 5 item_dim ids, and candidates for every transition that is
        not done (the reference fails on an empty one later, in np.argmax)."""
        vocab = self.actor.vocab_size
        n = len(train_data["done"])
        for i in range(n):
            cur, nxt = train_data["cur_state"][i], train_data["next_state"][i]
            self._check_state(cur, "cur_state[%d]" % i)
            self._check_state(nxt, "next_state[%d]" % i)
            ids_int32(train_data["action"][i], vocab, "action[%d]" % i)
            cand = ids_int32(nxt["candidate_items"], vocab, "next_state[%d] candidate_items" % i)
            if not train_data["done"][i] and len(nxt["candidate_items"]) == 0:
                raise ValueError("next_state[%d]: a transition that is not done needs candidate items" % i)
            if cand.size % self.item_dim:
                raise ValueError("next_state[%d] candidate_items: whole items of item_dim %d ids expected" % (i, self.item_dim))
        for i in range(n):
            self.buff.add((train_data["cur_state"][i], train_data["action"][i], train_data["reward"][i], train_data["next_state"][i],
                           train_data["done"][i]))

    def pack(self, minibatch):
        """The minibatch as flat arrays: the reference's q_input_batch (user, click, noclick, item), the next states once
        per transition (next_user, next_click, next_noclick), their candidates cand_item [n_cand, item_dim] behind
        cand_off [B + 1] (the reference tiles each next state over its candidates instead), reward (float64) and done."""
        ud, h = self.user_dim, self.item_dim * N_HISTORY
        i32 = lambda rows, w: np.asarray(rows).astype(np.int32).reshape(-1, w)
        counts = [len(nxt["candidate_items"]) for _, _, _, nxt, _ in minibatch]
        cand = [np.asarray(nxt["candidate_items"]).astype(np.int32).reshape(-1, self.item_dim) for _, _, _, nxt, _ in minibatch]
        return dict(user=i32([s["user"] for s, _, _, _, _ in minibatch], ud),
                    click=i32([s["clicked_items"] for s, _, _, _, _ in minibatch], h),
                    noclick=i32([s["viewed_items"] for s, _, _, _, _ in minibatch], h),
                    item=i32([a for _, a, _, _, _ in minibatch], self.item_dim),
                    next_user=i32([n["user"] for _, _, _, n, _ in minibatch], ud),
                    next_click=i32([n["clicked_items"] for _, _, _, n, _ in minibatch], h),
                    next_noclick=i32([n["viewed_items"] for _, _, _, n, _ in minibatch], h),
                    cand_off=np.concatenate([[0], np.cumsum(counts)]).astype(np.int32),
                    cand_item=np.concatenate(cand) if cand else np.zeros((0, self.item_dim), np.int32),
                    reward=np.array([r for _, _, r, _, _ in minibatch], np.float64),
                    done=np.array([bool(d) for _, _, _, _, d in minibatch], np.int32))

    # ---- training ---------------------------------------------------------------------------------------------------
    def train(self, **kwargs):
        """dqn_infoflw_alg.py:76-174: sample, target from the online actor's Q over every candidate, one fit step, and
        update_target every target_update_freq-th episode_num -> the loss before the update."""
        minibatch = self.buff.get_batch(self.batch_size)
        if len(minibatch) < self.batch_size:
            raise IndexError("list index out of range: {} transitions stored, batch_size {}".format(len(minibatch), self.batch_size))
        batch = self.pack(minibatch)
        fit_order(self.batch_size)       # model.fit's shuffle of its one minibatch
        loss = self.actor.train_transitions(batch, self.gamma)
        if kwargs["episode_num"] % self.target_update_freq == 0:
            self.update_target()
        return loss

    def restore(self, model_name=None, model_weights=None):
        """dqn_infoflw_alg.py:176-195: actor and target actor."""
        if model_weights:
            self.actor.set_weights(model_weights)
            self.target_actor.set_weights(model_weights)
        else:
            self.actor.load_model(model_name)
            self.target_actor.load_model(model_name)

    def update_target(self):
        self.target_actor.set_weights(self.actor.get_weights())

    def train_ready(self, elapsed_episode, **kwargs):
        """dqn_infoflw_alg.py:229-242: not ready before learning_starts episodes; then the caller's dist_dummy_model is
        called (KeyError without one)."""
        self._train_ready = True
        if elapsed_episode < self.learning_starts:
            self._train_ready = False
            if not kwargs.get("dist_dummy_model"):
                raise KeyError("rec need to dist dummy model.")
            kwargs["dist_dummy_model"]()
        return self._train_ready
