"""MuZero against tests/golden/muzero.npz, which the reference's own code produced (make_golden_muzero.py): the support
transforms of the float64 oracle, the Muzero learner's sampling, gathering and priorities over its own segment trees
(with a stand-in model whose value is a fixed function of the observation), and the int8 observation cast."""
import os
import random

import numpy as np

import muzero_oracle as mo
from xingtian_b200.algorithm.muzero import Muzero, PrioritizedBuffer

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "muzero.npz"))
RANGES = {"breakout_v": (0, 500), "breakout_r": (0, 50), "pong_v": (-21, 21), "pong_r": (-2, 2), "default_v": (0, 60000)}


def test_value_compression_against_reference():
    np.testing.assert_allclose(mo.h(GOLD["h_x"]), GOLD["h"], rtol=1e-15, atol=1e-15)
    np.testing.assert_allclose(mo.h_inv(GOLD["h"]), GOLD["h_inv"], rtol=1e-13, atol=1e-12)


def test_conver_value_and_value_transform_against_reference():
    for tag, (lo, hi) in RANGES.items():
        S = mo.support_size(lo, hi)
        np.testing.assert_allclose(mo.two_hot(GOLD["cv_in_" + tag], S, lo, hi), GOLD["cv_" + tag], rtol=0, atol=1e-12)
        np.testing.assert_allclose(mo.support_value(GOLD["vt_in_" + tag], lo, hi), GOLD["vt_" + tag], rtol=1e-12, atol=1e-9)


class _Actor(object):
    """the fixture's stand-in model: value = 0.01 * sum of the observation row; train records its minibatch"""
    td_step = 5

    def __init__(self):
        self.trained = []

    def value_inference(self, s):
        return 0.01 * np.asarray(s, np.float64).reshape(len(s), -1).sum(1)

    def train_and_values(self, image, actions, tv, tr, tp):
        self.trained.append((image, actions, tv, tr, tp))
        return 0.0, self.value_inference(image)


def test_learner_against_reference():
    actor = _Actor()
    alg = object.__new__(Muzero)
    alg.actor, alg.buff, alg.unroll_step, alg.batch_size = actor, PrioritizedBuffer(8, alpha=1), 5, 6
    random.seed(1234)
    for t in range(22):
        tr = {k: GOLD["traj%d_%s" % (t, k)] for k in ("cur_state", "action", "reward", "child_visits", "target_value")}
        tr["traj_id"] = t
        alg.prepare_data(tr)
        if t in (3, 12, 21):
            for _ in range(3):
                alg.train()
    assert len(actor.trained) == int(GOLD["n_train_steps"])
    for s, (img, act, tv, tr_, tp) in enumerate(actor.trained):
        np.testing.assert_array_equal(img, GOLD["step%d_image" % s])
        np.testing.assert_array_equal(act, GOLD["step%d_action" % s])
        np.testing.assert_array_equal(tv, GOLD["step%d_tv" % s])
        np.testing.assert_array_equal(tr_, GOLD["step%d_tr" % s])
        np.testing.assert_array_equal(tp, GOLD["step%d_tp" % s])
    buf = alg.buff
    assert len(buf) == int(GOLD["buf_len"])
    assert [d["traj_id"] for d in buf.storage] == list(GOLD["buf_ids"])
    # every priority, the batch-position writes of update_pri included, equals the reference's to the last bit
    np.testing.assert_array_equal([buf.it_sum[i] for i in range(len(buf))], GOLD["buf_pri"])
    np.testing.assert_array_equal(np.concatenate([[d["pos_buff"].it_sum[i] for i in range(len(d["pos_buff"]))]
                                                  for d in buf.storage]), GOLD["buf_pos_pri"])


def test_sample_total_excludes_last_item():
    b = PrioritizedBuffer(4, alpha=1)
    for p in (1.0, 2.0, 3.0, 100.0):
        b.add(object(), p)
    random.seed(0)
    _, _, idx = b.sample(64, 1)
    assert 3 not in idx       # the total spread over the draws is 1 + 2 + 3: the last item cannot be reached


def test_int8_cast_against_reference():
    decoded = mo.decode_obs(np.arange(256, dtype=np.uint8), "int8") / 255.0
    np.testing.assert_array_equal(decoded, GOLD["int8_cast"])

