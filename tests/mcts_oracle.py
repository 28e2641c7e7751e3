"""Float64 restatement of the reference's MuZero tree search (xt/agent/muzero/mcts.py, util.py) over N trees in lock step.

search() advances N independent trees together so that each simulation evaluates every leaf with ONE batched call of an
inference callback, as the device search does; with N = 1 it is the reference's Mcts.run_mcts step for step.  The tree
arithmetic is Python floats (float64) on priors widened from the network's float32 policy, the arithmetic NumPy 1.x
gave the reference.  StandIn is a small float32 network built from IEEE-exact elementwise operations only (no BLAS, no
transcendental functions), so it computes the same bits on every host; the golden fixture (tests/golden/mcts.npz) was
made by running the reference's own code on it."""
import math

import numpy as np

PB_C_BASE, PB_C_INIT, DISCOUNT, FRAC = 19652, 1.25, 0.997, 0.25


class StandIn(object):
    """initial(obs [N, D]) -> (policy [N, A] float32, hidden rows) and recurrent(hidden rows, action [N]) -> (value [N],
    reward [N], policy [N, A], hidden rows): softsign layers, a squared-distance policy, scalar heads; float32."""

    def __init__(self, obs_dim, A, H=4, seed=0):
        rng = np.random.default_rng(seed)
        f = lambda *s: rng.uniform(-1, 1, s).astype(np.float32)
        self.A, self.H = A, H
        self.w_obs, self.w_dyn, self.w_pol = f(obs_dim, H), f(H + A, H), f(H, A)
        self.w_val, self.w_rew = f(H), f(H + A)

    @staticmethod
    def _dot(x, w):     # x [K] . w [K, ...] with a fixed summation order
        acc = np.zeros(w.shape[1:], np.float32)
        for k in range(len(x)):
            acc = acc + np.float32(x[k]) * w[k]
        return acc

    def _policy(self, h):
        z = self._dot(h, self.w_pol)
        w = (z - z.min() + np.float32(0.25)) * (z - z.min() + np.float32(0.25))
        s = np.float32(0)
        for v in w:
            s = s + v
        return w / s

    def _hidden(self, x, w):
        y = self._dot(x, w)
        return y / (np.float32(1) + np.abs(y))

    def initial_one(self, obs):
        h = self._hidden(np.asarray(obs, np.float32).reshape(-1), self.w_obs)
        return self._policy(h), h

    def recurrent_one(self, hidden, action):
        x = np.concatenate([np.asarray(hidden, np.float32), np.eye(self.A, dtype=np.float32)[int(action)]])
        h = self._hidden(x, self.w_dyn)
        value = float(np.float32(3) * self._dot(h, self.w_val))
        reward = float(self._dot(x, self.w_rew))
        return value, reward, self._policy(h), h

    def initial(self, obs):
        out = [self.initial_one(o) for o in obs]
        return np.stack([p for p, _ in out]), [h for _, h in out]

    def recurrent(self, hidden, action):
        out = [self.recurrent_one(h, a) for h, a in zip(hidden, action)]
        return ([o[0] for o in out], [o[1] for o in out], np.stack([o[2] for o in out]), [o[3] for o in out])


class _Tree(object):
    """Node n's child edges: prior, visit count, value sum, expanded child node (-1: not expanded)."""

    def __init__(self, prior, hidden):
        self.prior, self.visits, self.vsum, self.child = [list(prior)], [[0] * len(prior)], [[0.0] * len(prior)], [[-1] * len(prior)]
        self.reward, self.hidden = [0.0], [hidden]
        self.root_visits, self.root_vsum = 0, 0.0
        self.min, self.max = float("inf"), -float("inf")

    def normalize(self, v):
        return (v - self.min) / (self.max - self.min) if self.max > self.min else v

    def update(self, v):
        self.max = max(self.max, v)
        self.min = min(self.min, v)


def search(initial, recurrent, obs, num_simulations, noise=None, pb_c_base=PB_C_BASE, pb_c_init=PB_C_INIT, discount=DISCOUNT,
           frac=FRAC):
    """-> (visit_counts [N, A] int64, root_value [N] float64, margin): margin is the smallest relative gap between the
    best and the second-best UCB score over every descent step whose parent has been visited (with N_p = 0 all scores
    are exactly 0 and the higher action wins by construction)."""
    policy, hidden = initial(obs)
    policy = np.asarray(policy, np.float64)
    N, A = policy.shape
    trees = []
    for e in range(N):
        prior = [float(p) for p in policy[e]]
        if noise is not None:
            prior = [p * (1 - frac) + float(nz) * frac for p, nz in zip(prior, noise[e])]
        trees.append(_Tree(prior, hidden[e]))
    margin = float("inf")
    for s in range(1, num_simulations + 1):
        paths = []
        for t in trees:
            node, np_, path = 0, t.root_visits, []
            while True:
                pb = math.log((np_ + pb_c_base + 1) / pb_c_base) + pb_c_init
                scores = []
                for a in range(A):
                    nc = t.visits[node][a]
                    sc = pb * (math.sqrt(np_) / (nc + 1)) * t.prior[node][a]
                    if nc > 0:
                        sc = sc + t.normalize(t.vsum[node][a] / nc)
                    scores.append(sc)
                best = max((sc, a) for a, sc in enumerate(scores))
                if np_ > 0 and A > 1:
                    second = max(sc for a, sc in enumerate(scores) if a != best[1])
                    margin = min(margin, (best[0] - second) / max(abs(best[0]), abs(second), 1e-300))
                a = best[1]
                path.append((node, a))
                c = t.child[node][a]
                if c < 0:
                    break
                np_, node = t.visits[node][a], c
            paths.append(path)
        value, reward, pol, hid = recurrent([t.hidden[p[-1][0]] for t, p in zip(trees, paths)], [p[-1][1] for p in paths])
        pol = np.asarray(pol, np.float64)
        for e, (t, path) in enumerate(zip(trees, paths)):
            p, a = path[-1]
            t.child[p][a] = s
            t.prior.append([float(x) for x in pol[e]])
            t.visits.append([0] * A)
            t.vsum.append([0.0] * A)
            t.child.append([-1] * A)
            t.reward.append(float(reward[e]))
            t.hidden.append(hid[e])
            v = float(value[e])
            for p, a in reversed(path):
                t.vsum[p][a] += v
                t.visits[p][a] += 1
                t.update(t.vsum[p][a] / t.visits[p][a])
                v = t.reward[t.child[p][a]] + discount * v
            t.root_vsum += v
            t.root_visits += 1
            t.update(t.root_vsum / t.root_visits)
    counts = np.array([[t.visits[0][a] for a in range(A)] for t in trees], np.int64)
    root_value = np.array([t.root_vsum / t.root_visits for t in trees], np.float64)
    return counts, root_value, margin
