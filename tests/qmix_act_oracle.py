"""NumPy restatement of the action choice of QMixModel.act (csrc/agent_act.cuh) from given uniforms: the rule of
EpsilonGreedyActionSelector.select_action with its random numbers taken from `u` instead of the global np.random stream."""
import numpy as np


def select_actions(q, avail, eps, u):
    """q [N, n, A] float32 Q values, avail [N, n, A] action weights, eps [N], u [N, 2, n] float64 -> int64 actions [N, n].
    greedy: np.argmax of q with the weights < 1e-6 at -inf; random: np.random.choice(A, p=avail/sum)'s inverse CDF at
    u[e, 1, a] (float64 cumsum, divided by its last element, searchsorted right); random when u[e, 0, a] < eps[e]."""
    q, avail, u = np.asarray(q), np.asarray(avail), np.asarray(u, np.float64)
    N, n, A = avail.shape
    masked = q.copy()
    masked[avail < 1e-6] = -float("inf")
    greedy = masked.argmax(axis=2)
    rnd = np.empty((N, n), np.int64)
    for e in range(N):
        for a in range(n):
            p = (avail[e, a] / avail[e, a].sum()).astype(np.float64)
            cdf = p.cumsum()
            cdf /= cdf[-1]
            rnd[e, a] = cdf.searchsorted(u[e, 1, a], side="right")
    pick = u[:, 0, :] < np.asarray(eps, np.float64).reshape(N, 1)
    return np.where(pick, rnd, greedy)
