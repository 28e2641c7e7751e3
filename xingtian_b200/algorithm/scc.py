"""SCCAlg (xt/algorithm/scc/scc_alg.py): QMixAlg's host side (episode buffer, agent inputs, epsilon-greedy selection,
target-sync rule), with the raw observations handed to SCCModel.train as its second argument."""
import numpy as np

from ..registry import Registers
from .qmix import QMixAlg


class _ObsSecond(object):
    """The actor as QMixAlg.train sees it: train(trajectories, *rest) becomes actor.train(trajectories, obs, *rest)."""

    def __init__(self, actor, obs):
        self._actor, self._obs = actor, obs

    def train(self, batch_trajectories, *rest):
        return self._actor.train(batch_trajectories, self._obs, *rest)

    def __getattr__(self, name):
        return getattr(self._actor, name)


@Registers.algorithm
class SCCAlg(QMixAlg):
    """SCCAlg (scc_alg.py:115-402): QMixAlg but for its name, the extra `obs = batch["obs"]` argument of train and the
    train_ready message."""

    def __init__(self, model_info, alg_config, **kwargs):
        super().__init__(model_info, alg_config, **kwargs)
        self.alg_name = "SCCAlg"

    def train(self, **kwargs):
        if self.device_replay:
            return super().train(**kwargs)     # SCCModel.train_replay reads the raw obs from the ring
        if not self.train_batch:
            return np.nan
        actor = self.actor
        self.actor = _ObsSecond(actor, self.train_batch["obs"])
        try:
            return super().train(**kwargs)
        finally:
            self.actor = actor

    def train_ready(self, elapsed_episode, **kwargs):
        if not self.buffer.can_sample(self.alg_config["batch_size"]) and not kwargs.get("dist_dummy_model"):
            raise KeyError("scc need to dist dummy model.")
        return super().train_ready(elapsed_episode, **kwargs)
