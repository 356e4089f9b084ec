"""RolloutStorage with the reference's constructor, buffers and methods
(habitat-baselines/habitat_baselines/common/rollout_storage.py:24-275; Storage ABC
common/storage.py:12-56), computing returns with the fused GAE kernel and handing minibatches
to the updater WITHOUT copying observations."""
from __future__ import annotations

import warnings
from typing import Iterator, Optional

import numpy as np
import torch

from .. import ops
from ..rl.resnet_policy import RolloutObservations
from . import spaces
from .baseline_registry import baseline_registry
from .tensor_dict import TensorDict


def get_action_space_info(ac_space):
    """utils/common.py get_action_space_info for the spaces the hot path supports: Discrete -> ((1,), True), a 1-D Box
    of A dimensions -> ((A,), False); other action spaces raise NotImplementedError."""
    dim = spaces.continuous_action_dim(ac_space)
    if dim is None:
        return (1,), True
    return (dim,), False


@baseline_registry.register_storage
class RolloutStorage:
    def __init__(self, numsteps, num_envs, observation_space, action_space, actor_critic,
                 is_double_buffered: bool = False):
        action_shape, discrete_actions = get_action_space_info(action_space)
        self.buffers = TensorDict()
        self.buffers["observations"] = TensorDict()
        for sensor in observation_space.spaces:
            sp = observation_space.spaces[sensor]
            self.buffers["observations"][sensor] = torch.from_numpy(
                np.zeros((numsteps + 1, num_envs, *sp.shape), dtype=sp.dtype))
        self.buffers["recurrent_hidden_states"] = torch.zeros(
            numsteps + 1, num_envs, actor_critic.num_recurrent_layers, actor_critic.recurrent_hidden_size)
        self.buffers["rewards"] = torch.zeros(numsteps + 1, num_envs, 1)
        self.buffers["value_preds"] = torch.zeros(numsteps + 1, num_envs, 1)
        self.buffers["returns"] = torch.zeros(numsteps + 1, num_envs, 1)
        self.buffers["action_log_probs"] = torch.zeros(numsteps + 1, num_envs, 1)
        self.buffers["actions"] = torch.zeros(numsteps + 1, num_envs, *action_shape)
        self.buffers["prev_actions"] = torch.zeros(numsteps + 1, num_envs, *action_shape)
        if discrete_actions:
            self.buffers["actions"] = self.buffers["actions"].long()
            self.buffers["prev_actions"] = self.buffers["prev_actions"].long()
        self.buffers["masks"] = torch.zeros(numsteps + 1, num_envs, 1, dtype=torch.bool)
        self.is_double_buffered = is_double_buffered
        self._nbuffers = 2 if is_double_buffered else 1
        self._num_envs = num_envs
        assert (self._num_envs % self._nbuffers) == 0
        self.num_steps = numsteps
        self.current_rollout_step_idxs = [0 for _ in range(self._nbuffers)]
        self.device = torch.device("cpu")
        self._adv = None  # advantages + stats written by the fused kernel in compute_returns
        self._adv_stats = None
        self._adv_valid = False

    @property
    def current_rollout_step_idx(self) -> int:
        assert all(s == self.current_rollout_step_idxs[0] for s in self.current_rollout_step_idxs)
        return self.current_rollout_step_idxs[0]

    def to(self, device):
        self.buffers.map_in_place(lambda v: v.to(device))
        self.device = torch.device(device)
        self._adv = None

    def insert(self, next_observations=None, next_recurrent_hidden_states=None, actions=None, action_log_probs=None,
               value_preds=None, rewards=None, next_masks=None, buffer_index: int = 0, **kwargs):
        if not self.is_double_buffered:
            assert buffer_index == 0
        next_step = dict(observations=next_observations, recurrent_hidden_states=next_recurrent_hidden_states,
                         prev_actions=actions, masks=next_masks)
        current_step = dict(actions=actions, action_log_probs=action_log_probs, value_preds=value_preds,
                            rewards=rewards)
        next_step = {k: v for k, v in next_step.items() if v is not None}
        current_step = {k: v for k, v in current_step.items() if v is not None}
        env_slice = slice(int(buffer_index * self._num_envs / self._nbuffers),
                          int((buffer_index + 1) * self._num_envs / self._nbuffers))
        if len(next_step) > 0:
            self.buffers.set((self.current_rollout_step_idxs[buffer_index] + 1, env_slice), next_step, strict=False)
        if len(current_step) > 0:
            self.buffers.set((self.current_rollout_step_idxs[buffer_index], env_slice), current_step, strict=False)
        self._adv_valid = False

    def advance_rollout(self, buffer_index: int = 0):
        self.current_rollout_step_idxs[buffer_index] += 1

    def after_update(self):
        self.buffers[0] = self.buffers[self.current_rollout_step_idx]
        self.current_rollout_step_idxs = [0 for _ in self.current_rollout_step_idxs]
        self._adv_valid = False

    def compute_returns(self, next_value, use_gae, gamma, tau):
        """One kernel launch instead of ~8 x T tiny ones (rollout_storage.py:174-205); the same
        launch also produces returns - value_preds over the whole buffer and its finite-entry
        statistics for PPO.get_advantages (rl/ppo/ppo.py:139-157)."""
        b = self.buffers
        if self.device.type != "cuda":
            raise ops._lib.Hb200Error("RolloutStorage.compute_returns: buffers must be on a CUDA device")
        if self._adv is None:
            self._adv = torch.empty_like(b["returns"])
            self._adv_stats = torch.zeros(4, dtype=torch.float64, device=self.device)
        nv = next_value.reshape(-1).to(torch.float32).contiguous()
        ops.gae_adv(b["rewards"], b["value_preds"], b["masks"], nv, b["returns"], self._adv, self._adv_stats,
                    self.current_rollout_step_idx, gamma, tau, use_gae)
        self._adv_valid = True

    def fused_advantages(self):
        """(advantages, stats) from the last compute_returns, or None if buffers changed since."""
        return (self._adv, self._adv_stats) if self._adv_valid else None

    def data_generator(self, advantages: Optional[torch.Tensor], num_mini_batch: int) -> Iterator[dict]:
        num_environments = self.buffers["returns"].size(1)
        assert num_environments >= num_mini_batch, (
            "Trainer requires the number of environments ({}) to be greater than or equal to the number of "
            "trainer mini batches ({}).".format(num_environments, num_mini_batch))
        if num_environments % num_mini_batch != 0:
            warnings.warn("Number of environments ({}) is not a multiple of the number of mini batches ({}).  This "
                          "results in mini batches of different sizes, which can harm training performance.".format(
                              num_environments, num_mini_batch))
        T = self.current_rollout_step_idx
        N = self._num_envs
        b = self.buffers
        # same env split as the reference: CPU RNG randperm, chunked (rollout_storage.py:236)
        for inds in torch.randperm(num_environments).chunk(num_mini_batch):
            inds_d = inds.to(self.device)
            n = inds.numel()
            # buffer row of frame (t, j) is t*N + inds[j]; frames flattened (t, j) like flatten(0, 1)
            rows = (torch.arange(T, device=self.device).view(T, 1) * N + inds_d.view(1, n)).reshape(-1).int()
            small = lambda v: v[0:T, inds_d].flatten(0, 1)  # noqa: E731  (small tensors only)
            batch = {k: small(b[k]) for k in ("rewards", "value_preds", "returns", "action_log_probs", "actions",
                                               "prev_actions", "masks")}
            if advantages is not None:
                batch["advantages"] = small(advantages)
            batch["recurrent_hidden_states"] = b["recurrent_hidden_states"][0, inds_d]
            flat_obs = {k: v.view(-1, *v.shape[2:]) for k, v in b["observations"].items()}
            batch["observations"] = RolloutObservations(flat_obs, rows)
            batch["env_inds"] = inds
            batch["rnn_build_seq_info"] = None  # the masked recurrence needs no packing metadata
            yield batch

    def insert_first_observations(self, batch):
        self.buffers["observations"][0] = batch

    def get_current_step(self, env_slice, buffer_index):
        return self.buffers[self.current_rollout_step_idxs[buffer_index], env_slice]

    def get_last_step(self):
        return self.buffers[self.current_rollout_step_idx]
