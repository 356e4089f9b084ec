"""SingleAgentAccessMgr: owns policy + updater + storage, built from the registry names in the config
(habitat-baselines/habitat_baselines/rl/ppo/single_agent_access_mgr.py:40-319), including the LambdaLR
linear decay, the clip decay of `pre_rollout`, the checkpoint / resume state dict layouts, and fine-tuning from a
pretrained checkpoint with an optionally frozen visual encoder (`rl.ddppo.pretrained*`, `train_encoder`,
`reset_critic`; :205-237, 300-319)."""
from __future__ import annotations

from typing import Any, Callable, Dict, Optional

import numpy as np
import torch
from torch import nn
from torch.optim.lr_scheduler import LambdaLR

from ..common import spaces
from ..common.baseline_registry import baseline_registry
from ..common.rollout_storage import RolloutStorage
from .ppo import DDPPO, PPO
from . import policy as _policy  # noqa: F401  (registers PointNavBaselinePolicy)
from .resnet_policy import VISUAL_FEATURES_KEY, PointNavResNetPolicy

CKPT_PREFIX = "actor_critic."


def linear_lr_schedule(percent_done: float) -> float:
    return 1 - percent_done


def get_rollout_obs_space(obs_space, actor_critic, config):
    """The rollout storage's observation space (single_agent_access_mgr.py:300-319): with a frozen encoder its output
    is stored too, as VISUAL_FEATURES_KEY in front of every raw key."""
    if getattr(config.habitat_baselines.rl.ddppo, "train_encoder", True):
        return obs_space
    box = spaces.Box(low=np.finfo(np.float32).min, high=np.finfo(np.float32).max,
                     shape=actor_critic.visual_encoder.output_shape, dtype=np.float32)
    return spaces.Dict({VISUAL_FEATURES_KEY: box, **obs_space.spaces})


def load_pretrained_state(path):
    """The `state_dict` of a habitat-baselines checkpoint ({"state_dict": {"actor_critic.<key>": tensor}, ...}), loaded
    on the CPU, with the prefix removed.  Keys without the prefix are refused: the reference strips the first
    len("actor_critic.") characters of every key unchecked, which turns a bare policy state_dict into nonsense keys."""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)   # trainer checkpoints also pickle the config
    sd = ckpt.get("state_dict") if isinstance(ckpt, dict) else None
    if not isinstance(sd, dict):
        raise ValueError(f"pretrained_weights {path!r}: expected a checkpoint {{'state_dict': {{'{CKPT_PREFIX}<key>': "
                         "tensor}}}}, found no 'state_dict' mapping")
    bad = [k for k in sd if not k.startswith(CKPT_PREFIX)]
    if bad:
        raise ValueError(f"pretrained_weights {path!r}: every state_dict key must start with {CKPT_PREFIX!r} (the "
                         f"format {{'state_dict': {{'{CKPT_PREFIX}<key>': tensor}}}}); {len(bad)} do not, e.g. "
                         f"{bad[:3]}")
    return {k[len(CKPT_PREFIX):]: v for k, v in sd.items()}


class SingleAgentAccessMgr:
    def __init__(self, config, env_spec, is_distrib: bool, device, percent_done_fn: Callable[[], float],
                 lr_schedule_fn: Optional[Callable[[float], float]] = None, agent_name=None):
        self._env_spec = env_spec          # needs .observation_space, .action_space
        self._config = config
        self._num_envs = config.habitat_baselines.num_environments
        self._device = device
        self._ppo_cfg = config.habitat_baselines.rl.ppo
        self._is_distributed = is_distrib
        self._percent_done_fn = percent_done_fn
        self.agent_name = agent_name if agent_name is not None else config.habitat.simulator.agents_order[0]
        self._is_static_encoder = not getattr(config.habitat_baselines.rl.ddppo, "train_encoder", True)
        self._actor_critic = self._create_policy()
        self._updater = self._create_updater(self._actor_critic)
        if self._updater.optimizer is None:
            self._lr_scheduler = None
        else:
            fn = linear_lr_schedule if lr_schedule_fn is None else lr_schedule_fn
            self._lr_scheduler = LambdaLR(optimizer=self._updater.optimizer, lr_lambda=lambda _: fn(self._percent_done_fn()))
        self._rollouts = None

    def _create_policy(self):
        hb = self._config.habitat_baselines
        dd = hb.rl.ddppo
        cls = baseline_registry.get_policy(hb.rl.policy[self.agent_name].name) or PointNavResNetPolicy
        if self._is_static_encoder:
            if getattr(hb, "force_blind_policy", False):
                raise NotImplementedError("train_encoder=False with a blind policy: there is no visual encoder to freeze")
            if not issubclass(cls, PointNavResNetPolicy):
                raise NotImplementedError(f"train_encoder=False is implemented for PointNavResNetPolicy only, not "
                                          f"{cls.__name__} (SimpleCNN)")
        ac = cls.from_config(self._config, self._env_spec.observation_space, self._env_spec.action_space,
                             agent_name=self.agent_name)
        if self._is_static_encoder and ac.net._goal_encoder_uuids:
            raise NotImplementedError(f"train_encoder=False with an image-goal encoder ({ac.net._goal_encoder_uuids}): "
                                      "that encoder keeps training in the reference; freezing only the main encoder "
                                      "is not implemented")
        loaded = False
        if getattr(dd, "pretrained", False) or getattr(dd, "pretrained_encoder", False):
            pretrained = load_pretrained_state(dd.pretrained_weights)
            if dd.pretrained:
                ac.load_state_dict(pretrained)
            else:   # the visual encoder's entries only, weights and RunningMeanAndVar buffers, strictly
                prefix = "net.visual_encoder."
                enc = {k: v for k, v in pretrained.items() if k.startswith(prefix)}
                want = {prefix + k for k in ac.net.visual_encoder.state_dict()}
                if set(enc) != want:
                    raise RuntimeError(f"pretrained_encoder: visual encoder keys differ from the checkpoint's: missing "
                                       f"{sorted(want - set(enc))[:5]}, unexpected {sorted(set(enc) - want)[:5]}")
                ac.load_state_dict({**ac.state_dict(), **enc})
            loaded = True
        if self._is_static_encoder:
            for p in ac.visual_encoder.parameters():
                p.requires_grad_(False)
        # a freshly built critic is already an orthogonal draw: re-drawing it only matters for loaded weights, and
        # skipping it keeps the seeded initial weights of a run from scratch unchanged
        if getattr(dd, "reset_critic", True) and loaded:
            nn.init.orthogonal_(ac.critic.fc.weight)
            nn.init.constant_(ac.critic.fc.bias, 0)
        return ac.to(self._device)

    def _create_updater(self, actor_critic):
        hb = self._config.habitat_baselines
        name = hb.distrib_updater_name if self._is_distributed else hb.updater_name
        cls = baseline_registry.get_updater(name) or (DDPPO if self._is_distributed else PPO)
        return cls.from_config(actor_critic, self._ppo_cfg)

    def init_distributed(self, find_unused_params: bool = True) -> None:
        if self._is_distributed:
            self._updater.init_distributed(find_unused_params=find_unused_params)

    def post_init(self, create_rollouts_fn: Optional[Callable] = None):
        hb = self._config.habitat_baselines
        cls = baseline_registry.get_storage(hb.rollout_storage_name) or RolloutStorage
        obs_space = get_rollout_obs_space(self._env_spec.observation_space, self._actor_critic, self._config)
        self._rollouts = cls(self._ppo_cfg.num_steps, self._num_envs, obs_space,
                             self._env_spec.action_space, self._actor_critic,
                             is_double_buffered=self._ppo_cfg.use_double_buffered_sampler)
        self._rollouts.to(self._device)

    @property
    def is_static_encoder(self) -> bool:
        """train_encoder=False: the visual encoder is frozen and its output is cached in the rollout storage"""
        return self._is_static_encoder

    @property
    def nbuffers(self):
        return 2 if self._ppo_cfg.use_double_buffered_sampler else 1

    @property
    def rollouts(self):
        return self._rollouts

    @property
    def actor_critic(self):
        return self._actor_critic

    @property
    def updater(self):
        return self._updater

    @property
    def policy_action_space(self):
        return self._actor_critic.policy_action_space

    def train(self):
        self._actor_critic.train()
        self._updater.train()

    def eval(self):
        self._actor_critic.eval()

    def get_resume_state(self) -> Dict[str, Any]:
        ret = {"state_dict": self._actor_critic.state_dict(), **self._updater.get_resume_state()}
        if self._lr_scheduler is not None:
            ret["lr_sched_state"] = self._lr_scheduler.state_dict()
        return ret

    def get_save_state(self):
        return {"state_dict": self._actor_critic.state_dict()}

    def load_ckpt_state_dict(self, ckpt: Dict) -> None:
        self._actor_critic.load_state_dict(ckpt["state_dict"])

    def load_state_dict(self, state: Dict) -> None:
        self._actor_critic.load_state_dict(state["state_dict"])
        if self._updater is not None:
            if "optim_state" in state:
                self._updater.optimizer.load_state_dict(state["optim_state"])
            if "lr_sched_state" in state and self._lr_scheduler is not None:
                self._lr_scheduler.load_state_dict(state["lr_sched_state"])

    def after_update(self):
        if self._ppo_cfg.use_linear_lr_decay and self._lr_scheduler is not None:
            self._lr_scheduler.step()
        self._updater.after_update()   # single_agent_access_mgr.py:291

    def pre_rollout(self):
        if self._ppo_cfg.use_linear_clip_decay:
            self._updater.clip_param = self._ppo_cfg.clip_param * (1 - self._percent_done_fn())
