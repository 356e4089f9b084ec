"""PPOTrainer ("ppo" / "ddppo") on the hb200 classes: the rollout loop, DD-PPO's preemption rule,
`_update_agent` and the post-update coalescing of habitat-baselines' trainer
(habitat-baselines/habitat_baselines/rl/ppo/ppo_trainer.py:172-292, 343-557, 641-801), with the
simulator replaced by an in-process synthetic VectorEnv that hands back DEVICE-resident observations
(the drop-in seam is `vector_env_factory._target_`, SURVEY.md section 8b).

The config is attribute-style (OmegaConf / SimpleNamespace / the dataclasses below) with the
reference's field names, so a Hydra-composed `habitat_baselines` config is accepted unchanged.
"""
from __future__ import annotations

import collections
import math
import time
from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import Dict, Optional

import numpy as np
import torch

from ..common import spaces
from ..common.baseline_registry import baseline_registry
from ..common.obs_transformers import ObsTransformPlan, apply_obs_transforms_obs_space, get_active_obs_transforms
from ..common.rollout_storage import RolloutStorage
from ..common.tensor_dict import TensorDict
from ..synthetic import cubemap_spaces, fill_image_, pointnav_spaces
import os

from .ppo import DDPPO, PPO  # noqa: F401  (registers the updaters)
from . import policy as _policy  # noqa: F401  (registers PointNavBaselinePolicy)
from .resnet_policy import VISUAL_FEATURES_KEY, ActionDistributionConfig, PointNavResNetPolicy  # noqa: F401
from .single_agent_access_mgr import SingleAgentAccessMgr


# ---- config (field names and defaults: habitat_baselines/config/default_structured_configs.py:288-363) ----
@dataclass
class PPOConfig:
    clip_param: float = 0.2
    ppo_epoch: int = 4
    num_mini_batch: int = 2
    value_loss_coef: float = 0.5
    entropy_coef: float = 0.01
    lr: float = 2.5e-4
    eps: float = 1e-5
    max_grad_norm: float = 0.5
    num_steps: int = 5
    use_gae: bool = True
    use_linear_lr_decay: bool = False
    use_linear_clip_decay: bool = False
    gamma: float = 0.99
    tau: float = 0.95
    reward_window_size: int = 50
    use_normalized_advantage: bool = False
    hidden_size: int = 512
    entropy_target_factor: float = 0.0
    use_adaptive_entropy_pen: bool = False
    use_clipped_value_loss: bool = True
    use_double_buffered_sampler: bool = False


@dataclass
class DDPPOConfig:
    sync_frac: float = 0.6
    distrib_backend: str = "NCCL"
    rnn_type: str = "LSTM"
    num_recurrent_layers: int = 2
    backbone: str = "resnet18"
    pretrained_weights: str = "data/ddppo-models/gibson-2plus-resnet50.pth"
    pretrained: bool = False           # load the whole policy from pretrained_weights
    pretrained_encoder: bool = False   # load only the visual encoder from pretrained_weights
    train_encoder: bool = True         # False: freeze the visual encoder and cache its output in the rollout
    reset_critic: bool = True          # re-draw the critic head after loading pretrained weights
    force_distributed: bool = False


@dataclass
class VERConfig:
    variable_experience: bool = True
    num_inference_workers: int = 2
    overlap_rollouts_and_learn: bool = False


def make_config(num_environments=4, total_num_steps=-1.0, num_updates=2, height=256, width=256, seed=100,
                obs_transforms=None, ddppo=None, continuous_actions=0, action_dist=None, trainer_name="ddppo",
                ver=None, step_time_spread=0.0, cubemap=None, **ppo_kw):
    """A habitat_baselines-shaped config for the synthetic PointNav DD-PPO run (ddppo_pointnav.yaml values).
    obs_transforms: {name: config node with `type` and the transformer's fields} (e.g. the ObjectNav YAMLs'
    resize_shortest_edge + center_cropper, common/obs_transformers.py); height / width are then the raw sensor size.
    ddppo: DDPPOConfig field overrides, e.g. dict(pretrained=True, pretrained_weights=path, train_encoder=False).
    continuous_actions = A > 0: continuous control -- a Box(-1, 1, (A,)) action space and the gaussian policy
    (monolithic.yaml), with action_dist the ActionDistributionConfig field overrides (e.g. social_nav.yaml's
    dict(use_std_param=True)).
    trainer_name="ver": Variable Experience Rollout (rl/ver_trainer.py) with `ver` the VERConfig field overrides;
    step_time_spread > 0 gives every synthetic environment step its own duration on a seeded virtual clock, so
    environments contribute unequal numbers of steps to a rollout.
    cubemap="rgb" / "depth": the synthetic environment is a cube-map rig (synthetic.cubemap_spaces) of six height x
    height faces `{cubemap}_0` .. `{cubemap}_5`, for CubeMap2Equirect / CubeMap2Fisheye."""
    ppo = PPOConfig(**{**dict(ppo_epoch=2, num_mini_batch=2, num_steps=128, max_grad_norm=0.2), **ppo_kw})
    agent = SimpleNamespace(name="PointNavResNetPolicy", action_distribution_type="categorical")
    if continuous_actions:
        agent.action_distribution_type = "gaussian"
        agent.action_dist = ActionDistributionConfig(**(action_dist or {}))
    if obs_transforms is not None:
        agent.obs_transforms = dict(obs_transforms)
    hb = SimpleNamespace(
        trainer_name=trainer_name, updater_name="PPO", distrib_updater_name="DDPPO", rollout_storage_name="RolloutStorage",
        num_environments=num_environments, total_num_steps=total_num_steps, num_updates=num_updates,
        log_interval=10, force_blind_policy=False, num_checkpoints=-1, checkpoint_interval=-1,
        checkpoint_folder="data/checkpoints",
        rl=SimpleNamespace(ppo=ppo, ddppo=DDPPOConfig(**(ddppo or {})), policy={"main_agent": agent},
                           ver=VERConfig(**(ver or {}))),
        eval=SimpleNamespace(extra_sim_sensors={}),
    )
    habitat = SimpleNamespace(seed=seed, simulator=SimpleNamespace(agents_order=["main_agent"]),
                              synthetic=SimpleNamespace(height=height, width=width, p_done=1.0 / 250.0,
                                                        continuous_actions=int(continuous_actions),
                                                        step_time_spread=float(step_time_spread),
                                                        cubemap=cubemap))
    return SimpleNamespace(habitat_baselines=hb, habitat=habitat)


# torch dtype of each image dtype a synthetic camera can have
_IMAGE_DTYPE = {np.dtype(np.uint8): torch.uint8, np.dtype(np.float32): torch.float32, np.dtype(np.int32): torch.int32}


# ---- synthetic VectorEnv ------------------------------------------------------------------------------
class SyntheticVectorEnv:
    """VectorEnv-shaped source of synthetic RGB-D PointNav observations born on the device
    (method surface: habitat/core/vector_env.py as used by ppo_trainer.py:136-157, 266-267, 388, 409-419)."""

    def __init__(self, num_envs, obs_space, act_space, device, seed, p_done, step_time_spread=0.0):
        self.num_envs = num_envs
        self.observation_spaces = [obs_space] * num_envs
        self.action_spaces = [act_space] * num_envs
        self.orig_action_spaces = self.action_spaces
        self.device = device
        self.gen = torch.Generator(device=device).manual_seed(seed)
        self.p_done = p_done
        self._pending = None
        # opt-in: every step of every environment takes 1 + spread * U[0, 1) time units on a virtual clock, drawn from
        # a generator of its own so the observation / reward stream is the same with or without it
        self.step_time_spread = float(step_time_spread)
        self.clock = np.random.default_rng(seed)

    def step_durations(self, n: int) -> np.ndarray:
        if self.step_time_spread <= 0.0:
            return np.ones(n)
        return 1.0 + self.step_time_spread * self.clock.random(n)

    def _obs(self, n=None):
        sp = self.observation_spaces[0].spaces
        out = {}
        n, d, g = self.num_envs if n is None else n, self.device, self.gen
        if "rgb" in sp:
            out["rgb"] = torch.randint(0, 256, (n, *sp["rgb"].shape), generator=g, device=d, dtype=torch.uint8)
        if "depth" in sp:
            out["depth"] = torch.rand((n, *sp["depth"].shape), generator=g, device=d)
        for k, s in sp.items():   # any other camera (the cube-map rig's faces), filled by dtype
            if k not in ("rgb", "depth") and len(s.shape) == 3:
                out[k] = torch.empty((n, *s.shape), dtype=_IMAGE_DTYPE[np.dtype(s.dtype)], device=d)
                fill_image_(out[k], g, d)
        goal = torch.rand(n, 2, generator=g, device=d)
        goal[:, 0] *= 10.0
        goal[:, 1] = goal[:, 1] * 2 * math.pi - math.pi
        out["pointgoal_with_gps_compass"] = goal
        return out

    def reset(self):
        return self._obs()

    def step(self, actions, n=None):
        """Batched step: (obs dict, rewards [N,1], dones [N] bool, infos).  n: step only that many environments (the
        VER trainer steps the ones whose previous step has completed)."""
        n, d, g = self.num_envs if n is None else n, self.device, self.gen
        dones = torch.rand(n, generator=g, device=d) < self.p_done
        rewards = torch.randn(n, 1, generator=g, device=d) * 0.1 + 2.5 * dones.float().view(n, 1)
        return self._obs(n), rewards, dones, [{} for _ in range(n)]

    # -- the per-environment surface the REFERENCE's trainer drives (ppo_trainer.py:388, 409-419, 266-267):
    #    async_step_at(i, a) for every env of a buffer, then wait_step_at(i) -> (obs, reward, done, info), post_step(obs)
    def async_step_at(self, index_env: int, action) -> None:
        if self._pending is None:
            self._pending = {"n": 0, "out": None}
        self._pending["n"] += 1

    def wait_step_at(self, index_env: int):
        if self._pending is None:
            raise RuntimeError("wait_step_at without a matching async_step_at")
        if self._pending["out"] is None:   # the whole batch is generated on the first wait of the round
            self._pending["out"] = self.step(None)
        obs, rewards, dones, infos = self._pending["out"]
        res = ({k: v[index_env] for k, v in obs.items()}, float(rewards[index_env]), bool(dones[index_env]),
               infos[index_env])
        self._pending["n"] -= 1
        if self._pending["n"] <= 0:
            self._pending = None
        return res

    def post_step(self, observations):
        return observations

    def close(self):
        pass


class SyntheticVectorEnvFactory:
    """Drop-in for `habitat_baselines.vector_env_factory._target_` (common/env_factory.py contract)."""

    def construct_envs(self, config, workers_ignore_signals=False, enforce_scenes_greater_eq_environments=False,
                       is_first_rank=True, device=None, rank=0):
        syn = config.habitat.synthetic
        if getattr(syn, "cubemap", None):
            obs_space, act_space = cubemap_spaces(syn.height, syn.cubemap)
        else:
            obs_space, act_space = pointnav_spaces(syn.height, syn.width)
        if getattr(syn, "continuous_actions", 0):   # the environment draws no random numbers for its actions
            act_space = spaces.Box(-1.0, 1.0, (syn.continuous_actions,), np.float32)
        n = config.habitat_baselines.num_environments
        return SyntheticVectorEnv(n, obs_space, act_space, device, config.habitat.seed + rank * n, syn.p_done,
                                  getattr(syn, "step_time_spread", 0.0))


# ---- the trainer -------------------------------------------------------------------------------------------
@baseline_registry.register_trainer(name="ddppo")
@baseline_registry.register_trainer(name="ppo")
class PPOTrainer:
    SHORT_ROLLOUT_THRESHOLD: float = 0.25  # ppo_trainer.py:78

    def __init__(self, config=None):
        self.config = config
        self.num_updates_done = 0
        self.num_steps_done = 0
        self._is_distributed = torch.distributed.is_available() and torch.distributed.is_initialized()
        self._last_fps = 0.0
        self._is_static_encoder = False
        self.timings = collections.defaultdict(float)

    # -- helpers mirroring BaseRLTrainer (common/base_trainer.py:226-267)
    def percent_done(self) -> float:
        hb = self.config.habitat_baselines
        if hb.num_updates != -1:
            return self.num_updates_done / hb.num_updates
        return self.num_steps_done / hb.total_num_steps

    def is_done(self) -> bool:
        return self.percent_done() >= 1.0

    def _all_reduce(self, t: torch.Tensor) -> torch.Tensor:
        if not self._is_distributed:
            return t
        orig = t.device
        t = t.to(self.device)
        torch.distributed.all_reduce(t)
        return t.to(orig)

    def _init_train(self):
        cfg = self.config
        hb = cfg.habitat_baselines
        ppo_cfg = hb.rl.ppo
        self._is_distributed = (torch.distributed.is_available() and torch.distributed.is_initialized()) or \
            getattr(hb.rl.ddppo, "force_distributed", False)
        rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
        self.device = torch.device("cuda", torch.cuda.current_device())
        # seed offset per rank (ppo_trainer.py:207-215)
        seed = cfg.habitat.seed + rank * hb.num_environments
        torch.manual_seed(seed)
        np.random.seed(seed)
        if torch.distributed.is_initialized():
            # the same TCPStore doubles as the preemption counter (ppo_trainer.py:216-219, 553, 776)
            store = torch.distributed.distributed_c10d._get_default_store()
            self.num_rollouts_done_store = torch.distributed.PrefixStore("rollout_tracker", store)
            if rank == 0:
                self.num_rollouts_done_store.set("num_done", "0")
            torch.distributed.barrier()
        self.envs = SyntheticVectorEnvFactory().construct_envs(cfg, device=self.device, rank=rank)
        obs_space, act_space = self.envs.observation_spaces[0], self.envs.action_spaces[0]
        # policy + updater + storage are owned by the agent access manager, built from the registry names in the config
        # (ppo_trainer.py:122-134, 246-259)
        self._env_spec = SimpleNamespace(observation_space=obs_space, action_space=act_space,
                                         orig_action_space=self.envs.orig_action_spaces[0])
        self._create_obs_transforms()
        self._action_bounds = None
        if spaces.continuous_action_dim(act_space) is not None:
            self._action_bounds = tuple(torch.as_tensor(b, dtype=torch.float32, device=self.device)
                                        for b in (act_space.low, act_space.high))
        self._agent = self._create_agent(None)
        if torch.distributed.is_initialized():
            self._agent.init_distributed(find_unused_params=False)
        self._agent.post_init(self._rollouts_factory())
        obs = self.envs.reset()
        if self._obs_plan:
            rest = self._obs_plan.apply_(obs, self.rollouts.buffers["observations"][0])
            self.rollouts.buffers["observations"].set(0, TensorDict.from_tree(rest), strict=False)
        elif self._agent.is_static_encoder:   # VISUAL_FEATURES_KEY is written below
            self.rollouts.buffers["observations"].set(0, TensorDict.from_tree(obs), strict=False)
        else:
            self.rollouts.insert_first_observations(TensorDict.from_tree(obs))
        # frozen encoder: still in training mode here, so this first call updates RunningMeanAndVar -- the only update
        # it ever gets, since rollouts run in eval mode and the learner never calls the encoder (ppo_trainer.py:261-279)
        self._is_static_encoder = self._agent.is_static_encoder
        if self._is_static_encoder:
            self._encode_visual_features(0)
        n = self.envs.num_envs
        self.current_episode_reward = torch.zeros(n, 1, device=self.device)
        self.running_episode_stats = dict(count=torch.zeros(n, 1, device=self.device),
                                          reward=torch.zeros(n, 1, device=self.device))
        self.window_episode_stats = collections.defaultdict(lambda: collections.deque(maxlen=ppo_cfg.reward_window_size))
        self._last_checkpoint_percent = -1.0
        self.t_start = time.time()

    def _encode_visual_features(self, slot: int) -> None:
        """The frozen main encoder on the observations of storage slot `slot` (batch N, after the observation transforms
        wrote them), its output written straight into that slot's VISUAL_FEATURES_KEY (ppo_trainer.py:467-471)."""
        obs = self.rollouts.buffers["observations"]
        t0 = time.perf_counter()
        self.actor_critic.encode_visual_features(obs[slot], obs[VISUAL_FEATURES_KEY][slot])
        self.timings["visual_features"] += time.perf_counter() - t0

    def _rollouts_factory(self):
        """create_rollouts_fn for SingleAgentAccessMgr.post_init: None builds the configured rollout storage."""
        return None

    def _create_obs_transforms(self):
        """ppo_trainer.py:110-113: the policy and the storage are built for the transformed observation space.  The
        active transforms run fused (ObsTransformPlan): one launch per env step writes the transformed keys straight
        into the rollout storage's next slot."""
        raw_space = self._env_spec.observation_space
        self.obs_transforms = get_active_obs_transforms(self.config)
        self._env_spec.observation_space = apply_obs_transforms_obs_space(raw_space, self.obs_transforms)
        self._obs_plan = ObsTransformPlan(self.obs_transforms, raw_space)

    def _create_agent(self, resume_state, **kwargs) -> SingleAgentAccessMgr:
        """ppo_trainer.py:122-134"""
        agent = SingleAgentAccessMgr(config=self.config, env_spec=self._env_spec, is_distrib=torch.distributed.is_initialized(),
                                     device=self.device, percent_done_fn=self.percent_done, **kwargs)
        if resume_state is not None:
            agent.load_state_dict(resume_state)
        return agent

    # the attributes round-1 callers (tests, bench) read
    @property
    def actor_critic(self):
        return self._agent.actor_critic

    @property
    def updater(self):
        return self._agent.updater

    @property
    def rollouts(self):
        return self._agent.rollouts

    # -- checkpoints (common/base_trainer.py:269-287, ppo_trainer.py:296-341)
    def should_checkpoint(self) -> bool:
        hb = self.config.habitat_baselines
        if getattr(hb, "num_checkpoints", -1) != -1:
            every = 1 / hb.num_checkpoints
            if self._last_checkpoint_percent + every < self.percent_done():
                self._last_checkpoint_percent = self.percent_done()
                return True
            return False
        interval = getattr(hb, "checkpoint_interval", -1)
        return interval > 0 and (self.num_updates_done % interval) == 0

    def save_checkpoint(self, file_name: str, extra_state: Optional[Dict] = None) -> None:
        ckpt = {**self._agent.get_save_state(), "config": self.config}
        if extra_state is not None:
            ckpt["extra_state"] = extra_state
        folder = self.config.habitat_baselines.checkpoint_folder
        os.makedirs(folder, exist_ok=True)
        torch.save(ckpt, os.path.join(folder, file_name))
        torch.save(ckpt, os.path.join(folder, "latest.pth"))

    def load_checkpoint(self, checkpoint_path: str, *args, **kwargs) -> Dict:
        return torch.load(checkpoint_path, *args, weights_only=False, **kwargs)

    def get_resume_state(self) -> Dict:
        """what ppo_trainer.py:707-726 hands to save_resume_state"""
        return dict(**self._agent.get_resume_state(), config=self.config,
                    requeue_stats=dict(num_steps_done=self.num_steps_done, num_updates_done=self.num_updates_done,
                                       _last_checkpoint_percent=self._last_checkpoint_percent,
                                       running_episode_stats=self.running_episode_stats,
                                       window_episode_stats=dict(self.window_episode_stats)))

    # -- one environment step for all envs (ppo_trainer.py:343-482, batched: observations never leave the GPU)
    def _rollout_step(self):
        r = self.rollouts
        step = r.get_current_step(slice(0, self.envs.num_envs), 0)
        t0 = time.perf_counter()
        ad = self.actor_critic.act(step["observations"], step["recurrent_hidden_states"], step["prev_actions"],
                                   step["masks"])
        self.timings["act"] += time.perf_counter() - t0
        env_actions = ad.env_actions
        if self._action_bounds is not None:   # ppo_trainer.py:379-385: the env gets the clipped action, storage not
            env_actions = torch.clamp(env_actions, *self._action_bounds)
        obs, rewards, dones, _ = self.envs.step(env_actions)
        not_done = (~dones).view(-1, 1)
        self.current_episode_reward += rewards
        self.running_episode_stats["reward"] += torch.where(not_done, torch.zeros_like(rewards), self.current_episode_reward)
        self.running_episode_stats["count"] += (~not_done).float()
        self.current_episode_reward.masked_fill_(~not_done, 0.0)
        if self._obs_plan:   # transformed keys go straight into slot t + 1; insert copies the rest
            obs = self._obs_plan.apply_(obs, r.buffers["observations"][r.current_rollout_step_idxs[0] + 1])
        r.insert(next_observations=TensorDict.from_tree(obs), next_recurrent_hidden_states=ad.rnn_hidden_states,
                 actions=ad.actions, action_log_probs=ad.action_log_probs, value_preds=ad.values, rewards=rewards,
                 next_masks=not_done)
        if self._is_static_encoder:
            self._encode_visual_features(r.current_rollout_step_idxs[0] + 1)
        r.advance_rollout()
        return self.envs.num_envs

    def should_end_early(self, rollout_step) -> bool:
        """DD-PPO straggler preemption (ppo_trainer.py:641-653)."""
        if not (self._is_distributed and torch.distributed.is_initialized()):
            return False
        hb = self.config.habitat_baselines
        return rollout_step >= hb.rl.ppo.num_steps * self.SHORT_ROLLOUT_THRESHOLD and \
            int(self.num_rollouts_done_store.get("num_done")) >= hb.rl.ddppo.sync_frac * torch.distributed.get_world_size()

    def _update_agent(self) -> Dict[str, float]:
        """get_value -> compute_returns -> update -> after_update (ppo_trainer.py:489-522)."""
        ppo_cfg = self.config.habitat_baselines.rl.ppo
        r = self.rollouts
        t0 = time.perf_counter()
        last = r.get_last_step()
        next_value = self.actor_critic.get_value(last["observations"], last["recurrent_hidden_states"],
                                                 last["prev_actions"], last["masks"])
        r.compute_returns(next_value, ppo_cfg.use_gae, ppo_cfg.gamma, ppo_cfg.tau)
        self._agent.train()
        losses = self._agent.updater.update(r)
        r.after_update()
        self._agent.after_update()   # LambdaLR(1 - percent_done) step + updater.after_update (ppo_trainer.py:519-521)
        self.timings["learn"] += time.perf_counter() - t0
        return losses

    def _coalesce_post_step(self, losses: Dict[str, float], count_steps_delta: int) -> Dict[str, float]:
        """ppo_trainer.py:524-557: two packed all-reduces; rank 0 resets the preemption counter."""
        order = sorted(self.running_episode_stats.keys())
        stats = self._all_reduce(torch.stack([self.running_episode_stats[k] for k in order], 0))
        for i, k in enumerate(order):
            self.window_episode_stats[k].append(stats[i].clone())
        if self._is_distributed and torch.distributed.is_initialized():
            names = sorted(losses.keys())
            vec = torch.tensor([losses[k] for k in names] + [count_steps_delta], dtype=torch.float32)
            vec = self._all_reduce(vec)
            count_steps_delta = int(vec[-1].item())
            vec /= torch.distributed.get_world_size()
            losses = {k: vec[i].item() for i, k in enumerate(names)}
            if torch.distributed.get_rank() == 0:
                self.num_rollouts_done_store.set("num_done", "0")
        self.num_steps_done += count_steps_delta
        return losses

    def train(self) -> Dict[str, float]:
        self._init_train()
        ppo_cfg = self.config.habitat_baselines.rl.ppo
        losses = {}
        while not self.is_done():
            self._agent.pre_rollout()   # linear clip decay, evaluated AFTER the previous update's increment (:705)
            self._agent.eval()
            count_steps_delta = 0
            t0 = time.perf_counter()
            for step in range(ppo_cfg.num_steps):
                count_steps_delta += self._rollout_step()
                if self.should_end_early(step + 1):
                    break
            torch.cuda.synchronize()
            self.timings["rollout"] += time.perf_counter() - t0
            if self._is_distributed and torch.distributed.is_initialized():
                self.num_rollouts_done_store.add("num_done", 1)
            losses = self._update_agent()
            torch.cuda.synchronize()
            self.num_updates_done += 1
            losses = self._coalesce_post_step(losses, count_steps_delta)
            if self.should_checkpoint():
                self.save_checkpoint(f"ckpt.{self.num_updates_done}.pth", dict(step=self.num_steps_done))
            self._last_fps = self.num_steps_done / max(time.time() - self.t_start, 1e-9)
        self.envs.close()
        return losses


from . import ver_trainer  # noqa: E402,F401  (registers the "ver" trainer)
