"""VERTrainer ("ver"): Variable Experience Rollout (habitat-baselines/habitat_baselines/rl/ver/ver_trainer.py) on the
hb200 classes.

The reference runs environment workers, inference workers and a report worker as processes.  Here the synthetic
environments are born on the device, so collection runs in the trainer process with the inference worker's
bookkeeping (rl/ver/inference_worker.py:219-450): act on the environments whose step has completed, write their steps
at the storage's `ptr`, stop at `num_steps_to_collect`, replay the last batch's steps with the new policy, and bump
the policy version after each update.  Which environments have completed a step comes from the synthetic
environment's virtual clock (`habitat.synthetic.step_time_spread`): with a spread, fast environments contribute more
steps to a rollout than slow ones, and the storage's importance weights correct for it.
"""
from __future__ import annotations

import time
from typing import Dict

import numpy as np
import torch

from ..common.baseline_registry import baseline_registry
from ..common.obs_transformers import get_active_obs_transforms
from ..common.tensor_dict import TensorDict
from ..common.ver_rollout_storage import VERRolloutStorage
from .ppo_trainer import PPOTrainer


@baseline_registry.register_trainer(name="ver")
class VERTrainer(PPOTrainer):
    # environments whose steps complete within this many time units of the earliest one are acted on together (the
    # reference's inference worker waits up to half its average step time to batch requests)
    BATCH_WINDOW = 0.5

    def _check_supported(self):
        hb = self.config.habitat_baselines
        ver = hb.rl.ver
        if ver.overlap_rollouts_and_learn:
            raise NotImplementedError("VER with overlap_rollouts_and_learn=True is not implemented")
        world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
        if world > 1 or getattr(hb.rl.ddppo, "force_distributed", False):
            raise NotImplementedError("distributed VER (it needs the preemption decider) is not implemented")
        if not getattr(hb.rl.ddppo, "train_encoder", True):
            raise NotImplementedError("VER with a frozen visual encoder (train_encoder=False) is not implemented")
        if get_active_obs_transforms(self.config):
            raise NotImplementedError("VER with observation transforms is not implemented: the fused transform writes "
                                      "the next step's [t + 1] slot, which VER's flat storage does not have")

    def _rollouts_factory(self):
        ver = self.config.habitat_baselines.rl.ver
        ppo_cfg = self.config.habitat_baselines.rl.ppo

        def create(device, **kwargs):
            r = VERRolloutStorage(ppo_cfg.num_steps, self.envs.num_envs, self._env_spec.observation_space,
                                  self._env_spec.action_space, self._agent.actor_critic,
                                  variable_experience=ver.variable_experience)
            r.to(device)
            return r
        return create

    def _init_train(self):
        self._check_supported()
        super()._init_train()
        n, dev = self.envs.num_envs, self.device
        self._variable_experience = self.config.habitat_baselines.rl.ver.variable_experience
        # what each environment last reported: observation, the reward of its last action, mask, episode and step ids
        obs = self.envs.reset()
        self._tx = TensorDict.from_tree(dict(
            observations=obs, rewards=torch.zeros(n, 1, device=dev), masks=torch.zeros(n, 1, dtype=torch.bool,
                                                                                      device=dev),
            episode_ids=torch.zeros(n, 1, dtype=torch.int64, device=dev),
            step_ids=torch.zeros(n, 1, dtype=torch.int64, device=dev),
            environment_ids=torch.arange(n, device=dev).view(n, 1)))
        self._now = 0.0
        self._ready_at = np.full(n, np.inf)     # completion time of each environment's step in flight
        self._new_reqs = list(range(n))
        self._replay_reqs = []
        self._n_replay_steps = 0

    # -- the inference worker's step (inference_worker.py:219-417), for the environments in self._new_reqs
    def _policy_step(self) -> int:
        r = self.rollouts
        if self._variable_experience:
            self._new_reqs.sort(key=lambda e: (r.actor_steps_collected[e], e))
            ptr = int(r.ptr[0])
            num = min(int(r.num_steps_to_collect - r.num_steps_collected[0]), len(self._new_reqs))
            r.ptr[:] = ptr + num
            self._replay_reqs += self._new_reqs[num:]
            self._new_reqs = self._new_reqs[:num]
        else:
            num = len(self._new_reqs)
            if np.any(r.current_steps[self._new_reqs] > r.num_steps):
                raise RuntimeError("VERTrainer: an environment stepped past num_steps")
        r.num_steps_collected += num - self._n_replay_steps
        final = int(r.num_steps_collected[0]) == r.num_steps_to_collect
        if final:
            r.rollout_done[:] = True
        reqs = self._new_reqs
        self._new_reqs = []
        if num == 0:
            return 0
        idx = torch.as_tensor(reqs, device=self.device)
        step = self._tx[idx]
        hidden = r.next_hidden_states[idx]
        prev_actions = r.next_prev_actions[idx]
        t0 = time.perf_counter()
        ad = self.actor_critic.act(dict(step["observations"]), hidden, prev_actions, step["masks"])
        self.timings["act"] += time.perf_counter() - t0
        if not final:
            r.next_hidden_states[idx] = ad.rnn_hidden_states
            r.next_prev_actions[idx] = ad.actions
        current = dict(masks=step["masks"], observations=step["observations"], actions=ad.actions,
                       action_log_probs=ad.action_log_probs, recurrent_hidden_states=hidden, prev_actions=prev_actions,
                       policy_version=r.current_policy_version.expand(num, 1), episode_ids=step["episode_ids"],
                       environment_ids=step["environment_ids"], step_ids=step["step_ids"], value_preds=ad.values,
                       returns=torch.full((num, 1), float("nan"), device=self.device))
        b = r.buffers
        if self._variable_experience:
            prev = r.prev_inds[reqs]
            r.prev_inds[reqs] = np.arange(ptr, ptr + num)
            has_prev = prev >= 0   # the reward of each environment's previous action belongs to its previous step
            if has_prev.any():
                b["rewards"][torch.as_tensor(prev[has_prev], device=self.device)] = \
                    step["rewards"][torch.as_tensor(np.nonzero(has_prev)[0], device=self.device)]
            rows = torch.arange(ptr, ptr + num, device=self.device)
        else:
            cur = torch.as_tensor(r.current_steps[reqs], device=self.device)
            ok = cur >= 1
            b["rewards"][cur[ok] - 1, idx[ok]] = step["rewards"][ok]
            rows = (cur, idx)
        self._write(b, rows, current)
        r.actor_steps_collected[reqs] += 1
        r.current_steps[reqs] += 1
        to_step = []
        for e in reqs:
            done_for_env = final if self._variable_experience else r.current_steps[e] == r.num_steps + 1
            (self._replay_reqs if done_for_env else to_step).append(e)
        if to_step:
            sel = [reqs.index(e) for e in to_step]
            self._env_step(to_step, ad.env_actions[sel])
        self._n_replay_steps = 0
        return num

    @staticmethod
    def _write(buffers, rows, values):
        for k, v in values.items():
            if isinstance(v, dict):
                VERTrainer._write(buffers[k], rows, v)
            else:
                buffers[k][rows] = v.reshape(buffers[k][rows].shape).to(buffers[k].dtype)

    def _env_step(self, envs, actions):
        """Start the next step of `envs`: its result is what they report once the virtual clock reaches it."""
        if self._action_bounds is not None:   # the environment gets the clipped action, the storage the sampled one
            actions = torch.clamp(actions, *self._action_bounds)
        k = len(envs)
        idx = torch.as_tensor(envs, device=self.device)
        obs, rewards, dones, _ = self.envs.step(actions, n=k)
        dones = dones.view(k, 1)
        cur = self.current_episode_reward
        cur[idx] += rewards
        self.running_episode_stats["reward"][idx] += torch.where(dones, cur[idx], torch.zeros_like(rewards))
        self.running_episode_stats["count"][idx] += dones.float()
        cur[idx] = cur[idx].masked_fill(dones, 0.0)
        tx = self._tx
        for key, v in obs.items():
            tx["observations"][key][idx] = v
        tx["rewards"][idx] = rewards
        tx["masks"][idx] = ~dones
        tx["episode_ids"][idx] += dones.long()
        tx["step_ids"][idx] = torch.where(dones, torch.zeros_like(tx["step_ids"][idx]), tx["step_ids"][idx] + 1)
        self._ready_at[envs] = self._now + self.envs.step_durations(k)

    def _wait_for_steps(self):
        """Advance the virtual clock to the next completed step; those completing within BATCH_WINDOW join it."""
        self._now = float(np.min(self._ready_at))
        done = np.nonzero(self._ready_at <= self._now + self.BATCH_WINDOW)[0]
        self._ready_at[done] = np.inf
        self._new_reqs += done.tolist()

    def _collect_rollout(self) -> int:
        """Returns the new environment steps of the rollout: num_steps_collected, which leaves out the replayed steps
        (each was counted in the rollout that first collected it)."""
        r = self.rollouts
        while not r.rollout_done[0]:
            if not self._new_reqs:
                self._wait_for_steps()
            self._policy_step()
        # finish_rollout (inference_worker.py:419-452): unprocessed and final-batch steps are replayed next rollout
        self._new_reqs = self._replay_reqs + self._new_reqs
        self._replay_reqs = []
        self._n_replay_steps = len(self._new_reqs)
        r.will_replay_step[self._new_reqs] = True
        return int(r.num_steps_collected[0])

    def _update_agent(self) -> Dict[str, float]:
        """compute_returns -> update -> after_update -> policy version + 1 (ver_trainer.py:377-427)."""
        ppo_cfg = self.config.habitat_baselines.rl.ppo
        r = self.rollouts
        t0 = time.perf_counter()
        r.compute_returns(ppo_cfg.use_gae, ppo_cfg.gamma, ppo_cfg.tau)
        self._agent.train()
        losses = self._agent.updater.update(r)
        r.after_update()
        r.increment_policy_version()
        self._agent.after_update()
        self.timings["learn"] += time.perf_counter() - t0
        return losses

    def train(self) -> Dict[str, float]:
        self._init_train()
        losses = {}
        while not self.is_done():
            self._agent.pre_rollout()
            self._agent.eval()
            t0 = time.perf_counter()
            count_steps_delta = self._collect_rollout()
            torch.cuda.synchronize()
            self.timings["rollout"] += time.perf_counter() - t0
            self.rollouts.after_rollout()
            losses = self._update_agent()
            torch.cuda.synchronize()
            self.num_updates_done += 1
            losses = self._coalesce_post_step(losses, count_steps_delta)
            if self.should_checkpoint():
                self.save_checkpoint(f"ckpt.{self.num_updates_done}.pth", dict(step=self.num_steps_done))
            self._last_fps = self.num_steps_done / max(time.time() - self.t_start, 1e-9)
        self.envs.close()
        return losses
