"""PPO / DDPPO updaters on the hb200 kernels, keeping the reference's interface
(habitat-baselines/habitat_baselines/rl/ppo/ppo.py:33-384 and rl/ddppo/algo/ddppo.py:59-157):
`from_config`, `update(rollouts) -> Dict[str, float]`, `get_advantages`, `_update_from_batch`
(overridable per-minibatch seam), `before_step` / `after_step`, `.optimizer` (Adam-compatible
state_dict, LambdaLR attaches to it), `.clip_param`, `init_distributed`, `get_resume_state`,
`load_state_dict`.

Per minibatch the reference runs ~9k ATen ops (forward, autograd backward, clip, foreach Adam);
here it is: policy.loss_and_backward (hand-written fwd+bwd kernels) -> [NCCL all-reduce of ONE flat
gradient buffer] -> fused norm + clip + Adam.
"""
from __future__ import annotations

import collections
from typing import Any, Dict, List, Optional

import torch
from torch import nn

from .. import ops
from .._lib import Hb200Error
from ..common.baseline_registry import baseline_registry

EPS_PPO = 1e-5


class FusedAdam(torch.optim.Optimizer):
    """torch.optim.Adam-compatible optimizer (same defaults, param_groups and state_dict layout:
    per-parameter `step`, `exp_avg`, `exp_avg_sq`) whose step is ONE kernel over the policy's flat
    parameter / gradient buffers, fused with clip_grad_norm_ (rl/ppo/ppo.py:112-137, 347-371)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, policy=None):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        foreach=True, capturable=False, differentiable=False, fused=None)
        super().__init__(params, defaults)
        self._policy = policy
        self._m = self._v = self._ws = self._gn = None
        self._step = 0
        self._flat_id = None

    def _bind(self):
        flat = self._policy.flatten_parameters_()
        plist = [p for g in self.param_groups for p in g["params"]]
        if len(plist) != len(flat["plist"]) or any(a is not b for a, b in zip(plist, flat["plist"])):
            raise Hb200Error("FusedAdam: optimizer parameters must be exactly the policy's parameters")
        if self._flat_id != id(flat["params"]):
            dev = flat["params"].device
            m, v = torch.zeros_like(flat["params"]), torch.zeros_like(flat["params"])
            for p, o in zip(plist, flat["offsets"]):  # carry over state loaded through load_state_dict
                st = self.state.get(p, {})
                if "exp_avg" in st:
                    m[o:o + p.numel()].copy_(st["exp_avg"].reshape(-1))
                    v[o:o + p.numel()].copy_(st["exp_avg_sq"].reshape(-1))
                    self._step = max(self._step, int(float(st.get("step", 0))))
                self.state[p] = dict(step=torch.tensor(float(self._step)), exp_avg=m[o:o + p.numel()].view(p.shape),
                                     exp_avg_sq=v[o:o + p.numel()].view(p.shape))
            self._m, self._v = m, v
            self._ws = ops.clip_adam_workspace(flat["n"], dev)
            self._gn = torch.zeros(1, device=dev)
            self._flat_id = id(flat["params"])
        return flat

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._flat_id = None  # re-bind: copies the loaded moments into the flat buffers
        self._step = 0

    @torch.no_grad()
    def step(self, max_grad_norm: Optional[float] = None, grad_scale: float = 1.0):
        flat = self._bind()
        g = self.param_groups[0]
        self._step += 1
        ops.clip_adam(flat["params"][: flat["n"]], flat["grads"][: flat["n"]], self._m[: flat["n"]],
                      self._v[: flat["n"]], g["lr"], g["betas"], g["eps"], g["weight_decay"], max_grad_norm or 0.0,
                      grad_scale, self._step, self._gn, self._ws)
        for st in self.state.values():
            st["step"].fill_(float(self._step))
        self._policy.mark_weights_changed()   # the kernel wrote the parameters behind torch's version counter
        return self._gn


@baseline_registry.register_updater
class PPO(nn.Module):
    @classmethod
    def from_config(cls, actor_critic, config):
        return cls(actor_critic=actor_critic, clip_param=config.clip_param, ppo_epoch=config.ppo_epoch,
                   num_mini_batch=config.num_mini_batch, value_loss_coef=config.value_loss_coef,
                   entropy_coef=config.entropy_coef, lr=config.lr, eps=config.eps,
                   max_grad_norm=config.max_grad_norm, use_clipped_value_loss=config.use_clipped_value_loss,
                   use_normalized_advantage=config.use_normalized_advantage,
                   entropy_target_factor=getattr(config, "entropy_target_factor", 0.0),
                   use_adaptive_entropy_pen=getattr(config, "use_adaptive_entropy_pen", False))

    def __init__(self, actor_critic, clip_param: float, ppo_epoch: int, num_mini_batch: int, value_loss_coef: float,
                 entropy_coef: float, lr: Optional[float] = None, eps: Optional[float] = None,
                 max_grad_norm: Optional[float] = None, use_clipped_value_loss: bool = False,
                 use_normalized_advantage: bool = True, entropy_target_factor: float = 0.0,
                 use_adaptive_entropy_pen: bool = False) -> None:
        super().__init__()
        if use_adaptive_entropy_pen:
            raise NotImplementedError("Lagrangian entropy coefficient (gaussian policies) is a 'next' row")
        self.actor_critic = actor_critic
        self.clip_param = clip_param
        self.ppo_epoch = ppo_epoch
        self.num_mini_batch = num_mini_batch
        self.value_loss_coef = value_loss_coef
        self.entropy_coef = entropy_coef
        self.max_grad_norm = max_grad_norm
        self.use_clipped_value_loss = use_clipped_value_loss
        self.use_normalized_advantage = use_normalized_advantage
        self.device = next(actor_critic.parameters()).device
        self.optimizer = self._create_optimizer(lr, eps)
        self.non_ac_params = [p for name, p in self.named_parameters() if not name.startswith("actor_critic.")]
        self._world = 1
        self._group = None

    def _create_optimizer(self, lr, eps):
        params = [p for p in self.parameters() if p.requires_grad]
        if len(params) == 0:
            return None
        return FusedAdam(params, lr=lr, eps=eps, policy=self.actor_critic)

    # ---- advantages (ppo.py:139-157) ------------------------------------------------------------
    def get_advantages(self, rollouts) -> torch.Tensor:
        fused = rollouts.fused_advantages() if hasattr(rollouts, "fused_advantages") else None
        if fused is None:  # storage without the fused kernel: tiny torch expression, not the hot path
            adv = rollouts.buffers["returns"] - rollouts.buffers["value_preds"]
            fin = adv[torch.isfinite(adv)].double()
            stats = torch.stack([fin.sum(), (fin * fin).sum(), torch.tensor(float(fin.numel()), device=adv.device,
                                                                            dtype=torch.float64), fin.sum() * 0])
        else:
            adv, stats = fused
        if not self.use_normalized_advantage:
            return adv
        if self._var_mean_overridden():   # a subclass supplied its own statistic (reference signature: x -> (var, mean))
            var, mean = self._compute_var_mean(adv[torch.isfinite(adv)])
            mean_var = torch.stack([mean.reshape(()), var.reshape(())]).float()
        else:
            mean_var = self._fused_var_mean(stats)
        ops.adv_normalize(adv, stats=stats if mean_var is None else None, mean_var=mean_var)
        if hasattr(rollouts, "_adv_valid"):
            rollouts._adv_valid = False  # normalised in place: must be recomputed next time
        return adv

    @staticmethod
    def _compute_var_mean(x):
        """The reference's overridable statistic (rl/ppo/ppo.py:160-162): (var, mean) of the finite advantages."""
        return torch.var_mean(x)

    def _var_mean_overridden(self) -> bool:
        fn = getattr(type(self)._compute_var_mean, "__func__", type(self)._compute_var_mean)
        return fn not in (PPO.__dict__["_compute_var_mean"].__func__, DDPPO.__dict__["_compute_var_mean"].__func__)

    def _fused_var_mean(self, stats):
        """None -> single-process unbiased torch.var_mean, evaluated inside the normalise kernel from the
        (sum, sumsq, n) the GAE launch already produced."""
        return None

    def _set_grads_to_none(self):
        pass  # gradients live in one flat buffer that loss_and_backward zero-fills

    # ---- one minibatch (ppo.py:164-299) ---------------------------------------------------------------
    def _update_from_batch(self, batch, epoch, rollouts, learner_metrics):
        ac = self.actor_critic
        metrics = ac.loss_and_backward(batch, self.clip_param, self.value_loss_coef, self.entropy_coef,
                                       self.use_clipped_value_loss)
        grad_norm = self.before_step()
        self.after_step()
        learner_metrics["_metrics"].append(metrics.clone())
        learner_metrics["grad_norm"].append(grad_norm.clone())
        learner_metrics["_is_last_epoch"].append(epoch == (self.ppo_epoch - 1))
        if "is_coeffs" in batch:   # VER's importance weights, unclamped (ppo.py:261-262)
            isc = batch["is_coeffs"].reshape(-1)
            learner_metrics["_ver_is_coeffs"].append(torch.stack([isc.min(), isc.mean(), isc.max()]))

    def before_step(self) -> torch.Tensor:
        """all-reduce (distributed) + clip_grad_norm_ + Adam, fused (ppo.py:347-371, 257-258)."""
        scale = 1.0
        if self._world > 1:
            flat = self.actor_critic.flatten_parameters_()
            tail = getattr(self, "_tail_work", None)
            if tail is not None:
                # the recurrent / head chunk is already in flight (started while the conv stack's backward was running);
                # reduce the rest now and join both
                work, off = tail
                self._tail_work = None
                if off > 0:
                    torch.distributed.all_reduce(flat["grads"][:off], group=self._group)
                work.wait()
            else:
                torch.distributed.all_reduce(flat["grads"], group=self._group)  # SUM over NVLink/NVSwitch
            scale = 1.0 / self._world                                      # DDP's mean, folded into the kernel
        return self.optimizer.step(max_grad_norm=self.max_grad_norm, grad_scale=scale)

    def after_step(self) -> None:
        pass

    def after_update(self) -> None:
        """Hook the agent access manager calls once per update (rl/ppo/updater.py; a no-op for PPO, the Lagrangian
        entropy coefficient of continuous-control policies clamps itself here in the reference)."""

    # ---- whole update (ppo.py:301-332) --------------------------------------------------------------------
    def update(self, rollouts) -> Dict[str, float]:
        advantages = self.get_advantages(rollouts)
        learner_metrics: Dict[str, List[Any]] = collections.defaultdict(list)
        for epoch in range(self.ppo_epoch):
            for batch in rollouts.data_generator(advantages, self.num_mini_batch):
                self._update_from_batch(batch, epoch, rollouts, learner_metrics)
        return self._reduce_metrics(learner_metrics)

    @staticmethod
    def _reduce_metrics(lm) -> Dict[str, float]:
        """Means over minibatches, ONE device->host copy (the reference does ~12 syncs)."""
        m = torch.stack(lm["_metrics"])                       # [n_mb, 12]
        gn = torch.stack(lm["grad_norm"]).reshape(-1, 1)
        last = torch.tensor(lm["_is_last_epoch"], device=m.device).view(-1, 1).float()
        frac = (m[:, 9:10] * last).sum() / last.sum().clamp(min=1)  # ppo_fraction_clipped: last epoch only
        parts = [m.mean(0), gn.mean(0), frac.view(1)]
        if lm.get("_ver_is_coeffs"):
            parts.append(torch.stack(lm["_ver_is_coeffs"]).mean(0))
        host = torch.cat(parts).cpu().tolist()
        out = {k: host[i] for i, k in enumerate(ops.METRIC_KEYS[:9])}
        out["ppo_fraction_clipped"] = host[13]
        out["grad_norm"] = host[12]
        if len(host) > 14:
            out.update(ver_is_coeffs_min=host[14], ver_is_coeffs_mean=host[15], ver_is_coeffs_max=host[16])
        return out

    def _evaluate_actions(self, *args, **kwargs):
        return self.actor_critic.evaluate_actions(*args, **kwargs)

    def before_backward(self, loss):
        return loss

    def after_backward(self, loss):
        pass

    def get_resume_state(self):
        return {"optim_state": self.optimizer.state_dict()}

    def load_state_dict(self, state, strict=True):
        if "optim_state" in state:
            self.optimizer.load_state_dict(state["optim_state"])
        else:
            super().load_state_dict(state, strict=strict)

    def init_distributed(self, find_unused_params: bool = True) -> None:
        pass


@baseline_registry.register_updater
class DDPPO(PPO):
    """Decentralised distributed PPO (rl/ddppo/algo/ddppo.py:87-157): one learner per GPU.
    Instead of wrapping evaluate_actions in DistributedDataParallel (bucketed hooks on ~80 tensors)
    the gradients already sit in ONE flat buffer, so the exchange is a single NCCL all-reduce per
    optimizer step; parameters and buffers are broadcast once from rank 0 like DDP does."""

    def init_distributed(self, find_unused_params: bool = True) -> None:
        import torch.distributed as dist

        if not dist.is_initialized():
            raise Hb200Error("DDPPO.init_distributed: torch.distributed is not initialised")
        self._world = dist.get_world_size()
        self._group = None
        ac = self.actor_critic
        ac.world_size, ac.dist_group = self._world, None
        flat = ac.flatten_parameters_()
        dist.broadcast(flat["params"], src=0)
        for b in ac.buffers():
            dist.broadcast(b, src=0)
        ac.mark_weights_changed()
        # overlap: the gradients of the recurrent encoder + heads (5.4 M of the 8.5 M parameters of config #2) are final
        # ~10 ms before the conv stack's; their all-reduce starts from the backward pass (DDP overlaps bucket by bucket
        # through autograd hooks, ddppo.py:110-152 -- here there are two buckets)
        off = ac.tail_offset() if hasattr(ac, "tail_offset") else flat["n"]
        self._tail_work = None
        if 0 < off < flat["n"] and hasattr(ac, "tail_grads_hook"):
            def start_tail(off=off, flat=flat):
                self._tail_work = (dist.all_reduce(flat["grads"][off: flat["n"]], group=self._group, async_op=True), off)
            ac.tail_grads_hook = start_tail

    @staticmethod
    def _compute_var_mean(x):
        """distributed_var_mean with the reference's signature and collectives (ddppo.py:59-84, 103-105); the built-in
        path below gets the same numbers from one packed all-reduce."""
        import torch.distributed as dist

        world = dist.get_world_size()
        mean = x.mean()
        dist.all_reduce(mean)
        mean = mean / world
        var = (x - mean).pow(2).mean()
        dist.all_reduce(var)
        return var / world, mean

    def _fused_var_mean(self, stats):
        """distributed_var_mean (ddppo.py:59-84): mean of the rank means, mean of the rank BIASED
        variances around the global mean -- reproduced with one packed all-reduce of (sum, sumsq, n)
        partial statistics per rank instead of two dependent scalar all-reduces."""
        import torch.distributed as dist

        if self._world <= 1:
            return None
        s = stats[:3]
        # mean = avg_r E_r[x];  var = avg_r E_r[(x - mean)^2] = avg_r E_r[x^2] - mean^2
        pack = torch.stack([s[0] / s[2], s[1] / s[2]])
        dist.all_reduce(pack, group=self._group)
        mean = pack[0] / self._world
        var = pack[1] / self._world - mean * mean
        return torch.stack([mean, var]).float()
