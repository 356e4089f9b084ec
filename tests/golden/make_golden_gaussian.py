"""Generates tests/golden/gaussian_{monolithic,social_nav}.pt by running the UNMODIFIED reference classes (through
oracle/ref_shim.py) with a gaussian PointNavResNetPolicy on a PointNav RGB-D rollout, T = 4, N = 2, 128 x 128, over a
Box(-1, 1, (3,)) action space, for the two shipped action_dist settings (monolithic.yaml: use_log_std; social_nav.yaml:
use_std_param + clamp_std).  Run where the reference tree is present:

    python tests/golden/make_golden_gaussian.py

Inputs and weights are regenerated from seeds (tests/golden/recipe.py and continuous_rollout below); the fixtures hold the
reference's outputs: returns / advantages, the minibatch's values, log-probs, entropy, losses and per-frame hidden
state, every parameter gradient (norms; whole tensors for the head, the critic and the previous-action embedding), and
after one PPO.update its metrics and the parameters (norms; whole tensors for the same small ones).
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import ref_shim  # noqa: E402
from recipe import recipe_state_dict, synthetic_rollout  # noqa: E402

A = 3
CASES = {
    "gaussian_monolithic": dict(T=4, N=2, H=128, W=128, layers=2, seed=51, action_dist=dict(use_log_std=True)),
    "gaussian_social_nav": dict(T=4, N=2, H=128, W=128, layers=2, seed=52,
                                action_dist=dict(use_log_std=True, clamp_std=True, use_std_param=True)),
}
PPO_KW = dict(clip_param=0.2, ppo_epoch=1, num_mini_batch=1, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4,
              eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True, use_normalized_advantage=False)
SMALL = ("action_distribution.", "critic.", "net.prev_action_embedding.")   # recorded whole


def action_dist_config(overrides):
    """ActionDistributionConfig with the reference's defaults (config/default_structured_configs.py:69-86)"""
    c = dict(use_log_std=True, use_softplus=False, std_init=-1.0, log_std_init=0.0, use_std_param=False,
             clamp_std=True, min_std=1e-6, max_std=1, min_log_std=-5, max_log_std=2, action_activation="tanh",
             scheduled_std=False)
    c.update(overrides)
    return SimpleNamespace(**c)


def continuous_rollout(c, n_actions: int):
    """synthetic_rollout's buffers for a Box action space: f32 [T+1, N, A] actions / previous actions in [-1.5, 1.5)
    and old log-probs near a unit Gaussian's (the gaussian policies start with a std near 1)"""
    bufs, next_value = synthetic_rollout(c["T"], c["N"], c["H"], c["W"], 4, 2 * c["layers"], 512, c["seed"])
    g = torch.Generator().manual_seed(c["seed"] + 7)
    shape = (c["T"] + 1, c["N"], n_actions)
    bufs["actions"] = torch.rand(shape, generator=g) * 3.0 - 1.5
    bufs["prev_actions"] = torch.rand(shape, generator=g) * 3.0 - 1.5
    bufs["action_log_probs"] = (-n_actions * 0.5 * np.log(2 * np.pi) - 0.5 * (bufs["actions"] ** 2).sum(-1, keepdim=True)
                                + 0.2 * torch.randn(c["T"] + 1, c["N"], 1, generator=g))
    return bufs, next_value


def main():
    R = ref_shim.ref()
    torch.set_num_threads(8)
    sp = R.spaces
    for name, c in CASES.items():
        torch.manual_seed(c["seed"])
        obs_space = sp.Dict({
            "rgb": sp.Box(0, 255, (c["H"], c["W"], 3), np.uint8),
            "depth": sp.Box(0, 1, (c["H"], c["W"], 1), np.float32),
            "pointgoal_with_gps_compass": sp.Box(-1e9, 1e9, (2,), np.float32),
        })
        act_space = sp.Box(-1.0, 1.0, (A,), np.float32)
        pc = SimpleNamespace(action_distribution_type="gaussian", action_dist=action_dist_config(c["action_dist"]))
        pol = R.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=c["layers"],
                                     rnn_type="LSTM", resnet_baseplanes=32, backbone="resnet18",
                                     normalize_visual_inputs=True, policy_config=pc)
        shapes = {k: tuple(v.shape) for k, v in pol.state_dict().items()}
        pol.load_state_dict(recipe_state_dict(shapes, c["seed"]))
        st = R.RolloutStorage(c["T"], c["N"], obs_space, act_space, pol)
        bufs, next_value = continuous_rollout(c, A)
        for k, v in bufs["observations"].items():
            st.buffers["observations"][k].copy_(v)
        for k in ("recurrent_hidden_states", "masks", "rewards", "value_preds", "returns", "action_log_probs",
                  "actions", "prev_actions"):
            st.buffers[k].copy_(bufs[k])
        st.current_rollout_step_idxs = [c["T"]]
        out = {"case": c, "shapes": shapes}
        st.compute_returns(next_value, True, 0.99, 0.95)
        out["returns"] = st.buffers["returns"].clone()
        out["value_preds_after"] = st.buffers["value_preds"].clone()
        ppo = R.PPO(pol, **PPO_KW)
        out["advantages"] = ppo.get_advantages(st).clone()
        # --- one minibatch (all envs): evaluate_actions + the PPO loss + backward
        pol.train()
        torch.manual_seed(1000 + c["seed"])
        batch = next(iter(st.data_generator(out["advantages"], 1)))
        out["mb_env_inds_seed"] = 1000 + c["seed"]
        stats_before = {k: v.clone() for k, v in pol.state_dict().items() if "running_mean_and_var" in k}
        values, lp, ent, hid, _ = pol.evaluate_actions(batch["observations"], batch["recurrent_hidden_states"],
                                                       batch["prev_actions"], batch["masks"], batch["actions"],
                                                       batch["rnn_build_seq_info"])
        out["eval_values"], out["eval_log_probs"], out["eval_entropy"] = values.detach(), lp.detach(), ent.detach()
        out["eval_hidden"] = hid.detach()
        ratio = torch.exp(lp - batch["action_log_probs"])
        s1 = batch["advantages"] * ratio
        s2 = batch["advantages"] * torch.clamp(ratio, 0.8, 1.2)
        action_loss = -torch.min(s1, s2)
        delta = values.detach() - batch["value_preds"]
        vv = torch.where(delta.abs() < 0.2, values, batch["value_preds"] + delta.clamp(-0.2, 0.2))
        value_loss = 0.5 * (vv - batch["returns"]) ** 2
        total = 0.5 * value_loss.mean() + action_loss.mean() - 0.01 * ent.mean()
        pol.zero_grad()
        total.backward()
        out["mb_losses"] = dict(value_loss=value_loss.mean().item(), action_loss=action_loss.mean().item(),
                                dist_entropy=ent.mean().item(), total=total.item())
        out["grad_norms"] = {k: p.grad.norm().item() for k, p in pol.named_parameters()}
        out["grads_small"] = {k: p.grad.clone() for k, p in pol.named_parameters() if k.startswith(SMALL)}
        pol.load_state_dict({**pol.state_dict(), **stats_before})
        pol.zero_grad()
        # --- one PPO.update (ppo.py:301-332)
        torch.manual_seed(2000 + c["seed"])
        out["update_metrics"] = ppo.update(st)
        sd = pol.state_dict()
        out["param_norms_after_update"] = {k: v.float().norm().item() for k, v in sd.items()}
        out["params_small_after_update"] = {k: v.clone() for k, v in sd.items() if k.startswith(SMALL)}
        torch.save(out, os.path.join(HERE, f"{name}.pt"))
        print(name, "losses", out["mb_losses"], "update", {k: round(v, 6) for k, v in out["update_metrics"].items()})


if __name__ == "__main__":
    main()
