"""Generates tests/golden/ver_update_{small,skill}.pt: one PPO.update of the UNMODIFIED reference (through
oracle/ref_shim.py) over a VER buffer, so the packed learner fed by VERRolloutStorage.data_generator can be compared with
it (tests/test_gpu_ver.py).  Run where the reference tree is present:

    python tests/golden/make_golden_ver_update.py

Cases (tests/ver_reference.py UPDATE_CASES): a small categorical LSTM policy (4 environments, num_steps 16) and an
rl_skill.yaml-shaped Gaussian one (18 environments, num_steps 128, 2 minibatches, LSTM-512x2, 7 actions), 64 x 64 RGB-D.
The reference's VERRolloutStorage is driven through two scripted rollouts (episodes ending mid-rollout, unequal steps per
environment, stale and in-flight steps); the float contents are then refilled from a seed (fill_float_buffers), so the
fixture keeps only the bookkeeping arrays.  Per minibatch it records the frame indices, the losses and, before
clipping, every parameter gradient's norm and the head / critic / previous-action gradients whole; then the update's
metrics and the parameter norms after it.
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
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_shim  # noqa: E402
from make_golden_gaussian import action_dist_config  # noqa: E402
from recipe import recipe_state_dict  # noqa: E402
import ver_reference as VR  # noqa: E402


def main():
    R = ref_shim.ref()
    from habitat_baselines.rl.ver.ver_rollout_storage import VERRolloutStorage
    torch.set_num_threads(8)
    sp = R.spaces
    for name, c in VR.UPDATE_CASES.items():
        torch.manual_seed(c["seed"])
        obs_space = sp.Dict({"rgb": sp.Box(0, 255, (c["H"], c["W"], 3), np.uint8),
                             "depth": sp.Box(0, 1, (c["H"], c["W"], 1), np.float32),
                             "pointgoal_with_gps_compass": sp.Box(-1e9, 1e9, (2,), np.float32)})
        if c["gaussian"]:
            act_space = sp.Box(-1.0, 1.0, (c["gaussian"],), np.float32)
            pc = SimpleNamespace(action_distribution_type="gaussian", action_dist=action_dist_config({}))
        else:
            act_space, pc = sp.Discrete(4), None
        pol = R.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=c["layers"],
                                     rnn_type="LSTM", resnet_baseplanes=32, backbone="resnet18",
                                     normalize_visual_inputs=True, policy_config=pc)
        shapes = {k: tuple(v.shape) for k, v in pol.state_dict().items()}
        pol.load_state_dict(recipe_state_dict(shapes, c["seed"]))
        st = VERRolloutStorage(c["T"], c["N"], obs_space, act_space, pol, variable_experience=True)
        sc = VR.Script(seed=c["seed"], n_envs=c["N"], p_done=c["p_done"])
        VR.drive_rollout(st, sc)
        st.after_rollout()
        st.after_update()
        st.increment_policy_version()
        VR.drive_rollout(st, sc)
        st.after_rollout()
        VR.fill_float_buffers(st.buffers, c["seed"] + 1)
        out = dict(case=c, shapes=shapes, ids={k: st.buffers[k].clone() for k in VR.ID_KEYS},
                   policy_version=int(st.current_policy_version.item()))
        st.compute_returns(True, 0.99, 0.95)
        out["returns"] = st.buffers["returns"].clone()
        ppo = R.PPO(pol, use_normalized_advantage=c["normalized"], **VR.UPDATE_PPO_KW)
        mbs = []
        orig_update, orig_step = ppo._update_from_batch, ppo.before_step

        def before_step():
            named = list(pol.named_parameters())
            mbs[-1]["grad_norms"] = {k: p.grad.norm().item() for k, p in named}
            mbs[-1]["grads_small"] = {k: p.grad.clone() for k, p in named if k.startswith(VR.SMALL_PARAMS)}
            return orig_step()

        def update_from_batch(batch, epoch, rollouts, lm):
            mbs.append(dict(n_frames=int(batch["masks"].shape[0]), num_seqs=int(len(
                batch["rnn_build_seq_info"]["cpu_sequence_lengths"])),
                t_max=int(batch["rnn_build_seq_info"]["cpu_sequence_lengths"][0])))
            orig_update(batch, epoch, rollouts, lm)
            mbs[-1].update({k: float(lm[k][-1]) for k in ("value_loss", "action_loss", "dist_entropy")})
            mbs[-1].update({k: float(lm[k][-1]) for k in ("ver_is_coeffs_min", "ver_is_coeffs_mean",
                                                          "ver_is_coeffs_max")})
        ppo.before_step = before_step
        ppo._update_from_batch = update_from_batch
        np.random.seed(c["seed"] + 2)
        out["update_metrics"] = ppo.update(st)
        out["minibatches"] = mbs
        out["param_norms_after_update"] = {k: v.float().norm().item() for k, v in pol.state_dict().items()}
        torch.save(out, os.path.join(HERE, f"{name}.pt"))
        print(name, [(m["n_frames"], m["num_seqs"], m["t_max"], round(m["value_loss"], 5)) for m in mbs],
              {k: round(v, 5) for k, v in out["update_metrics"].items()})


if __name__ == "__main__":
    main()
