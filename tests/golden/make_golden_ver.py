"""Generates tests/golden/ver_storage.pt by running the UNMODIFIED reference VERRolloutStorage (through
oracle/ref_shim.py) on CPU through three scripted VER rollouts (tests/ver_reference.py: 6 environments, num_steps 8,
environment 0 slow enough to contribute a single step, episodes ending mid-rollout, so stale steps with finite and NaN
returns and in-flight steps appear).  Run where the reference tree is present:

    python tests/golden/make_golden_ver.py

Per rollout it records the buffers after after_rollout, the returns after compute_returns (gamma 0.99, tau 0.95; the
third rollout with use_gae=False), the frame indices of two minibatches for np.random.seed(100 + rollout), and the
buffers and auxiliary state after after_update.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_shim  # noqa: E402
import ver_reference as VR  # noqa: E402

ROLLOUTS = 3
USE_GAE = (True, True, False)


def main():
    ref_shim.install()
    gs = sys.modules["gym.spaces"]
    from habitat_baselines.rl.ver.ver_rollout_storage import VERRolloutStorage, generate_ver_mini_batches

    obs = gs.Dict({"pointgoal_with_gps_compass": gs.Box(-1e9, 1e9, (2,), np.float32)})
    r = VERRolloutStorage(VR.NUM_STEPS, VR.N_ENVS, obs, gs.Discrete(4), VR.FakeActorCritic(), variable_experience=True)
    sc = VR.Script(seed=7)
    rec = []
    for k in range(ROLLOUTS):
        VR.drive_rollout(r, sc)
        r.after_rollout()
        after_rollout = VR.snapshot(r)
        r.compute_returns(USE_GAE[k], VR.GAMMA, VR.TAU)
        returns = r.buffers["returns"].clone()
        np.random.seed(100 + k)
        mbs = [torch.from_numpy(m.copy()) for m in generate_ver_mini_batches(
            2, r.sequence_lengths, r.num_seqs_at_step, r.select_inds, r.last_sequence_in_batch_mask,
            r.episode_ids_cpu)]
        r.after_update()
        r.increment_policy_version()
        rec.append(dict(after_rollout=after_rollout, returns=returns, minibatches=mbs, after_update=VR.snapshot(r),
                        use_gae=USE_GAE[k]))
    out = os.path.join(HERE, "ver_storage.pt")
    torch.save(dict(rollouts=rec, gamma=VR.GAMMA, tau=VR.TAU, seed=7), out)
    counts = [np.bincount(x["after_rollout"]["environment_ids"].view(-1).numpy(), minlength=VR.N_ENVS) for x in rec]
    print(out, "steps per environment per rollout:", [c.tolist() for c in counts])


if __name__ == "__main__":
    main()
