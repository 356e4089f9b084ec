"""CPU: VER's packed-sequence returns (tests/ver_reference.py, float64) and VERRolloutStorage's bookkeeping against the
reference's VERRolloutStorage, recorded in tests/golden/ver_storage.pt; the ver trainer's config and refusals."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ver_reference as VR  # noqa: E402

from habitat_lab_b200.common.ver_rollout_storage import (  # noqa: E402
    VERRolloutStorage, build_pack_info_from_episode_ids, generate_ver_mini_batches)

GOLD = torch.load(os.path.join(HERE, "golden", "ver_storage.pt"), weights_only=False)


def _pack(snap):
    return build_pack_info_from_episode_ids(*(snap[k].view(-1).numpy() for k in ("episode_ids", "environment_ids",
                                                                                 "step_ids")))


@pytest.mark.parametrize("k", range(3))
def test_restatement_matches_reference_returns(k):
    ro = GOLD["rollouts"][k]
    a = ro["after_rollout"]
    got = VR.ver_gae_reference(a["rewards"], a["value_preds"], a["returns"], a["is_stale"], _pack(a), GOLD["gamma"],
                               GOLD["tau"], ro["use_gae"])
    want = ro["returns"].view(-1).numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = np.isfinite(want)
    assert np.all(np.abs(got[fin].astype(np.float64) - want[fin]) <= VR.bar(want[fin]))
    assert fin.sum() == VR.NUM_STEPS * VR.N_ENVS


def test_fixture_covers_the_cases():
    """single-step environments, episodes ending mid-rollout, stale steps, in-flight steps.  A stale step is always an
    in-flight environment's previous bootstrap step here, so its return is NaN; stale steps with finite returns are
    covered by the kernel tests on generated buffers (test_gpu_ver.py)."""
    seen = dict(single=False, stale_nan=False, in_flight=False, short_seq=False)
    for ro in GOLD["rollouts"]:
        a = ro["after_rollout"]
        counts = np.bincount(a["environment_ids"].view(-1).numpy(), minlength=VR.N_ENVS)
        seen["single"] |= bool((counts == 1).any())
        stale = a["is_stale"].view(-1).numpy()
        fin = np.isfinite(a["returns"].view(-1).numpy())
        seen["stale_nan"] |= bool((stale & ~fin).any())
        seen["in_flight"] |= bool((~ro["after_rollout"]["will_replay_step"].numpy()).any())
        seen["short_seq"] |= bool((_pack(a)["sequence_lengths"] == 1).any())
    assert all(seen.values()), seen


@pytest.mark.parametrize("perturb", ["zero_bootstrap", "tau"])
def test_perturbed_restatement_misses_the_bar(perturb):
    worst = 0.0
    for ro in GOLD["rollouts"][:2]:
        a = ro["after_rollout"]
        kw = dict(keep_stale=perturb != "keep_stale", zero_bootstrap=perturb != "zero_bootstrap")
        got = VR.ver_gae_reference(a["rewards"], a["value_preds"], a["returns"], a["is_stale"], _pack(a),
                                   GOLD["gamma"], GOLD["tau"], use_gae=perturb != "tau", **kw)
        want = ro["returns"].view(-1).numpy()
        both = np.isfinite(want) & np.isfinite(got)
        err = np.abs(got[both].astype(np.float64) - want[both]) / np.maximum(VR.bar(want[both]), 1e-30)
        worst = max(worst, float(err.max(initial=0.0)))
    assert worst >= 10.0


def test_storage_bookkeeping_matches_reference():
    obs, act = VR.make_spaces()
    r = VERRolloutStorage(VR.NUM_STEPS, VR.N_ENVS, obs, act, VR.FakeActorCritic(), variable_experience=True)
    sc = VR.Script(seed=GOLD["seed"])
    for k, ro in enumerate(GOLD["rollouts"]):
        VR.drive_rollout(r, sc)
        r.after_rollout()
        _same(VR.snapshot(r), ro["after_rollout"], f"after_rollout {k}")
        r.buffers["returns"].copy_(ro["returns"])      # compute_returns itself runs on the GPU (test_gpu_ver.py)
        r.build_pack_info()
        np.random.seed(100 + k)
        p = r._pack
        mbs = list(generate_ver_mini_batches(2, p["sequence_lengths"], p["num_seqs_at_step"], p["select_inds"],
                                             p["last_sequence_in_batch_mask"]))
        assert [m.tolist() for m in mbs] == [m.tolist() for m in ro["minibatches"]]
        r.after_update()
        r.increment_policy_version()
        _same(VR.snapshot(r), ro["after_update"], f"after_update {k}")


def _same(got, want, what):
    for key, w in want.items():
        g = got[key]
        if torch.is_tensor(w):
            assert torch.equal(torch.nan_to_num(g, nan=1e30), torch.nan_to_num(w, nan=1e30)), (what, key)
        else:
            assert g == w, (what, key)


def test_is_coeffs_are_steps_per_environment():
    a = GOLD["rollouts"][1]["after_rollout"]
    env = a["environment_ids"].view(-1)
    count = torch.bincount(env, minlength=VR.N_ENVS).float()
    assert torch.equal(a["is_coeffs"].view(-1), ((VR.NUM_STEPS + 1) / count)[env])


def test_pack_info_matches_reference_builder():
    from oracle import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("reference tree not present")
    ref_shim.install()
    from habitat_baselines.rl.models.rnn_state_encoder import build_pack_info_from_episode_ids as ref_build
    rng = np.random.default_rng(0)
    for _ in range(100):
        N, T = int(rng.integers(1, 7)), int(rng.integers(1, 12))
        ep = np.cumsum(rng.random((T, N)) < 0.3, 0)
        env = np.tile(np.arange(N), (T, 1))
        st = np.tile(np.arange(T)[:, None], (1, N))
        perm = rng.permutation(T * N)
        args = [x.reshape(-1)[perm] for x in (ep, env, st)]
        a, b = ref_build(*args), build_pack_info_from_episode_ids(*args)
        for key in a:
            assert np.array_equal(a[key], b[key]), key


def test_ver_config_and_registry():
    from habitat_lab_b200.common.baseline_registry import baseline_registry
    from habitat_lab_b200.rl.ppo_trainer import make_config
    from habitat_lab_b200.rl.ver_trainer import VERTrainer

    cfg = make_config(trainer_name="ver", ver=dict(num_inference_workers=1), step_time_spread=0.5,
                      continuous_actions=3)
    hb = cfg.habitat_baselines
    assert baseline_registry.get_trainer(hb.trainer_name) is VERTrainer
    assert hb.rl.ver.variable_experience and not hb.rl.ver.overlap_rollouts_and_learn
    assert cfg.habitat.synthetic.step_time_spread == 0.5
    assert make_config().habitat.synthetic.step_time_spread == 0.0


@pytest.mark.parametrize("case", ["overlap", "distributed", "frozen_encoder", "obs_transforms"])
def test_ver_refusals(case):
    from types import SimpleNamespace

    from habitat_lab_b200.rl.ppo_trainer import make_config
    from habitat_lab_b200.rl.ver_trainer import VERTrainer

    kw = dict(trainer_name="ver")
    if case == "overlap":
        kw["ver"] = dict(overlap_rollouts_and_learn=True)
    elif case == "distributed":
        kw["ddppo"] = dict(force_distributed=True)
    elif case == "frozen_encoder":
        kw["ddppo"] = dict(train_encoder=False)
    else:
        kw["obs_transforms"] = {"center_cropper": SimpleNamespace(type="CenterCropper", height=64, width=64,
                                                                  channels_last=True, trans_keys=("rgb", "depth"))}
    with pytest.raises(NotImplementedError):
        VERTrainer(make_config(**kw))._init_train()
