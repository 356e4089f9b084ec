"""CPU: fine-tuning from a pretrained checkpoint with a frozen visual encoder (`rl.ddppo.pretrained`,
`pretrained_encoder`, `pretrained_weights`, `train_encoder`, `reset_critic`) against the reference's own
SingleAgentAccessMgr._create_policy, get_rollout_obs_space, PPO optimizer and encoder calls
(habitat-baselines/habitat_baselines/rl/ppo/single_agent_access_mgr.py:205-237, 300-319, rl/ppo/ppo.py:112-113,
rl/ppo/ppo_trainer.py:261-279, 467-471), run on the CPU through oracle/ref_shim.  No GPU: the policy objects here are
parameter holders."""
import collections
import sys
import types
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
H = W = 128
CONFIGS = {   # BASELINE config #2 (PointNav, ResNet18 + LSTM) and #3 (ObjectNav sensors, ResNet50 + GRU)
    2: dict(backbone="resnet18", rnn_type="LSTM", num_recurrent_layers=2),
    3: dict(backbone="resnet50", rnn_type="GRU", num_recurrent_layers=1),
}


def _spaces(sp, kind):
    od = collections.OrderedDict()
    od["rgb"] = sp.Box(0, 255, (H, W, 3), np.uint8)
    if kind == "imagegoal":
        od["imagegoal"] = sp.Box(0, 255, (H, W, 3), np.uint8)
    else:
        od["depth"] = sp.Box(0, 1, (H, W, 1), np.float32)
    if kind == 2:
        od["pointgoal_with_gps_compass"] = sp.Box(-1e9, 1e9, (2,), np.float32)
    else:
        if kind == 3:
            od["semantic"] = sp.Box(0, 2 ** 30, (H, W, 1), np.int32)
            od["objectgoal"] = sp.Box(0, 20, (1,), np.int64)
        od["compass"] = sp.Box(-np.pi, np.pi, (1,), np.float32)
        od["gps"] = sp.Box(-1e9, 1e9, (2,), np.float32)
    return sp.Dict(od), sp.Discrete(4)


def _config(kind, **ddppo):
    from habitat_lab_b200.rl.ppo_trainer import make_config

    cfg = make_config(num_environments=4, height=H, width=W, num_steps=8,
                      ddppo={**CONFIGS.get(kind, CONFIGS[2]), **ddppo})
    cfg.habitat_baselines.rl.auxiliary_losses = {}   # read by the reference's from_config
    return cfg


def _native(kind, seed=0, policy_name="PointNavResNetPolicy", **ddppo):
    from habitat_lab_b200.common import spaces
    from habitat_lab_b200.rl.single_agent_access_mgr import SingleAgentAccessMgr

    cfg = _config(kind, **ddppo)
    cfg.habitat_baselines.rl.policy["main_agent"].name = policy_name
    obs, act = _spaces(spaces, kind)
    torch.manual_seed(seed)
    spec = SimpleNamespace(observation_space=obs, action_space=act, orig_action_space=act)
    return SingleAgentAccessMgr(config=cfg, env_spec=spec, is_distrib=False, device=torch.device("cpu"),
                                percent_done_fn=lambda: 0.0), cfg, obs


def _ref_modules():
    R = ref_shim.ref()
    if "habitat_baselines.rl.ppo.single_agent_access_mgr" not in sys.modules:
        # the hierarchical (rearrange) policy is imported for its registration only and needs the simulator's task
        # package: an empty stand-in keeps the module importable
        hrl = types.ModuleType("habitat_baselines.rl.hrl.hierarchical_policy")
        hrl.HierarchicalPolicy = type("HierarchicalPolicy", (), {})
        sys.modules.setdefault("habitat_baselines.rl.hrl", types.ModuleType("habitat_baselines.rl.hrl"))
        sys.modules.setdefault("habitat_baselines.rl.hrl.hierarchical_policy", hrl)
    import habitat_baselines.rl.ppo.single_agent_access_mgr as M

    return R, M


def _reference(kind, seed=0, **ddppo):
    """the reference's _create_policy on the same config (the bound method's state is its five attributes)"""
    R, M = _ref_modules()
    cfg = _config(kind, **ddppo)
    obs, act = _spaces(R.spaces, kind)
    torch.manual_seed(seed)
    fake = SimpleNamespace(_config=cfg, agent_name="main_agent", _device=torch.device("cpu"),
                           _env_spec=SimpleNamespace(observation_space=obs, action_space=act, orig_action_space=act),
                           _is_static_encoder=not cfg.habitat_baselines.rl.ddppo.train_encoder)
    return M.SingleAgentAccessMgr._create_policy(fake), cfg, obs


def _checkpoint(tmp_path, kind=2, prefix="actor_critic."):
    """a habitat-baselines checkpoint written from a reference policy built on the CPU, with non-trivial
    RunningMeanAndVar buffers so that loading them is visible"""
    R = ref_shim.ref()
    obs, act = _spaces(R.spaces, kind)
    torch.manual_seed(1234)
    pol = R.PointNavResNetPolicy(obs, act, hidden_size=512, resnet_baseplanes=32, normalize_visual_inputs=True,
                                 **CONFIGS[kind])
    sd = pol.state_dict()
    for v in sd.values():   # GroupNorm's ones / zeros would otherwise load unseen
        v.add_(0.01 * torch.randn_like(v))
    rmv = "net.visual_encoder.running_mean_and_var."
    sd[rmv + "_mean"].uniform_(0.2, 0.6)
    sd[rmv + "_var"].uniform_(0.01, 0.1)
    sd[rmv + "_count"].fill_(4096.0)
    path = tmp_path / "pretrained.pth"
    torch.save({"state_dict": {prefix + k: v for k, v in sd.items()}, "extra_state": {"step": 1}}, path)
    return str(path), {k: v.clone() for k, v in sd.items()}


@needs_ref
@pytest.mark.parametrize("kind", [2, 3])
def test_rollout_obs_space_matches_reference(kind):
    from habitat_lab_b200.rl.single_agent_access_mgr import get_rollout_obs_space
    _, M = _ref_modules()

    mgr, cfg, obs = _native(kind, train_encoder=False)
    ref_ac, rcfg, robs = _reference(kind, train_encoder=False)
    got = get_rollout_obs_space(obs, mgr.actor_critic, cfg)
    want = M.get_rollout_obs_space(robs, ref_ac, rcfg)
    assert list(got.spaces) == list(want.spaces) and list(got.spaces)[0] == "visual_features"
    for k, w in want.spaces.items():
        g = got.spaces[k]
        assert g.shape == w.shape and np.dtype(g.dtype) == np.dtype(w.dtype), k
        assert np.array_equal(g.low, w.low) and np.array_equal(g.high, w.high), k
    assert got.spaces["visual_features"].shape == tuple(mgr.actor_critic.net.visual_encoder.output_shape)
    # with the encoder trained the storage keeps the environment's space
    mgr2, cfg2, obs2 = _native(kind)
    assert get_rollout_obs_space(obs2, mgr2.actor_critic, cfg2) is obs2


@needs_ref
def test_pretrained_loads_the_whole_policy(tmp_path):
    path, sd = _checkpoint(tmp_path)
    mgr, _, _ = _native(2, pretrained=True, pretrained_weights=path, reset_critic=False)
    got = mgr.actor_critic.state_dict()
    assert set(got) == set(sd)
    for k, v in sd.items():
        assert torch.equal(got[k], v), k
    ref_ac, _, _ = _reference(2, pretrained=True, pretrained_weights=path, reset_critic=False)
    for k, v in ref_ac.state_dict().items():
        assert torch.equal(got[k], v), k


@needs_ref
def test_pretrained_encoder_loads_only_the_visual_encoder(tmp_path):
    path, sd = _checkpoint(tmp_path)
    fresh = _native(2, seed=7)[0].actor_critic.state_dict()
    got = _native(2, seed=7, pretrained_encoder=True, pretrained_weights=path,
                  reset_critic=False)[0].actor_critic.state_dict()
    changed = {k for k in fresh if not torch.equal(fresh[k], got[k])}
    enc = {k for k in fresh if k.startswith("net.visual_encoder.")}
    assert changed == enc, (sorted(changed - enc)[:5], sorted(enc - changed)[:5])
    for k in enc:
        assert torch.equal(got[k], sd[k]), k
    ref_ac, _, _ = _reference(2, pretrained_encoder=True, pretrained_weights=path, reset_critic=False)
    ref_sd = ref_ac.state_dict()
    for k in enc:
        assert torch.equal(got[k], ref_sd[k]), k


@needs_ref
def test_reset_critic_redraws_the_loaded_critic(tmp_path):
    path, sd = _checkpoint(tmp_path)
    ac = _native(2, pretrained=True, pretrained_weights=path, reset_critic=True)[0].actor_critic
    w, b = ac.critic.fc.weight.detach(), ac.critic.fc.bias.detach()
    assert w.norm().item() == pytest.approx(1.0, abs=1e-5)        # orthogonal_ of a 1 x 512 matrix: a unit row
    assert torch.count_nonzero(b) == 0
    assert not torch.equal(w, sd["critic.fc.weight"])
    for k, v in sd.items():
        if not k.startswith("critic."):
            assert torch.equal(ac.state_dict()[k], v), k
    # a run from scratch keeps its seeded initial critic
    a = _native(2, seed=3)[0].actor_critic.critic.fc.weight
    b2 = _native(2, seed=3, reset_critic=False)[0].actor_critic.critic.fc.weight
    assert torch.equal(a, b2)


@needs_ref
def test_checkpoint_without_the_prefix_is_refused(tmp_path):
    path, _ = _checkpoint(tmp_path, prefix="")
    with pytest.raises(ValueError, match="actor_critic"):
        _native(2, pretrained=True, pretrained_weights=path)
    with pytest.raises(ValueError, match="actor_critic"):
        _native(2, pretrained_encoder=True, pretrained_weights=path)


@needs_ref
@pytest.mark.parametrize("kind", [2, 3])
def test_frozen_trainable_set_and_optimizer_match_reference(kind):
    R, _ = _ref_modules()
    mgr, _, _ = _native(kind, train_encoder=False)
    ref_ac, _, _ = _reference(kind, train_encoder=False)
    trainable = [n for n, p in mgr.actor_critic.named_parameters() if p.requires_grad]
    assert trainable == [n for n, p in ref_ac.named_parameters() if p.requires_grad]
    assert not any(n.startswith("net.visual_encoder.") for n in trainable)
    ref_ppo = R.PPO(ref_ac, clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01,
                    lr=2.5e-4, eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True, use_normalized_advantage=False)
    got = mgr.updater.optimizer.param_groups[0]["params"]
    want = ref_ppo.optimizer.param_groups[0]["params"]
    assert [tuple(p.shape) for p in got] == [tuple(p.shape) for p in want]
    assert sum(p.numel() for p in got) == sum(p.numel() for p in want)
    # the optimizer state layout is the reference's: a reference resume state loads
    sd = ref_ppo.optimizer.state_dict()
    mgr.updater.optimizer.load_state_dict(sd)


def test_unsupported_frozen_configurations_raise():
    with pytest.raises(NotImplementedError, match="SimpleCNN"):
        _native(2, policy_name="PointNavBaselinePolicy", train_encoder=False)
    with pytest.raises(NotImplementedError, match="image-goal"):
        _native("imagegoal", train_encoder=False)
    from habitat_lab_b200.common import spaces
    from habitat_lab_b200.rl.single_agent_access_mgr import SingleAgentAccessMgr

    cfg = _config(2, train_encoder=False)
    cfg.habitat_baselines.force_blind_policy = True
    obs, act = _spaces(spaces, 2)
    with pytest.raises(NotImplementedError, match="blind"):
        SingleAgentAccessMgr(config=cfg, env_spec=SimpleNamespace(observation_space=obs, action_space=act),
                             is_distrib=False, device=torch.device("cpu"), percent_done_fn=lambda: 0.0)


@needs_ref
def test_reference_updates_running_mean_and_var_once():
    """What the native trainer mirrors: the reference's frozen-encoder calls (ppo_trainer.py:261-279 in training mode
    right after post_init, :467-471 in the eval-mode rollout, under inference_mode) update RunningMeanAndVar on the first
    batch only, and the learner's evaluate_actions reads `visual_features` without calling the encoder."""
    R, _ = _ref_modules()
    ac, _, obs_space = _reference(2, train_encoder=False)
    enc = ac.visual_encoder
    rmv = enc.running_mean_and_var
    calls = []
    enc.register_forward_hook(lambda *a: calls.append(1))
    N = 4
    g = torch.Generator().manual_seed(0)

    def batch():
        return {"rgb": torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8),
                "depth": torch.rand(N, H, W, 1, generator=g),
                "pointgoal_with_gps_compass": torch.rand(N, 2, generator=g)}

    assert ac.training
    with torch.inference_mode():
        first = batch()
        feats0 = enc(first)
    assert float(rmv._count) == N
    stats = (rmv._mean.clone(), rmv._var.clone())
    ac.eval()
    with torch.inference_mode():
        for _ in range(3):
            enc(batch())
    assert float(rmv._count) == N and torch.equal(rmv._mean, stats[0]) and torch.equal(rmv._var, stats[1])
    # the features of the first batch are those of the updated statistics: an eval-mode call reproduces them
    with torch.inference_mode():
        assert torch.equal(enc(first), feats0)
    assert tuple(feats0.shape[1:]) == tuple(enc.output_shape)
    calls.clear()
    ac.train()
    ob = dict(batch(), visual_features=feats0.clone())
    hid = torch.zeros(N, ac.net.num_recurrent_layers, 512)
    ac.evaluate_actions(ob, hid, torch.zeros(N, 1, dtype=torch.long), torch.ones(N, 1, dtype=torch.bool),
                        torch.zeros(N, 1, dtype=torch.long), None)
    assert not calls and float(rmv._count) == N
