"""CPU checks of the Gaussian action head: the float64 restatement the GPU tests judge the kernels by equals the
reference's GaussianNet / CustomNormal and its PPO loss, fp32 stays within its bars and every perturbed restatement
misses them by at least 10x; config parsing, checkpoint layout and rollout storage shapes match the reference; the
combinations that are not implemented raise NotImplementedError.  No GPU: policy objects here are parameter holders."""
import itertools
from types import SimpleNamespace

import pytest
import torch

import gaussian_reference as G
from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")

FLAG_MIXES = [dict(use_log_std=lg, use_softplus=sp, use_std_param=pa, clamp_std=cl, action_activation=act)
              for lg, sp, pa, cl, act in itertools.product([True, False], [True, False], [True, False],
                                                           [True, False], ["tanh", ""])]


def _ref_gaussian():
    ref_shim.install()
    from habitat_baselines.utils.common import CustomNormal, GaussianNet
    return GaussianNet, CustomNormal


def _cfg(**kw):
    base = dict(use_log_std=True, use_softplus=False, std_init=-1.0, log_std_init=0.0, use_std_param=False,
                clamp_std=True, min_std=1e-6, max_std=1, min_log_std=-5, max_log_std=2, action_activation="tanh",
                scheduled_std=False)
    base.update(kw)
    return SimpleNamespace(**base)


@needs_ref
@pytest.mark.parametrize("mix", FLAG_MIXES, ids=lambda m: "-".join(f"{k}={v}" for k, v in m.items()))
def test_restatement_is_reference_gaussian_net(mix):
    """head() + log_prob_entropy() in float64 = the reference's GaussianNet / CustomNormal, gradients included"""
    GaussianNet, _ = _ref_gaussian()
    torch.manual_seed(3)
    A, H, B = 3, 32, 9
    net = GaussianNet(H, A, _cfg(**mix)).double()
    flags, lo, hi = G.bounds(mix)
    assert (net.min_std, net.max_std) == pytest.approx((lo, hi))
    x = torch.randn(B, H, dtype=torch.float64, requires_grad=True)
    d = net(x)
    a = d.sample().detach()
    lp, ent = d.log_probs(a), d.entropy()
    (lp.sum() + 0.3 * ent.sum()).backward()
    ref_grads = [x.grad.clone()] + [p.grad.clone() for p in net.parameters()]
    std_p = net.std.detach() if net.std is not None else None
    P = dict(w_mu=net.mu_maybe_std.weight.detach(), b_mu=net.mu_maybe_std.bias.detach(), std=std_p)
    P = {k: None if v is None else v.clone().requires_grad_(True) for k, v in P.items()}
    x2 = x.detach().clone().requires_grad_(True)
    mu, std, _, _ = G.head(x2, P["w_mu"], P["b_mu"], P["std"], torch.zeros(1, H, dtype=torch.float64),
                           torch.zeros(1, dtype=torch.float64), flags, lo, hi)
    lp2, ent2 = G.log_prob_entropy(mu, std, a)
    # GaussianNet casts mu_maybe_std to fp32 (`.float()`): the comparison is at fp32 precision
    close = lambda a, b: torch.testing.assert_close(a, b.double(), rtol=2e-5, atol=2e-6)  # noqa: E731
    close(mu, d.mean)
    close(lp2, lp.squeeze(-1))
    close(ent2, ent.squeeze(-1))
    (lp2.sum() + 0.3 * ent2.sum()).backward()
    got = [x2.grad] + ([P["std"].grad] if net.std is not None else []) + [P["w_mu"].grad, P["b_mu"].grad]
    for g, r in zip(got, ref_grads):
        close(g, r)


@needs_ref
@pytest.mark.parametrize("mix", [dict(), dict(use_std_param=True)], ids=["monolithic", "social_nav"])
def test_restatement_is_reference_ppo_loss(mix):
    """loss() = the reference's PPO._update_from_batch driven with its GaussianNet / CustomNormal head and a linear
    critic on the same minibatch: the losses and metrics it records and the gradients it leaves (lr = 0 and an
    unreachable max_grad_norm, so the optimizer step and the clip leave parameters and gradients as backward made them)"""
    import collections
    GaussianNet, _ = _ref_gaussian()
    from habitat_baselines.rl.ppo.ppo import PPO
    params, x, case, (flags, lo, hi) = G.make_case(40, 32, 4, mix, seed=5)
    ref = G.loss(params, x, case, flags, lo, hi)

    class GaussianActorCritic(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.action_distribution = GaussianNet(32, 4, _cfg(**mix))
            self.critic = torch.nn.Linear(32, 1)

        def evaluate_actions(self, obs, h, pa, m, actions, info):
            dist = self.action_distribution(obs)
            return self.critic(obs), dist.log_probs(actions), dist.entropy(), h, {}

        def policy_parameters(self):
            return self.parameters()

        def aux_loss_parameters(self):
            return {}

    ac = GaussianActorCritic()
    gn = ac.action_distribution
    with torch.no_grad():
        gn.mu_maybe_std.weight.copy_(params["w_mu"])
        gn.mu_maybe_std.bias.copy_(params["b_mu"])
        if params["std"] is not None:
            gn.std.copy_(params["std"])
        ac.critic.weight.copy_(params["w_val"])
        ac.critic.bias.copy_(params["b_val"])
    ppo = PPO(ac, clip_param=case["clip"], ppo_epoch=1, num_mini_batch=1, value_loss_coef=case["c_v"],
              entropy_coef=case["c_e"], lr=0.0, eps=1e-5, max_grad_norm=1e30, use_clipped_value_loss=True,
              use_normalized_advantage=False)
    obs = x.clone().requires_grad_(True)
    batch = dict(observations=obs, recurrent_hidden_states=None, prev_actions=None, masks=None, actions=case["actions"],
                 action_log_probs=case["old_lp"][:, None], advantages=case["adv"][:, None],
                 value_preds=case["old_v"][:, None], returns=case["ret"][:, None])
    metrics = collections.defaultdict(list)
    ppo._update_from_batch(batch, 0, None, metrics)
    # the reference computes in fp32 (GaussianNet casts to fp32): agreement with the float64 restatement at fp32 level
    close = lambda a, b: torch.testing.assert_close(a.double(), b.double(), rtol=1e-4, atol=1e-6)  # noqa: E731
    names = ("value_loss", "action_loss", "dist_entropy", "value_pred_min", "value_pred_mean", "value_pred_max",
             "prob_ratio_min", "prob_ratio_mean", "prob_ratio_max")
    for i, k in enumerate(names):
        close(torch.as_tensor(metrics[k][0]).detach(), ref["metrics"][i])
    close(torch.as_tensor(metrics["ppo_fraction_clipped"][0]).detach(), ref["metrics"][9])
    close(obs.grad, ref["d_features"])
    close(gn.mu_maybe_std.weight.grad, ref["d_w_mu"])
    close(gn.mu_maybe_std.bias.grad, ref["d_b_mu"])
    close(ac.critic.weight.grad, ref["d_w_val"])
    close(ac.critic.bias.grad, ref["d_b_val"])
    if params["std"] is not None:
        close(gn.std.grad, ref["d_std"])


@pytest.mark.parametrize("mix", FLAG_MIXES, ids=lambda m: "-".join(f"{k}={v}" for k, v in m.items()))
@pytest.mark.parametrize("A,H,B", [(1, 32, 37), (7, 128, 200), (16, 64, 64)])
def test_fp32_within_bars_and_perturbations_miss(mix, A, H, B):
    """fp32 autograd of the same op sequence stays within every bar; each perturbation that changes a result misses
    its bar by at least 10x"""
    params, x, case, (flags, lo, hi) = G.make_case(B, H, A, mix, seed=A * 100 + H + B, std_at_bounds=True)
    ref = G.loss(params, x, case, flags, lo, hi)
    bar = G.bars(params, x, case, flags, lo, hi, ref)
    f32 = G.loss(params, x, case, flags, lo, hi, dtype=torch.float32)
    for k in G.COMPARED:
        if k in ref:
            assert G.ratio_to_bar(f32[k], ref[k], bar[k]) <= 1.0, k
    assert G.ratio_to_bar(f32["metrics"][:9], ref["metrics"][:9], bar["metrics"][:9]) <= 1.0
    for p in G.PERTURBATIONS:
        pr = G.loss(params, x, case, flags, lo, hi, perturb=p)
        diffs = [k for k in G.COMPARED if k in ref and not torch.allclose(pr[k], ref[k], rtol=1e-9, atol=0)]
        if not diffs:
            continue
        worst = max(G.ratio_to_bar(pr[k], ref[k], bar[k]) for k in diffs)
        assert worst >= 10.0, (p, diffs, worst)


def test_at_bounds_case_exercises_the_clamp_edge():
    """with std_at_bounds the clamp-edge perturbation changes the gradient (so the GPU matrix covers that edge)"""
    params, x, case, (flags, lo, hi) = G.make_case(37, 32, 2, dict(use_std_param=True), seed=1, std_at_bounds=True)
    ref = G.loss(params, x, case, flags, lo, hi)
    pr = G.loss(params, x, case, flags, lo, hi, perturb="clamp_grad_blocked_at_bounds")
    assert not torch.equal(pr["d_std"], ref["d_std"])


# ---- configuration, checkpoint layout, storage, refusals ---------------------------------------------------------
def test_config_fields_parsed():
    import habitat_lab_b200 as hb
    torch.manual_seed(0)
    for mix in FLAG_MIXES:
        gn = hb.GaussianNet(64, 3, _cfg(**mix, min_std=0.01, max_std=2.0, min_log_std=-4, max_log_std=1))
        flags, lo, hi = G.bounds(dict(mix, min_std=0.01, max_std=2.0, min_log_std=-4, max_log_std=1))
        assert gn.flags == flags
        assert (gn.min_std, gn.max_std) == pytest.approx((lo, hi))
        assert (gn.std is not None) == mix["use_std_param"]
    gn = hb.GaussianNet(64, 3, None)   # the reference's defaults
    assert gn.flags == G.LOG_STD | G.CLAMP_STD | G.TANH and (gn.min_std, gn.max_std) == (-5, 2)


@needs_ref
@pytest.mark.parametrize("mix", [dict(), dict(clamp_std=True, use_std_param=True)], ids=["monolithic", "social_nav"])
def test_state_dict_matches_reference(mix):
    """the gaussian PointNavResNetPolicy's state_dict keys / shapes / initial head values equal the reference's"""
    import habitat_lab_b200 as hb
    from habitat_lab_b200.synthetic import pointnav_spaces
    R = ref_shim.ref()
    obs, _ = pointnav_spaces(64, 64)
    pc = SimpleNamespace(action_distribution_type="gaussian", action_dist=_cfg(**mix))
    torch.manual_seed(7)
    ours = hb.PointNavResNetPolicy(obs, hb.spaces.Box(-1.0, 1.0, (5,)), hidden_size=64, num_recurrent_layers=2,
                                   rnn_type="LSTM", policy_config=pc).state_dict()
    rs = R.spaces.Dict({k: R.spaces.Box(v.low, v.high, v.shape, v.dtype) for k, v in obs.spaces.items()})
    torch.manual_seed(7)
    ref = R.PointNavResNetPolicy(rs, R.spaces.Box(-1.0, 1.0, (5,)), hidden_size=64, num_recurrent_layers=2,
                                 rnn_type="LSTM", policy_config=pc).state_dict()
    assert list(ours.keys()) == list(ref.keys())
    for k in ref:
        assert ours[k].shape == ref[k].shape, k
    assert "net.prev_action_embedding.weight" in ours and ours["net.prev_action_embedding.weight"].shape == (32, 5)


def test_rollout_storage_box_shapes():
    import habitat_lab_b200 as hb
    from habitat_lab_b200.synthetic import pointnav_spaces
    obs, _ = pointnav_spaces(32, 32)
    pol = SimpleNamespace(num_recurrent_layers=4, recurrent_hidden_size=16)
    st = hb.RolloutStorage(6, 3, obs, hb.spaces.Box(-1.0, 1.0, (4,)), pol)
    for k in ("actions", "prev_actions"):
        assert st.buffers[k].shape == (7, 3, 4) and st.buffers[k].dtype == torch.float32
    st = hb.RolloutStorage(6, 3, obs, hb.spaces.Discrete(4), pol)
    assert st.buffers["actions"].shape == (7, 3, 1) and st.buffers["actions"].dtype == torch.int64


def test_not_implemented_combinations():
    import habitat_lab_b200 as hb
    from habitat_lab_b200.common.rollout_storage import get_action_space_info
    from habitat_lab_b200.rl.ppo_trainer import make_config
    from habitat_lab_b200.rl.single_agent_access_mgr import SingleAgentAccessMgr
    from habitat_lab_b200.synthetic import pointnav_spaces
    obs, disc = pointnav_spaces(32, 32)
    box = hb.spaces.Box(-1.0, 1.0, (2,))
    with pytest.raises(NotImplementedError):
        hb.PPO(SimpleNamespace(), 0.2, 1, 1, 0.5, 0.01, use_adaptive_entropy_pen=True)
    cfg = make_config(continuous_actions=2)
    with pytest.raises(NotImplementedError):
        hb.PointNavBaselinePolicy.from_config(cfg, obs, box)
    cfg = make_config(continuous_actions=2, ddppo=dict(train_encoder=False))
    env = SimpleNamespace(observation_space=obs, action_space=box, orig_action_space=box)
    with pytest.raises(NotImplementedError, match="gaussian"):
        SingleAgentAccessMgr(cfg, env, False, torch.device("cpu"), lambda: 0.0)
    multi = type("MultiDiscrete", (), {"shape": (2,), "nvec": [3, 3]})()
    for sp in (multi, hb.spaces.Dict(a=box)):
        with pytest.raises(NotImplementedError):
            get_action_space_info(sp)
        with pytest.raises(NotImplementedError):
            hb.PointNavResNetPolicy(obs, sp, hidden_size=32,
                                    policy_config=SimpleNamespace(action_distribution_type="gaussian"))
    with pytest.raises(NotImplementedError):   # gaussian needs a Box, categorical a Discrete
        hb.PointNavResNetPolicy(obs, disc, hidden_size=32, policy_config=SimpleNamespace(action_distribution_type="gaussian"))


def test_make_config_default_unchanged():
    from habitat_lab_b200.rl.ppo_trainer import SyntheticVectorEnvFactory, make_config
    cfg = make_config()
    agent = cfg.habitat_baselines.rl.policy["main_agent"]
    assert agent.action_distribution_type == "categorical" and not hasattr(agent, "action_dist")
    env = SyntheticVectorEnvFactory().construct_envs(cfg, device=torch.device("cpu"))
    assert type(env.action_spaces[0]).__name__ == "Discrete"
    cfg = make_config(continuous_actions=3, action_dist=dict(use_std_param=True))
    env = SyntheticVectorEnvFactory().construct_envs(cfg, device=torch.device("cpu"))
    assert env.action_spaces[0].shape == (3,) and float(env.action_spaces[0].low[0]) == -1.0
    assert cfg.habitat_baselines.rl.policy["main_agent"].action_dist.use_std_param
