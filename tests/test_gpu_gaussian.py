"""The Gaussian action head on the GPU: gaussian_act / gaussian_ppo_loss against the float64 restatement
(tests/gaussian_reference.py) within its per-element bars over every flag mix, action count, hidden size and batch;
clamp bounds and NaN inputs; argument refusal; the continuous previous-action embedding; GraphedActor replay; and one
trainer update on the continuous synthetic environment, bit-identical across two runs."""
import itertools
import math

import pytest
import torch

import gaussian_reference as G

pytestmark = pytest.mark.gpu

MIXES = [dict(use_log_std=lg, use_softplus=sp, use_std_param=pa, clamp_std=cl, action_activation=act)
         for lg, sp, pa, cl, act in itertools.product([True, False], [True, False], [True, False], [True, False],
                                                      ["tanh", ""])]
MIX_ID = lambda m: "".join(k[4] if k != "action_activation" else "t" for k, v in m.items() if v)  # noqa: E731


def _dev(params, x, case):
    d = torch.device("cuda")
    P = {k: None if v is None else v.to(d).contiguous() for k, v in params.items()}
    C = {k: (v.to(d).contiguous() if isinstance(v, torch.Tensor) else v) for k, v in case.items()}
    return P, x.to(d).contiguous(), C


def _run_loss(hb, P, x, C, flags, lo, hi, compute_grads=True):
    B, H = x.shape
    A = C["actions"].shape[1]
    L = P["w_mu"].shape[0]
    z = lambda *s: torch.full(s, float("nan"), device="cuda")  # noqa: E731
    out = dict(values=z(B), log_probs=z(B), entropy=z(B), metrics=z(12))
    if compute_grads:
        out.update(d_features=z(B, H), d_w_mu=z(L, H), d_b_mu=z(L), d_w_val=z(1, H), d_b_val=z(1),
                   d_std=z(A) if P["std"] is not None else None)
    ws = hb.ops.gaussian_ppo_loss_workspace(B, H, A, "cuda")
    hb.ops.gaussian_ppo_loss(x, P["w_mu"], P["b_mu"], P["std"], P["w_val"], P["b_val"], C["actions"], C["old_lp"],
                             C["adv"], C["old_v"], C["ret"], flags, lo, hi, C["clip"], C["c_v"], C["c_e"],
                             C["use_clipped_value_loss"], compute_grads, out, ws, is_coeffs=C.get("is_coeffs"))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items() if v is not None}


def _check(got, ref, bar, B):
    for k in G.COMPARED:
        if k in ref and k in got:
            r = G.ratio_to_bar(got[k].reshape(ref[k].shape), ref[k], bar[k])
            assert r <= 1.0, (k, r)
    r = G.ratio_to_bar(got["metrics"][:9], ref["metrics"][:9], bar["metrics"][:9])
    assert r <= 1.0, ("metrics", r)
    # fraction clipped: the same count of clipped frames (no frame near a boundary); the kernel rounds count / B to fp32
    assert round(float(got["metrics"][9]) * B) == round(float(ref["metrics"][9]) * B)


@pytest.mark.parametrize("mix", MIXES, ids=MIX_ID)
@pytest.mark.parametrize("A", [1, 2, 7, 16])
def test_loss_every_flag_mix(hb, mix, A):
    params, x, case, (flags, lo, hi) = G.make_case(37, 64, A, mix, seed=A, std_at_bounds=True)
    ref = G.loss(params, x, case, flags, lo, hi)
    bar = G.bars(params, x, case, flags, lo, hi, ref)
    _check(_run_loss(hb, *_dev(params, x, case), flags, lo, hi), ref, bar, 37)


@pytest.mark.parametrize("mix", [dict(), dict(use_std_param=True), dict(use_log_std=False, use_softplus=True)],
                         ids=["monolithic", "social_nav", "softplus"])
@pytest.mark.parametrize("H", [32, 64, 128, 256, 512])
@pytest.mark.parametrize("B", [1, 37, 4096])
def test_loss_shapes(hb, mix, H, B):
    A = 7
    params, x, case, (flags, lo, hi) = G.make_case(B, H, A, mix, seed=H + B)
    case["is_coeffs"] = torch.rand(B, generator=torch.Generator().manual_seed(B)) * 1.5
    ref = G.loss(params, x, case, flags, lo, hi)
    bar = G.bars(params, x, case, flags, lo, hi, ref)
    got = _run_loss(hb, *_dev(params, x, case), flags, lo, hi)
    _check(got, ref, bar, B)
    again = _run_loss(hb, *_dev(params, x, case), flags, lo, hi)
    for k in got:   # frame sums in a fixed order: the same bits every run
        assert torch.equal(got[k].nan_to_num(1234.5), again[k].nan_to_num(1234.5)), k


@pytest.mark.parametrize("what", ["features", "action", "old_log_prob", "std_param"])
def test_loss_nan_reaches_what_autograd_reaches(hb, what):
    mix = dict(use_std_param=True) if what == "std_param" else dict()
    params, x, case, (flags, lo, hi) = G.make_case(37, 64, 3, mix, seed=9)
    if what == "features":
        x[5, 3] = float("nan")
    elif what == "action":
        case["actions"][6, 1] = float("nan")
    elif what == "old_log_prob":
        case["old_lp"][7] = float("nan")
    else:
        params["std"][1] = float("nan")
    ref = G.loss(params, x, case, flags, lo, hi)
    got = _run_loss(hb, *_dev(params, x, case), flags, lo, hi)
    for k in G.COMPARED:
        if k in ref:
            assert torch.equal(torch.isnan(got[k].reshape(ref[k].shape)), torch.isnan(ref[k])), k
    assert torch.equal(torch.isnan(got["metrics"][:11]), torch.isnan(ref["metrics"]))


@pytest.mark.parametrize("mix", MIXES[::3], ids=MIX_ID)
@pytest.mark.parametrize("H", [32, 512])
@pytest.mark.parametrize("B", [1, 64, 4096])
def test_act_tail(hb, mix, H, B):
    """actions = mu + eps * std for a given eps (mu when eps is NULL), their log-probability and the value"""
    A = 5
    params, x, case, (flags, lo, hi) = G.make_case(B, H, A, mix, seed=B + H)
    eps = torch.randn(B, A, generator=torch.Generator().manual_seed(3))
    P, xd, _ = _dev(params, x, case)
    for e in (None, eps):
        ref, bar = G.act_bars(params, x, flags, lo, hi, e)
        a = torch.full((B, A), float("nan"), device="cuda")
        lp, v = torch.full((B,), float("nan"), device="cuda"), torch.full((B,), float("nan"), device="cuda")
        hb.ops.gaussian_act(xd, P["w_mu"], P["b_mu"], P["std"], P["w_val"], P["b_val"],
                            None if e is None else e.cuda(), flags, lo, hi, a, lp, v)
        torch.cuda.synchronize()
        for k, t in (("actions", a), ("log_probs", lp), ("values", v)):
            r = G.ratio_to_bar(t.cpu(), ref[k], bar[k])
            assert r <= 1.0, (k, e is None, r)


def test_bad_arguments_refused_before_writing(hb):
    from habitat_lab_b200 import Hb200Error
    params, x, case, (flags, lo, hi) = G.make_case(8, 64, 3, dict(), seed=1)
    P, xd, C = _dev(params, x, case)
    a = torch.full((8, 3), 7.0, device="cuda")
    lp, v = torch.full((8,), 7.0, device="cuda"), torch.full((8,), 7.0, device="cuda")
    bad = [dict(x=xd[:, :48].contiguous()), dict(flags=flags | 64), dict(std=torch.zeros(3, device="cuda")),
           dict(a=torch.full((8, 17), 7.0, device="cuda"))]
    for b in bad:
        with pytest.raises(Hb200Error):
            hb.ops.gaussian_act(b.get("x", xd), P["w_mu"], P["b_mu"], b.get("std", P["std"]), P["w_val"], P["b_val"],
                                None, b.get("flags", flags), lo, hi, b.get("a", a), lp, v)
    torch.cuda.synchronize()
    assert bool((a == 7).all() and (lp == 7).all() and (v == 7).all())
    metrics = torch.full((12,), 7.0, device="cuda")
    with pytest.raises(Hb200Error):
        hb.ops.gaussian_ppo_loss(xd, P["w_mu"], P["b_mu"], P["std"], P["w_val"], P["b_val"], C["actions"], C["old_lp"],
                                 C["adv"], C["old_v"], C["ret"], flags, lo, hi, 0.2, 0.5, 0.01, True, True,
                                 dict(metrics=metrics), hb.ops.gaussian_ppo_loss_workspace(8, 64, 3, "cuda"))
    torch.cuda.synchronize()
    assert bool((metrics == 7).all())


def test_prev_action_linear(hb):
    """Linear(A, 32)(masks * prev_actions) into the RNN-input columns, and its weight gradient in a fixed order"""
    g = torch.Generator().manual_seed(0)
    B, A, ld, col = 300, 5, 100, 40
    pa, m = torch.randn(B, A, generator=g), torch.rand(B, generator=g) > 0.3
    w, b = torch.randn(32, A, generator=g), torch.randn(32, generator=g)
    dout = torch.randn(B, ld, generator=g)
    out = torch.zeros(B, ld, device="cuda")
    hb.ops.prev_action_linear_fwd(pa.cuda(), m.cuda(), w.cuda(), b.cuda(), out, col)
    xin = (m[:, None].double() * pa.double())
    ref = xin @ w.double().T + b.double()
    bar = 16 * G.U * ((xin.abs() @ w.double().abs().T) + b.double().abs()) * A ** 0.5
    assert G.ratio_to_bar(out[:, col:col + 32].cpu(), ref, bar) <= 1.0
    assert bool((out[:, :col] == 0).all() and (out[:, col + 32:] == 0).all())
    dw, db = torch.zeros(32, A, device="cuda"), torch.zeros(32, device="cuda")
    outs = []
    for _ in range(2):
        dw.zero_(), db.zero_()
        hb.ops.prev_action_linear_bwd(pa.cuda(), m.cuda(), dout.cuda(), col, dw, db)
        outs.append((dw.cpu().clone(), db.cpu().clone()))
    d = dout[:, col:col + 32].double()
    rw, rb = d.T @ xin, d.sum(0)
    bw = 16 * G.U * B ** 0.5 * (d.abs().T @ xin.abs())
    bb = 16 * G.U * B ** 0.5 * d.abs().sum(0)
    assert G.ratio_to_bar(outs[0][0], rw, bw) <= 1.0 and G.ratio_to_bar(outs[0][1], rb, bb) <= 1.0
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def _policy(hb, A, mix, H=128):
    from types import SimpleNamespace
    from habitat_lab_b200.synthetic import pointnav_spaces
    obs, _ = pointnav_spaces(64, 64)
    pc = SimpleNamespace(action_distribution_type="gaussian", action_dist=SimpleNamespace(**mix))
    torch.manual_seed(0)
    pol = hb.PointNavResNetPolicy(obs, hb.spaces.Box(-1.0, 1.0, (A,)), hidden_size=H, num_recurrent_layers=2,
                                  rnn_type="LSTM", policy_config=pc, normalize_visual_inputs=True).cuda()
    return pol, obs


@pytest.mark.parametrize("mix", [dict(), dict(use_std_param=True)], ids=["monolithic", "social_nav"])
def test_graphed_actor_equals_eager(hb, mix):
    pol, obs = _policy(hb, 3, mix)
    pol.eval()
    N = 4
    g = torch.Generator(device="cuda").manual_seed(1)
    o = {"rgb": torch.randint(0, 256, (N, 64, 64, 3), generator=g, device="cuda", dtype=torch.uint8),
         "depth": torch.rand(N, 64, 64, 1, generator=g, device="cuda"),
         "pointgoal_with_gps_compass": torch.rand(N, 2, generator=g, device="cuda")}
    hid = torch.randn(N, pol.num_recurrent_layers, 128, generator=g, device="cuda")
    pa = torch.randn(N, 3, generator=g, device="cuda")
    mk = torch.tensor([True, False, True, True], device="cuda").view(N, 1)
    ga = hb.GraphedActor(pol, o, hid, pa, mk, deterministic=True)
    got = ga(o, hid, pa, mk)
    ref = pol.act(o, hid, pa, mk, deterministic=True)
    for k in ("actions", "values", "action_log_probs", "rnn_hidden_states"):
        assert torch.equal(getattr(got, k), getattr(ref, k)), k
    assert getattr(got, "actions").shape == (N, 3)


def _train_once(hb):
    from habitat_lab_b200.rl.ppo_trainer import PPOTrainer, make_config
    cfg = make_config(num_environments=4, num_updates=1, height=64, width=64, seed=11, continuous_actions=3,
                      action_dist=dict(use_std_param=True), num_steps=8, num_mini_batch=1, ppo_epoch=1,
                      hidden_size=128)
    tr = PPOTrainer(cfg)
    tr._init_train()
    for _ in range(8):
        tr._rollout_step()
    losses = tr._update_agent()
    torch.cuda.synchronize()
    acts = tr.rollouts.buffers["actions"][:8].clone()
    return tr.actor_critic.flatten_parameters_()["params"].clone(), losses, acts, tr


def test_trainer_update_continuous_is_deterministic(hb):
    p1, l1, a1, tr = _train_once(hb)
    p2, l2, a2, _ = _train_once(hb)
    assert torch.equal(p1, p2)
    assert l1 == l2
    assert a1.dtype == torch.float32 and a1.shape[-1] == 3 and torch.isfinite(a1).all()
    assert torch.equal(a1, a2)
    assert torch.isfinite(p1).all()
    ac = tr.actor_critic
    assert ac.action_distribution.std.grad is not None and ac.action_distribution.std.grad.abs().sum() > 0


# ---- the whole gaussian policy against the unmodified reference (tests/golden/make_golden_gaussian.py) --------------
def _golden_policy(hb, name):
    from types import SimpleNamespace
    from helpers import load_golden, recipe_state_dict
    from make_golden_gaussian import continuous_rollout
    from habitat_lab_b200.synthetic import pointnav_spaces
    Gd = load_golden(name)
    c = Gd["case"]
    obs_space, _ = pointnav_spaces(c["H"], c["W"])
    act_space = hb.spaces.Box(-1.0, 1.0, (3,))
    pc = SimpleNamespace(action_distribution_type="gaussian", action_dist=SimpleNamespace(**c["action_dist"]))
    pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=c["layers"],
                                  rnn_type="LSTM", resnet_baseplanes=32, backbone="resnet18",
                                  normalize_visual_inputs=True, policy_config=pc)
    shapes = {k: tuple(v.shape) for k, v in pol.state_dict().items()}
    assert shapes == {k: tuple(v) for k, v in Gd["shapes"].items()}, "state_dict layout differs from the reference"
    pol.load_state_dict(recipe_state_dict(Gd["shapes"], c["seed"]))
    pol.to("cuda")
    st = hb.RolloutStorage(c["T"], c["N"], obs_space, act_space, pol)
    bufs, next_value = continuous_rollout(c, 3)
    for k, v in bufs["observations"].items():
        st.buffers["observations"][k].copy_(v)
    for k in ("recurrent_hidden_states", "masks", "rewards", "value_preds", "returns", "action_log_probs", "actions",
              "prev_actions"):
        st.buffers[k].copy_(bufs[k])
    st.current_rollout_step_idxs = [c["T"]]
    st.to("cuda")
    return Gd, pol, st, next_value.cuda(), c


def _cos(a, b):
    a, b = a.flatten().double().cpu(), b.flatten().double().cpu()
    return float(a @ b / (a.norm() * b.norm() + 1e-30))


@pytest.mark.parametrize("name", ["gaussian_monolithic", "gaussian_social_nav"])
def test_policy_minibatch_vs_reference(hb, name):
    """evaluate + loss + backward of the whole gaussian policy (conv stack, continuous previous-action input, LSTM,
    Gaussian head) vs the reference; tolerances as tests/test_gpu_policy.py's for the 8-frame fixtures (fp16 / bf16
    conv stack, TF32 dense layers)"""
    Gd, pol, st, _, c = _golden_policy(hb, name)
    pol.train()
    st.buffers["value_preds"].copy_(Gd["value_preds_after"])
    st.buffers["returns"].copy_(Gd["returns"])
    torch.manual_seed(Gd["mb_env_inds_seed"])
    batch = next(iter(st.data_generator(Gd["advantages"].cuda(), 1)))
    metrics = pol.loss_and_backward(batch, 0.2, 0.5, 0.01, True).cpu()
    torch.cuda.synchronize()
    last = pol._last
    assert (last["values"].cpu() - Gd["eval_values"].view(-1)).abs().max().item() < 5e-3
    assert (last["log_probs"].cpu() - Gd["eval_log_probs"].view(-1)).abs().max().item() < 5e-3
    assert (last["entropy"].cpu() - Gd["eval_entropy"].view(-1)).abs().max().item() < 5e-4
    assert (last["hidden_out"].cpu() - Gd["eval_hidden"]).abs().max().item() < 5e-3
    L = Gd["mb_losses"]
    got = dict(value_loss=metrics[0].item(), action_loss=metrics[1].item(), dist_entropy=metrics[2].item(),
               total=metrics[10].item())
    for k in got:
        assert got[k] == pytest.approx(L[k], rel=1e-3, abs=2e-4), (k, got[k], L[k])
    bad = []
    for k, prm in pol.named_parameters():
        gn_ref, gn = Gd["grad_norms"][k], prm.grad.norm().item()
        tol = (0.20 if prm.dim() == 1 else 0.15) if "visual_encoder" in k else 2e-2
        if abs(gn - gn_ref) > tol * gn_ref + 1e-7:
            bad.append((k, gn, gn_ref))
    assert not bad, bad
    # the head, the critic and the previous-action embedding whole: d_std and the Linear(A, 32) gradient included
    for k, g_ref in Gd["grads_small"].items():
        g = dict(pol.named_parameters())[k].grad
        assert _cos(g, g_ref) > 0.999, (k, _cos(g, g_ref))


@pytest.mark.parametrize("name", ["gaussian_monolithic", "gaussian_social_nav"])
def test_policy_ppo_update_vs_reference(hb, name):
    """one PPO.update (GAE, minibatch, loss + backward, clip + Adam) vs the reference: metrics and the parameters after
    the step (the std parameter through the flat buffer and FusedAdam)"""
    Gd, pol, st, next_value, c = _golden_policy(hb, name)
    pol.train()
    ppo = hb.PPO(pol, clip_param=0.2, ppo_epoch=1, num_mini_batch=1, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4,
                 eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True, use_normalized_advantage=False)
    st.compute_returns(next_value, True, 0.99, 0.95)
    torch.manual_seed(2000 + c["seed"])
    metrics = ppo.update(st)
    ref = Gd["update_metrics"]
    for k in ("value_loss", "action_loss", "dist_entropy"):
        assert metrics[k] == pytest.approx(ref[k], rel=5e-3, abs=5e-4), k
    for k in ("value_pred_mean", "prob_ratio_mean", "value_pred_min", "value_pred_max", "prob_ratio_min", "prob_ratio_max"):
        assert metrics[k] == pytest.approx(ref[k], rel=2e-2, abs=2e-2), k
    assert metrics["grad_norm"] == pytest.approx(ref["grad_norm"], rel=3e-2)
    assert metrics["ppo_fraction_clipped"] == pytest.approx(ref["ppo_fraction_clipped"], abs=0.13)   # one frame of 8
    sd = pol.state_dict()
    for k, n_ref in Gd["param_norms_after_update"].items():
        worst = 2 * 2.5e-4 * math.sqrt(sd[k].numel())
        assert sd[k].float().norm().item() == pytest.approx(n_ref, rel=1e-3, abs=0.25 * worst + 1e-5), k
    # Adam's first step moves each element by about lr * sign(gradient): elements may differ by 2 lr only where the
    # two gradients' signs differ, which the gradient check above allows for a few elements at most
    for k, p_ref in Gd["params_small_after_update"].items():
        far = ((sd[k].cpu() - p_ref).abs() > 0.5 * 2.5e-4).float().mean().item()
        assert far <= 0.02, (k, far)
    if "action_distribution.std" in Gd["params_small_after_update"]:
        from helpers import recipe_state_dict
        before = recipe_state_dict(Gd["shapes"], c["seed"])["action_distribution.std"]
        assert not torch.equal(sd["action_distribution.std"].cpu(), before)   # FusedAdam moved the std parameter
