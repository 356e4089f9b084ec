"""CPU checks of the float64 references that tests/test_gpu_ppo_tail.py judges the PPO tail kernels by, and of their
bars: the references equal the oracle (compute_returns / get_advantages, fp32 autograd of ppo_loss) and torch's own
clip_grad_norm_ + Adam, fp32 restatements stay within every bar, every perturbed reference misses it by at least 10x,
and the NaN table: which outputs a NaN in each input reaches."""
import math

import pytest
import torch

import ppo_reference as R
from oracle import torch_oracle as O


def _rollout(T, N, Ta, seed, p_done=1 / 25):
    g = torch.Generator().manual_seed(seed)
    masks = torch.rand(Ta, N, generator=g) > p_done
    rewards = torch.randn(Ta, N, generator=g) * 0.1 + 2.5 * (~masks).float()
    values = torch.randn(Ta, N, generator=g)
    stale = torch.randn(Ta, N, generator=g)
    stale[Ta - 1, 0] = math.inf
    return rewards, values, masks, torch.randn(N, generator=g), stale


@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("T,N,Ta", [(1, 3, 2), (33, 5, 36), (70, 4, 71)])
def test_gae_reference_is_oracle(T, N, Ta, use_gae):
    """float64 GAE = oracle.compute_returns + get_advantages in float64 (stale rows kept, bootstrap row written)"""
    r, v, m, nv, stale = _rollout(T, N, Ta, T + N)
    ref = R.gae(r, v, m, nv, stale, T, 0.99, 0.95, use_gae)
    g, gt = R.gae_discounts(0.99, 0.95)
    d = lambda t: t.double().unsqueeze(-1)  # noqa: E731
    vo = d(v).clone()
    ro = O.compute_returns(d(r), vo, m.unsqueeze(-1), d(nv), T, use_gae, g, gt / g)
    keep = torch.ones(Ta, dtype=torch.bool)
    keep[: T + (0 if use_gae else 1)] = False
    ro = torch.where(keep.view(-1, 1, 1), d(stale), ro).squeeze(-1)
    torch.testing.assert_close(ref["returns"], ro, rtol=1e-12, atol=1e-12, equal_nan=True)
    ao = O.get_advantages(ro, vo.squeeze(-1), normalize=False)
    torch.testing.assert_close(ref["adv"][:T], ao[:T], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["values"].double(), vo.squeeze(-1), rtol=0, atol=0)


@pytest.mark.parametrize("gamma,tau", [(0.99, 0.95), (1.0, 1.0)])
@pytest.mark.parametrize("T,N,pattern", [(2, 3, "random"), (31, 4, "random"), (65, 5, "random"), (128, 9, "random"),
                                         (256, 3, "random"), (64, 4, "chunk_bounds"), (128, 3, "ones")])
def test_gae_bars(T, N, pattern, gamma, tau):
    """the fp32 recurrence stays within the bar, and every perturbation that changes the result misses it 10x"""
    r, v, m, nv, stale = _rollout(T, N, T + 2, 3 * T + N)
    if pattern == "chunk_bounds":
        m[(T + 31) // 32 :: (T + 31) // 32] = False
    elif pattern == "ones":
        m[:] = True
    ref = R.gae(r, v, m, nv, stale, T, gamma, tau)
    f = R.gae(r, v, m, nv, stale, T, gamma, tau, dtype=torch.float32)
    ratio = max(R.ratio_to_bar(f[k], ref[k], ref["bar"]) for k in ("returns", "adv"))
    guards = {}
    for p in R.GAE_PERTURBATIONS:
        pr = R.gae(r, v, m, nv, stale, T, gamma, tau, perturb=p)
        if pr is not None and not torch.equal(pr["returns"], ref["returns"]):
            guards[p] = R.ratio_to_bar(pr["returns"], ref["returns"], ref["bar"])
    print(f"  GAE T{T} N{N} {pattern} g{gamma} t{tau}: fp32 / bar {ratio:.3g}; perturbed / bar {guards}")
    assert ratio <= 1.0
    assert guards and min(guards.values()) >= 10.0, guards
    if gamma != tau == 0.95:
        assert "gamma_for_gt" in guards


@pytest.mark.parametrize("n", [7, 1000, 16384])
def test_adv_normalize_bars(n):
    """both normalisation modes equal oracle.get_advantages; fp32 stays within the bar, perturbations miss it 10x"""
    g = torch.Generator().manual_seed(n)
    adv = 0.1 * torch.randn(n, generator=g) + 0.03
    adv[0] = math.inf
    ref, bar = R.adv_normalize(adv)
    o = O.get_advantages(adv.double(), torch.zeros(n, dtype=torch.float64), normalize=True)
    torch.testing.assert_close(ref[1:], o[1:], rtol=1e-9, atol=1e-12)   # eps: fp32 1e-5 against 1e-5
    mv = torch.tensor([0.02, 0.013])
    ref1, bar1 = R.adv_normalize(adv, mean_var=mv)
    o1 = O.get_advantages(adv.double(), torch.zeros(n, dtype=torch.float64), True, (mv[1].double(), mv[0].double()))
    torch.testing.assert_close(ref1[1:], o1[1:], rtol=1e-6, atol=1e-9)   # O adds eps in double, the kernel in fp32
    f, _ = R.adv_normalize(adv, dtype=torch.float32)
    ratios = [R.ratio_to_bar(f, ref, bar)]
    guards = {p: R.ratio_to_bar(R.adv_normalize(adv, perturb=p)[0], ref, bar) for p in R.NORM_PERTURBATIONS}
    print(f"  normalize n{n}: fp32 / bar {ratios}; perturbed / bar {guards}")
    assert max(ratios) <= 1.0
    assert guards["eps_outside"] >= 10.0
    if n - 1 <= 2 ** 14:
        assert guards["biased_var"] >= 10.0


def _loss_args(c, clip_v=True):
    return (c["feat"], c["w_act"], c["b_act"], c["w_val"], c["b_val"], c["actions"], c["old_lp"], c["adv"],
            c["old_v"], c["ret"], c["is_coeffs"], 0.2, 0.5, 0.01, clip_v)


@pytest.mark.parametrize("is_mode", ["none", "rand"])
@pytest.mark.parametrize("clip_v", [True, False])
def test_loss_reference_is_oracle(is_mode, clip_v):
    """float64 reference = fp32 autograd of oracle.heads + ppo_loss, to fp32 accuracy"""
    c = _without_fp32_ties(R.make_loss_case(96, 64, 4, seed=1, is_mode=is_mode))
    ref = R.ppo_loss(*_loss_args(c, clip_v))
    req = [t.clone().requires_grad_(True) for t in (c["feat"], c["w_act"], c["b_act"], c["w_val"], c["b_val"])]
    v, lp, ent = O.heads(*req, c["actions"])
    batch = dict(action_log_probs=c["old_lp"].view(-1, 1), advantages=c["adv"].view(-1, 1),
                 value_preds=c["old_v"].view(-1, 1), returns=c["ret"].view(-1, 1))
    if c["is_coeffs"] is not None:
        batch["is_coeffs"] = c["is_coeffs"].view(-1, 1)
    o = O.ppo_loss(v, lp, ent, batch, R.f32(0.2), R.f32(0.5), R.f32(0.01), clip_v)
    o["total_loss"].backward()
    got = dict(zip(R.GRADS, (t.grad for t in req)), values=v, log_probs=lp, entropy=ent)
    got.update({k: o[k].detach() for k in R.METRICS})
    ratios = R.loss_ratios(got, ref)
    assert max(ratios.values()) <= 1.0, ratios


def _without_fp32_ties(c, clip=0.2):
    """the case without frames whose fp32 ratio is within 1e-5 of 1 +- clip: there the two fp32 surrogates can round
    to the same value, and torch's autograd then splits the gradient of torch.min between them, where the kernel
    gives it to the unclipped one (the float64 reference does not tie on them)"""
    lp = R.heads(c["feat"], c["w_act"], c["b_act"], c["w_val"], c["b_val"], dtype=torch.float32)["logp"]
    ratio = torch.exp(lp.gather(1, c["actions"].view(-1, 1)).view(-1) - c["old_lp"])
    one, cl = torch.tensor(1.0), torch.tensor(R.f32(clip))
    keep = ((ratio - (one - cl)).abs() > 1e-5) & ((ratio - (one + cl)).abs() > 1e-5)
    return {k: (v[keep] if k in ("feat", "actions", "old_lp", "adv", "old_v", "ret", "is_coeffs") and v is not None
                else v) for k, v in c.items()}


@pytest.mark.parametrize("large", [False, True], ids=["ordinary", "large_logits"])
@pytest.mark.parametrize("B,H,A,is_mode,clip_v", [(64, 32, 1, "none", True), (96, 64, 4, "rand", True),
                                                  (80, 128, 8, "ones", False), (130, 512, 2, "none", True)])
def test_loss_bars(B, H, A, is_mode, clip_v, large):
    """the fp32 restatement stays within every bar, and every loss perturbation misses its bar 10x"""
    c = _without_fp32_ties(R.make_loss_case(B, H, A, seed=B + H, is_mode=is_mode, b_act_zero=(A == 8),
                                            large_logits=large))
    ref = R.ppo_loss(*_loss_args(c, clip_v))
    f = R.ppo_loss(*_loss_args(c, clip_v), dtype=torch.float32)
    ratios = R.loss_ratios(f, ref)
    guards = {}
    for p in R.LOSS_PERTURBATIONS:
        pg = R.perturb_grads(ref, p)
        if pg is not None:
            guards[p] = max(R.ratio_to_bar(pg[k], ref[k], ref["bars"][k]) for k in R.GRADS)
    wguards = R.weight_grad_guards(ref)
    print(f"  loss B{B} H{H} A{A} {is_mode}: fp32 / bar max {max(ratios.values()):.3g}; perturbed / bar {guards}; "
          f"weight-gradient faults / bar {wguards}")
    if not large:   # (frames at |z| ~ 1e3 set the weight-gradient bars; see make_loss_case)
        assert wguards and min(wguards.values()) >= 10.0, wguards
    assert ratios.pop("ppo_fraction_clipped") <= 1.0   # whole frames: only the ambiguous ones may differ
    assert max(ratios.values()) <= 1.0, ratios
    assert "entropy_no_h" in guards or A == 1
    assert "grad_through_clip" in guards or A == 1   # A = 1: p = 1, no logit gradient at all
    assert not guards or min(guards.values()) >= 10.0, guards


@pytest.mark.parametrize("wd,gs,mx,step", [(0.0, 1.0, 0.2, 1), (0.01, 0.5, 0.2, 2), (0.0, 1 / 3, 1e9, 10),
                                          (0.01, 1.0, 0.0, 10000)])
def test_adam_reference_is_torch(wd, gs, mx, step):
    """float64 clip_adam = torch's clip_grad_norm_ + Adam (foreach) in float64 after step - 1 earlier steps"""
    gen = torch.Generator().manual_seed(step)
    n = 1003
    p = torch.randn(n, generator=gen)
    m = torch.randn(n, generator=gen) * 1e-3
    v = torch.rand(n, generator=gen) * 1e-5
    g = torch.randn(n, generator=gen) * 0.05
    ref = R.clip_adam(p, g, m, v, 2.5e-4, (0.9, 0.999), 1e-5, wd, mx, gs, step)
    tp = torch.nn.Parameter(p.double().clone())
    opt = torch.optim.Adam([tp], lr=R.f32(2.5e-4), betas=(R.f32(0.9), R.f32(0.999)), eps=R.f32(1e-5),
                           weight_decay=R.f32(wd), foreach=True)
    tp.grad = g.double() * R.f32(gs)
    norm = torch.nn.utils.clip_grad_norm_([tp], R.f32(mx)) if mx > 0 else None
    opt.step()   # initialise state, then overwrite it with the given moments and step
    st = opt.state[tp]
    tp.data.copy_(p.double())
    st["exp_avg"].copy_(m.double())
    st["exp_avg_sq"].copy_(v.double())
    st["step"].fill_(step - 1)
    tp.grad = g.double() * R.f32(gs)
    if mx > 0:
        norm = torch.nn.utils.clip_grad_norm_([tp], R.f32(mx))
        torch.testing.assert_close(ref["norm"], norm, rtol=1e-14, atol=0)
    opt.step()
    for k, t in (("params", tp.detach()), ("exp_avg", st["exp_avg"]), ("exp_avg_sq", st["exp_avg_sq"])):
        torch.testing.assert_close(ref[k], t, rtol=1e-12, atol=1e-15, msg=lambda s, k=k: f"{k}: {s}")
    f = R.clip_adam(p, g, m, v, 2.5e-4, (0.9, 0.999), 1e-5, wd, mx, gs, step, dtype=torch.float32)
    ratios = {k: R.ratio_to_bar(f[k], ref[k], ref["bar_" + k]) for k in ("params", "exp_avg", "exp_avg_sq", "norm")}
    guards = {}
    for pt in R.ADAM_PERTURBATIONS:
        pr = R.clip_adam(p, g, m, v, 2.5e-4, (0.9, 0.999), 1e-5, wd, mx, gs, step, perturb=pt)
        if pr is not None and not torch.equal(pr["params"], ref["params"]):
            guards[pt] = R.ratio_to_bar(pr["params"], ref["params"], ref["bar_params"])
    print(f"  adam wd{wd} gs{gs:.3g} mx{mx} step{step}: fp32 / bar {ratios}; perturbed / bar {guards}")
    assert max(ratios.values()) <= 1.0
    assert guards["eps_in_sqrt"] >= 10.0
    if step <= 10:
        assert guards["bias_step"] >= 10.0
    if "scale_after_norm" in guards:
        assert guards["scale_after_norm"] >= 10.0


# ---------------------------------------------------------------------------------------------------------------------
# the NaN table
# ---------------------------------------------------------------------------------------------------------------------
NAN_FRAME = 5
# injection -> (frame outputs at NAN_FRAME that become NaN, metrics that become NaN, gradients that become NaN:
#               "row" = the d_features row of NAN_FRAME only, "all" = every element)
NAN_TABLE = {
    "feature_row": ({"values", "log_probs", "entropy"},
                    {"value_loss", "action_loss", "dist_entropy", "value_pred_min", "value_pred_mean",
                     "value_pred_max", "prob_ratio_min", "prob_ratio_mean", "prob_ratio_max", "total_loss"},
                    {"d_features": "row", "d_w_act": "all", "d_b_act": "all", "d_w_val": "all"}),
    "old_log_prob": (set(), {"action_loss", "prob_ratio_min", "prob_ratio_mean", "prob_ratio_max", "total_loss"},
                     {"d_features": "row", "d_w_act": "all", "d_b_act": "all"}),
    "advantage": (set(), {"action_loss", "total_loss"}, {"d_features": "row", "d_w_act": "all", "d_b_act": "all"}),
    "old_value": (set(), {"value_loss", "total_loss"}, {}),
    "return": (set(), {"value_loss", "total_loss"},
               {"d_features": "row", "d_w_val": "all", "d_b_val": "all"}),
    "is_coeff": (set(), {"value_loss", "action_loss", "dist_entropy", "total_loss"},
                 {"d_features": "row", "d_w_act": "all", "d_b_act": "all", "d_w_val": "all", "d_b_val": "all"}),
    "bad_action": ({"log_probs"}, {"action_loss", "prob_ratio_min", "prob_ratio_mean", "prob_ratio_max", "total_loss"},
                   {"d_features": "row", "d_w_act": "all", "d_b_act": "all"}),
}


def nan_case(inject, B=64, H=32, A=4, bad_action=None):
    """a loss case with frame NAN_FRAME poisoned by `inject` (the frame's value is in the unclipped regime, its ratio
    inside the clip range, so every path of the frame is live); bad_action: the action value for 'bad_action'"""
    c = R.make_loss_case(B, H, A, seed=11, is_mode="rand")
    f = NAN_FRAME
    c["old_lp"][f] = c["old_lp"][f] * 0 + R.heads(c["feat"], c["w_act"], c["b_act"], c["w_val"], c["b_val"])[
        "logp"][f, c["actions"][f]].float()
    c["old_v"][f] = R.heads(c["feat"], c["w_act"], c["b_act"], c["w_val"], c["b_val"])["values"][f].float()
    c["is_coeffs"][f] = 0.5
    nan = float("nan")
    if inject == "feature_row":
        c["feat"][f] = nan
    elif inject == "old_log_prob":
        c["old_lp"][f] = nan
    elif inject == "advantage":
        c["adv"][f] = nan
    elif inject == "old_value":
        c["old_v"][f] = nan
    elif inject == "return":
        c["ret"][f] = nan
    elif inject == "is_coeff":
        c["is_coeffs"][f] = nan
    elif inject == "bad_action":
        c["actions"][f] = A if bad_action is None else bad_action
    return c


def nan_pattern(out, B):
    """{output: 'none' / 'row' / 'all' / 'frame'} of which elements are NaN"""
    pat = {}
    for k in ("values", "log_probs", "entropy"):
        nn_ = torch.isnan(out[k].view(-1))
        pat[k] = "frame" if (nn_.sum() == 1 and bool(nn_[NAN_FRAME])) else ("none" if not nn_.any() else "other")
    for k in R.METRICS:
        pat[k] = "nan" if bool(torch.isnan(torch.as_tensor(out[k])).any()) else "none"
    for k in R.GRADS:
        nn_ = torch.isnan(out[k])
        if not nn_.any():
            pat[k] = "none"
        elif bool(nn_.all()):
            pat[k] = "all"
        elif k == "d_features" and bool(nn_[NAN_FRAME].all()) and nn_.sum() == nn_.shape[1]:
            pat[k] = "row"
        else:
            pat[k] = "other"
    return pat


def expected_pattern(inject):
    frame, mets, grads = NAN_TABLE[inject]
    pat = {k: ("frame" if k in frame else "none") for k in ("values", "log_probs", "entropy")}
    pat.update({k: ("nan" if k in mets else "none") for k in R.METRICS})
    pat.update({k: grads.get(k, "none") for k in R.GRADS})
    return pat


@pytest.mark.parametrize("inject", list(NAN_TABLE))
def test_nan_table(inject):
    """which outputs of the float64 reference a NaN in one input reaches (use_clipped_value_loss on: an old value of
    NaN sends the frame down the clipped branch, whose value gradient is 0)"""
    for bad in ((-1, 4) if inject == "bad_action" else (None,)):
        c = nan_case(inject, bad_action=bad)
        ref = R.ppo_loss(*_loss_args(c, True))
        assert nan_pattern(ref, 64) == expected_pattern(inject)


def test_nan_table_adam():
    """one NaN gradient makes every parameter and moment NaN when clipping (clip_grad_norm_'s clamp propagates the
    NaN norm), only its own element without clipping; an inf gradient gives NaN at its element and a zero update
    elsewhere when clipping"""
    n = 1003
    gen = torch.Generator().manual_seed(0)
    p, m, v = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-3, torch.rand(n, generator=gen) * 1e-5
    g = torch.randn(n, generator=gen) * 0.05
    g[17] = math.nan
    r = R.clip_adam(p, g, m, v, 2.5e-4, (0.9, 0.999), 1e-5, 0.0, 0.2, 1.0, 3)
    assert all(bool(torch.isnan(r[k]).all()) for k in ("params", "exp_avg", "exp_avg_sq", "norm"))
    r = R.clip_adam(p, g, m, v, 2.5e-4, (0.9, 0.999), 1e-5, 0.0, 0.0, 1.0, 3)
    for k in ("params", "exp_avg", "exp_avg_sq"):
        assert torch.isnan(r[k]).nonzero().view(-1).tolist() == [17]
    g[17] = math.inf
    r = R.clip_adam(p, g, m, v, 2.5e-4, (0.9, 0.999), 1e-5, 0.0, 0.2, 1.0, 3)
    tp = torch.nn.Parameter(p.double().clone())
    tp.grad = g.double().clone()
    torch.nn.utils.clip_grad_norm_([tp], R.f32(0.2))
    torch.testing.assert_close(tp.grad, g.double() * 0 * torch.where(torch.isinf(g), math.nan, 1.0).double(),
                               equal_nan=True)
    assert torch.isnan(r["params"]).nonzero().view(-1).tolist() == [17]
    assert bool(torch.isinf(r["norm"]))
