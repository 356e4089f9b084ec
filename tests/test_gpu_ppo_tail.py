"""GPU parity of the PPO tail kernels (csrc/rl_kernels.cu: GAE, adv_normalize, PPO loss, grad_sqnorm + clip_adam;
csrc/elementwise.cu: heads_fwd, heads_act) against the float64 references and bars of tests/ppo_reference.py.

Every case also runs the perturbed references of its kernel and requires each that changes the exact result to miss
the bar by at least 10x, so a bar too loose to see those faults fails here.  NaN inputs must reach exactly the outputs
the reference's NaN table (tests/test_ppo_reference_cpu.py) names, and leave every other output bit-identical to a
clean run.
"""
import math

import pytest
import torch

import ppo_reference as R
from test_ppo_reference_cpu import NAN_FRAME, NAN_TABLE, _loss_args, expected_pattern, nan_case, nan_pattern

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

DEV = "cuda"


def _gpu(t):
    return None if t is None else t.to(DEV).contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# GAE
# ---------------------------------------------------------------------------------------------------------------------
def _rollout(T, N, pattern, seed, extra=3):
    """fp32 [Ta, N] operands with Ta = T + 1 + extra (t_cur < t_alloc - 1) and non-finite stale rows"""
    Ta = T + 1 + extra
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(Ta, N, generator=g) > 1 / 25
    L = (T + 31) // 32
    if pattern == "ones":
        m[:] = True
    elif pattern == "zeros":
        m[:] = False
    elif pattern == "chunk_bounds":     # dones exactly where warp chunks meet
        m[:] = True
        m[L:T + 1:L] = False
    elif pattern == "ends":             # dones at t = 0 and at t = T - 1
        m[:] = True
        m[0] = False
        m[T - 1] = False
        m[T] = False
    rewards = torch.randn(Ta, N, generator=g) * 0.1 + 2.5 * (~m).float()
    values = torch.randn(Ta, N, generator=g)
    stale = torch.randn(Ta, N, generator=g)
    stale[T + 1:, 0] = math.inf
    stale[Ta - 1, N - 1] = math.nan
    values[Ta - 1, N // 2] = -math.inf
    return rewards, values, m, torch.randn(N, generator=g), stale


def _run_gae(hb, ops, c, T, gamma, tau, variant, use_gae=True):
    r, v, m, nv, stale = (_gpu(t) for t in c)
    ret, adv = stale.clone(), torch.empty_like(stale)
    stats = torch.zeros(4, dtype=torch.float64, device=DEV)
    ops.gae_adv(r, v, m, nv, ret, adv, stats, T, gamma, tau, use_gae, variant)
    torch.cuda.synchronize()
    return dict(returns=ret, adv=adv, values=v, stats=stats)


GAE_SHAPES = [(T, N, "random") for T in (1, 2, 31, 32, 33, 63, 65, 128, 256) for N in (1, 3, 4, 5, 129, 2048)] + \
    [(T, 129, p) for T in (65, 128) for p in ("ones", "zeros", "chunk_bounds", "ends")]


@pytest.mark.parametrize("gamma,tau", [(0.99, 0.95), (1.0, 1.0)], ids=["damped", "undamped"])
@pytest.mark.parametrize("T,N,pattern", GAE_SHAPES, ids=[f"T{T}-N{N}-{p}" for T, N, p in GAE_SHAPES])
def test_gae(hb, T, N, pattern, gamma, tau):
    """variant 2 (warp scan) within the bar, variant 1 within it too, variant 0 = the variant the auto rule names bit
    for bit; bootstrap / stale rows exact; the statistics' count exact and sums within their fp64 bound"""
    from habitat_lab_b200 import ops

    c = _rollout(T, N, pattern, seed=T * 7919 + N)
    ref = R.gae(*[_gpu(t) for t in c], T, gamma, tau)
    out = {vr: _run_gae(hb, ops, c, T, gamma, tau, vr) for vr in (1, 2, 0)}
    auto = 2 if (N < 8192 and T >= 32) else 1
    for k in ("returns", "adv", "values"):   # (the statistics are fp64 atomics: order-dependent in the last bits)
        assert torch.equal(out[0][k].nan_to_num(7.0), out[auto][k].nan_to_num(7.0)), k
    worst = 0.0
    for vr in (1, 2):
        for k in ("returns", "adv"):
            worst = max(worst, R.ratio_to_bar(out[vr][k], ref[k], ref["bar"]))
        assert torch.equal(out[vr]["values"], ref["values"])
        st, rs = out[vr]["stats"].tolist(), R.adv_stats(out[vr]["adv"])
        assert st[2] == rs["count"]
        assert abs(st[0] - rs["sum"]) <= rs["bar_sum"] and abs(st[1] - rs["sumsq"]) <= rs["bar_sumsq"]
    assert worst <= 1.0, worst
    guards = {}
    for p in R.GAE_PERTURBATIONS:
        pr = R.gae(*[_gpu(t) for t in c], T, gamma, tau, perturb=p)
        if pr is not None and not torch.equal(pr["returns"].nan_to_num(), ref["returns"].nan_to_num()):
            guards[p] = R.ratio_to_bar(pr["returns"], ref["returns"], ref["bar"])
    print(f"  GAE T{T} N{N} {pattern}: kernel / bar {worst:.3g}; perturbed / bar {guards}")
    assert not guards or min(guards.values()) >= 10.0, guards


@pytest.mark.parametrize("T,N", [(1, 3), (33, 5), (128, 64)])
def test_gae_without_gae(hb, T, N):
    """use_gae = 0: the discounted-return scan (always the serial kernel) within the bar"""
    from habitat_lab_b200 import ops

    c = _rollout(T, N, "random", seed=T + N)
    ref = R.gae(*[_gpu(t) for t in c], T, 0.99, 0.95, use_gae=False)
    out = _run_gae(hb, ops, c, T, 0.99, 0.95, 0, use_gae=False)
    assert R.ratio_to_bar(out["returns"], ref["returns"], ref["bar"]) <= 1.0
    assert R.ratio_to_bar(out["adv"], ref["adv"], ref["bar"]) <= 1.0


@pytest.mark.parametrize("n", [7, 1000, 16384, 262_147])
@pytest.mark.parametrize("mode", [0, 1])
def test_adv_normalize(hb, n, mode):
    """both modes within the bar (non-finite entries stay non-finite); perturbed references miss it 10x"""
    from habitat_lab_b200 import ops

    g = torch.Generator().manual_seed(n + mode)
    adv = 0.1 * torch.randn(n, generator=g) + 0.03
    adv[0] = math.inf
    a = adv.to(DEV)
    if mode == 0:
        s = R.adv_stats(a)
        stats = torch.tensor([s["sum"], s["sumsq"], s["count"], 0.0], dtype=torch.float64, device=DEV)
        ops.adv_normalize(a, stats=stats)
        ref, bar = R.adv_normalize(adv.to(DEV))
    else:
        mv = torch.tensor([0.02, 0.013])
        ops.adv_normalize(a, mean_var=mv.to(DEV))
        ref, bar = R.adv_normalize(adv.to(DEV), mean_var=mv)
    torch.cuda.synchronize()
    r = R.ratio_to_bar(a, ref, bar)
    assert r <= 1.0, r
    if mode == 0:
        guards = {p: R.ratio_to_bar(R.adv_normalize(adv.to(DEV), perturb=p)[0], ref, bar)
                  for p in R.NORM_PERTURBATIONS}
        print(f"  normalize n{n}: kernel / bar {r:.3g}; perturbed / bar {guards}")
        assert guards["eps_outside"] >= 10.0
        if n - 1 <= 2 ** 14:
            assert guards["biased_var"] >= 10.0


# ---------------------------------------------------------------------------------------------------------------------
# PPO loss
# ---------------------------------------------------------------------------------------------------------------------
def _loss_out(B, H, A, fill=None):
    e = (lambda *s: torch.full(s, fill, device=DEV)) if fill is not None else (lambda *s: torch.empty(*s, device=DEV))
    return dict(values=e(B), log_probs=e(B), entropy=e(B), d_features=e(B, H), d_w_act=e(A, H), d_b_act=e(A),
                d_w_val=e(H), d_b_val=e(1), metrics=torch.empty(12, device=DEV))


def _run_loss(ops, c, clip_v, compute_grads=True, out=None, stream=None):
    B, H = c["feat"].shape
    A = c["w_act"].shape[0]
    out = out or _loss_out(B, H, A)
    g = {k: _gpu(c[k]) for k in ("feat", "w_act", "b_act", "w_val", "b_val", "actions", "old_lp", "adv", "old_v",
                                  "ret", "is_coeffs")}
    ws = ops.ppo_loss_workspace(B, H, A, DEV)
    ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream())
    with ctx:
        ops.ppo_loss(g["feat"], g["w_act"], g["b_act"], g["w_val"].reshape(1, -1), g["b_val"], g["actions"],
                     g["old_lp"], g["adv"], g["old_v"], g["ret"], 0.2, 0.5, 0.01, clip_v, compute_grads, out, ws,
                     is_coeffs=g["is_coeffs"])
    torch.cuda.synchronize()
    res = {k: v for k, v in out.items() if k != "metrics"}
    res.update({k: out["metrics"][i] for i, k in enumerate(R.METRICS)})
    return res


def _ref_on_gpu(c, clip_v):
    return R.ppo_loss(*[_gpu(t) if isinstance(t, torch.Tensor) else t for t in _loss_args(c, clip_v)])


def _check_loss(hb, c, clip_v, label, weight_guards=True):
    from habitat_lab_b200 import ops

    got = _run_loss(ops, c, clip_v)
    ref = _ref_on_gpu(c, clip_v)
    ratios = R.loss_ratios(got, ref)
    guards = {}
    for p in R.LOSS_PERTURBATIONS:
        pg = R.perturb_grads(ref, p)
        if pg is not None:
            guards[p] = max(R.ratio_to_bar(pg[k], ref[k], ref["bars"][k]) for k in R.GRADS)
    wguards = R.weight_grad_guards(ref)
    worst = max(ratios, key=ratios.get)
    print(f"  loss {label}: worst {worst} {ratios[worst]:.3g} of the bar, {ref['n_amb']} ambiguous frames; "
          f"perturbed / bar {guards}; weight-gradient faults / bar min {min(wguards.values(), default=None)}")
    assert max(ratios.values()) <= 1.0, ratios
    assert not guards or min(guards.values()) >= 10.0, guards
    if weight_guards:
        assert wguards and min(wguards.values()) >= 10.0, wguards
    return got


LOSS_SHAPES = [(257, H, A) for H in (32, 64, 128, 256, 512) for A in (1, 2, 4, 8)] + \
    [(B, 512, A) for A in (4, 8) for B in (1, 7, 8, 9, 63, 64, 65, 2047, 2111, 2112, 2113, 4096, 16384)]


@pytest.mark.parametrize("B,H,A", LOSS_SHAPES, ids=[f"B{B}-H{H}-A{A}" for B, H, A in LOSS_SHAPES])
def test_ppo_loss_shapes(hb, B, H, A):
    """every NJ instantiation, A = 1..8, batches around the persistent grid (cdiv(B, 8) = 264 blocks at B = 2112)
    and uneven weight-gradient slabs; every frame regime of make_loss_case"""
    c = R.make_loss_case(B, H, A, seed=B * 31 + H + A, b_act_zero=(H == 512), large_logits=False)
    _check_loss(hb, c, True, f"B{B} H{H} A{A}")


LARGE_Z_SHAPES = [(257, H, A) for H in (32, 512) for A in (2, 4, 8)] + [(4096, 512, 4)]


@pytest.mark.parametrize("B,H,A", LARGE_Z_SHAPES, ids=[f"B{B}-H{H}-A{A}" for B, H, A in LARGE_Z_SHAPES])
def test_ppo_loss_large_logits(hb, B, H, A):
    """every regime of make_loss_case with frames at |z| ~ 1e3 (probabilities that underflow to 0).  Their features
    are ~1e3 times the others', so their legitimate fp32 error sets the weight-gradient bars: the faults of the
    weight-gradient path are checked by test_ppo_loss_shapes, not here"""
    c = R.make_loss_case(B, H, A, seed=B * 17 + H + A, b_act_zero=(A == 4))
    _check_loss(hb, c, True, f"large |z| B{B} H{H} A{A}", weight_guards=False)


@pytest.mark.parametrize("clip_v", [True, False], ids=["clip_v", "no_clip_v"])
@pytest.mark.parametrize("is_mode", ["none", "rand", "ones"])
def test_ppo_loss_variants(hb, clip_v, is_mode):
    c = R.make_loss_case(1000, 512, 4, seed=5, is_mode=is_mode, large_logits=False)
    _check_loss(hb, c, clip_v, f"{is_mode} clip_v={clip_v}")


def test_ppo_loss_no_grads_and_repeatable(hb):
    """compute_grads = 0 gives bit-identical forward outputs and leaves the gradient buffers untouched; two launches
    and one on a side stream are bit-identical"""
    from habitat_lab_b200 import ops

    B, H, A = 4096, 512, 4
    c = R.make_loss_case(B, H, A, seed=3, is_mode="rand")
    a = _run_loss(ops, c, True)
    b = _run_loss(ops, c, True)
    s = _run_loss(ops, c, True, stream=torch.cuda.Stream())
    for k in a:
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], s[k]), k
    sentinel = _loss_out(B, H, A, fill=-12345.0)
    n = _run_loss(ops, c, True, compute_grads=False, out=sentinel)
    for k in ("values", "log_probs", "entropy") + R.METRICS:
        assert torch.equal(n[k], a[k]), k
    for k in R.GRADS:
        assert bool((n[k] == -12345.0).all()), k


# ---------------------------------------------------------------------------------------------------------------------
# NaN propagation
# ---------------------------------------------------------------------------------------------------------------------
# outputs an injection changes without making them NaN (a NaN old value or feature row takes the value-clipped
# branch, whose value gradient is 0 instead of the clean run's)
CHANGED_FINITE = {"feature_row": {"d_b_val"}, "old_value": {"d_features", "d_w_val", "d_b_val"}}
# (those are compared with the float64 reference within their bars)


@pytest.mark.parametrize("inject", list(NAN_TABLE))
def test_ppo_loss_nan(hb, inject):
    """the kernel's NaN pattern equals the reference's NaN table (actions -1 and A for the out-of-range action), and
    every output the injection does not reach is bit-identical to the clean run"""
    from habitat_lab_b200 import ops

    clean = _run_loss(ops, nan_case(None), True)
    frame, mets, grads = NAN_TABLE[inject]
    for bad in ((-1, 4) if inject == "bad_action" else (None,)):
        got = _run_loss(ops, nan_case(inject, bad_action=bad), True)
        pat = nan_pattern({k: v.cpu() for k, v in got.items()}, 64)
        assert pat == expected_pattern(inject), (bad, pat)
        if inject in CHANGED_FINITE:
            ref = R.ppo_loss(*_loss_args(nan_case(inject, bad_action=bad), True))
            ratios = R.loss_ratios({k: v.cpu() for k, v in got.items()}, ref, keys=sorted(CHANGED_FINITE[inject]))
            assert max(ratios.values()) <= 1.0, ratios
        for k, v in got.items():
            if k in mets or grads.get(k) == "all" or k in CHANGED_FINITE.get(inject, ()) and k != "d_features":
                continue
            keep = torch.ones(v.shape[0] if v.dim() else 1, dtype=torch.bool, device=DEV)
            if k in frame or (k == "d_features" and (k in grads or k in CHANGED_FINITE.get(inject, ()))):
                keep[NAN_FRAME] = False
            assert torch.equal(v.reshape(keep.shape[0], -1)[keep], clean[k].reshape(keep.shape[0], -1)[keep]), k


def test_clip_adam_nan_and_inf(hb):
    """a NaN gradient makes every parameter and moment NaN under clipping (clip_grad_norm_'s clamp propagates it) and
    only its own element without; an inf gradient gives what torch gives: NaN at that element under clipping"""
    from habitat_lab_b200 import ops

    n = 1003
    gen = torch.Generator().manual_seed(0)
    p, m, v = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-3, torch.rand(n, generator=gen) * 1e-5
    for val, mx in ((math.nan, 0.2), (math.nan, 0.0), (math.inf, 0.2), (math.inf, 0.0)):
        g = torch.randn(n, generator=gen) * 0.05
        g[17] = val
        got = _run_adam(ops, p, g, m, v, 2.5e-4, 0.0, mx, 1.0, 3)
        ref = R.clip_adam(p, g, m, v, 2.5e-4, (0.9, 0.999), 1e-5, 0.0, mx, 1.0, 3)
        for k in ("params", "exp_avg", "exp_avg_sq"):
            assert torch.equal(torch.isnan(got[k]).cpu(), torch.isnan(ref[k])), (val, mx, k)
            assert R.ratio_to_bar(got[k], ref[k], ref["bar_" + k]) <= 1.0, (val, mx, k)


# ---------------------------------------------------------------------------------------------------------------------
# heads
# ---------------------------------------------------------------------------------------------------------------------
def _heads_case(B, H, A, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, generator=g)
    x[1::5] *= 300.0 / math.sqrt(H)    # |z| ~ 1e2 .. 1e3: probabilities that underflow
    return (x, torch.randn(A, H, generator=g) * (2.0 / math.sqrt(H)), torch.randn(A, generator=g) * 0.3,
            torch.randn(1, H, generator=g) * 0.05, torch.randn(1, generator=g))


HEAD_SHAPES = [(H, A) for H in (32, 100, 512, 1024) for A in (1, 4, 7, 8, 9)]


@pytest.mark.parametrize("H,A", HEAD_SHAPES, ids=[f"H{H}-A{A}" for H, A in HEAD_SHAPES])
def test_heads(hb, H, A):
    """heads_fwd logits / values and heads_act log-probabilities / values within the bar; the mode is the float64
    argmax except within the bar of a tie; the inverse-CDF pick on a dense u grid (0 and 1 - 2^-24 included) never
    takes a zero-probability action and is the float64 pick except within the bar of a CDF boundary"""
    from habitat_lab_b200 import ops

    B = 97
    ops_in = [_gpu(t) for t in _heads_case(B, H, A, seed=H * 10 + A)]
    ref = R.heads(*ops_in)
    logits, values = torch.empty(B, A, device=DEV), torch.empty(B, 1, device=DEV)
    ops.heads_fwd(*ops_in, logits, values)
    torch.cuda.synchronize()
    assert R.ratio_to_bar(logits, ref["logits"], ref["logits_bar"]) <= 1.0
    assert R.ratio_to_bar(values.view(-1), ref["values"], ref["values_bar"]) <= 1.0
    us = [None] + [torch.full((B,), u, device=DEV) for u in (0.0, 1.0 - 2 ** -24)] + \
        [torch.linspace(0, 1 - 2 ** -24, B, device=DEV).roll(k) for k in range(0, 64, 8)]
    cdf = ref["logp"].exp().cumsum(-1)
    cbar = (ref["logp"].exp() * (ref["logp_bar"] + R.K * R.U)).cumsum(-1) + R.K * R.U * A
    for u in us:
        lp, val = torch.empty(B, A, device=DEV), torch.empty(B, 1, device=DEV)
        act, alp = torch.full((B, 1), -1, device=DEV, dtype=torch.int64), torch.empty(B, 1, device=DEV)
        ops.heads_act(*ops_in, u, lp, val, act, alp)
        torch.cuda.synchronize()
        assert R.ratio_to_bar(lp, ref["logp"], ref["logp_bar"]) <= 1.0
        assert R.ratio_to_bar(val.view(-1), ref["values"], ref["values_bar"]) <= 1.0
        assert torch.equal(alp, lp.gather(1, act))
        a = act.view(-1)
        if u is None:
            best = ref["logp"].max(-1, keepdim=True).values
            near = ref["logp"] >= best - 2 * ref["logp_bar"].max(-1, keepdim=True).values
            assert bool(near.gather(1, act).all())
        else:
            assert bool((lp.gather(1, act).exp() > 0).all())     # never a zero-probability action
            ud = u.double().view(-1, 1)
            lo = (cdf < ud - cbar).sum(-1).clamp(max=A - 1)
            hi = (cdf <= ud + cbar).sum(-1).clamp(max=A - 1)
            # u past the kernel's rounded total (only within the bar of cdf[-1]): the last non-zero-probability action
            last_nz = (torch.arange(A, device=DEV) * (lp.exp() > 0)).max(-1).values
            top = torch.where((ud + cbar[:, -1:] >= cdf[:, -1:]).view(-1), torch.maximum(hi, last_nz), hi)
            assert bool(((a >= lo) & (a <= top)).all())


def test_heads_act_mode_ties(hb):
    """bitwise-equal weight rows (and biases) give bitwise-equal logits; the mode takes the first of them"""
    from habitat_lab_b200 import ops

    for A, rows in ((4, (1, 3)), (9, (2, 8)), (8, (0, 7))):
        x, wa, ba, wv, bv = _heads_case(64, 512, A, seed=A)
        x = x.abs()
        wa[rows[0]] = wa[rows[1]] = wa.abs().max() + 0.1
        ba[rows[0]] = ba[rows[1]] = 1.0
        ins = [_gpu(t) for t in (x, wa, ba, wv, bv)]
        lp, val = torch.empty(64, A, device=DEV), torch.empty(64, 1, device=DEV)
        act, alp = torch.empty(64, 1, device=DEV, dtype=torch.int64), torch.empty(64, 1, device=DEV)
        ops.heads_act(*ins, None, lp, val, act, alp)
        torch.cuda.synchronize()
        assert torch.equal(lp[:, rows[0]], lp[:, rows[1]])
        assert bool((act.view(-1) == rows[0]).all())


@pytest.mark.parametrize("H,A", [(512, 4), (32, 8), (128, 1)])
def test_act_log_probs_match_the_loss(hb, H, A):
    """the act-time action_log_probs and the loss kernel's log_probs of the same features agree within the sum of
    their bars: the PPO ratio at epoch 0 is 1 to within the bar"""
    from habitat_lab_b200 import ops

    B = 512
    x, wa, ba, wv, bv = (_gpu(t) for t in _heads_case(B, H, A, seed=H + A))
    lp, val = torch.empty(B, A, device=DEV), torch.empty(B, 1, device=DEV)
    act, alp = torch.empty(B, 1, device=DEV, dtype=torch.int64), torch.empty(B, 1, device=DEV)
    ops.heads_act(x, wa, ba, wv, bv, torch.rand(B, device=DEV), lp, val, act, alp)
    c = dict(feat=x, w_act=wa, b_act=ba, w_val=wv, b_val=bv, actions=act.view(-1), old_lp=alp.view(-1),
             adv=torch.randn(B, device=DEV), old_v=val.view(-1), ret=val.view(-1), is_coeffs=None)
    got = _run_loss(ops, c, True)
    ref = R.heads(x, wa, ba, wv, bv)
    bar = 2 * ref["logp_bar"].gather(1, act).view(-1)
    assert bool(((got["log_probs"] - alp.view(-1)).abs() <= bar).all())
    assert R.ratio_to_bar(got["prob_ratio_max"] - 1, torch.zeros(()), bar.max()) <= 1.0
    assert R.ratio_to_bar(got["prob_ratio_min"] - 1, torch.zeros(()), bar.max()) <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# clip + Adam
# ---------------------------------------------------------------------------------------------------------------------
def _run_adam(ops, p, g, m, v, lr, wd, mx, gs, step, hyper=False):
    n = p.numel()
    n_pad = (n + 3) // 4 * 4
    flat = torch.zeros(4, n_pad, device=DEV)
    for i, t in enumerate((p, g, m, v)):
        flat[i, :n] = t.to(DEV)
    gn = torch.zeros(1, device=DEV)
    hyp = torch.tensor([lr], device=DEV) if hyper else None
    ops.clip_adam(flat[0, :n], flat[1, :n], flat[2, :n], flat[3, :n], 0.0 if hyper else lr, (0.9, 0.999), 1e-5, wd,
                  mx, gs, step, gn, ops.clip_adam_workspace(n, DEV), hyper=hyp)
    torch.cuda.synchronize()
    return dict(params=flat[0, :n], exp_avg=flat[2, :n], exp_avg_sq=flat[3, :n], norm=gn[0])


def _adam_case(n, seed):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=gen) * 1e-3, torch.randn(n, generator=gen) * 0.05,
            torch.randn(n, generator=gen) * 1e-3, torch.rand(n, generator=gen) * 1e-5)


def _check_adam(hb, n, mx, wd, gs, step, hyper):
    from habitat_lab_b200 import ops

    p, g, m, v = _adam_case(n, seed=n + step)
    got = _run_adam(ops, p, g, m, v, 2.5e-4, wd, mx, gs, step, hyper)
    d = [t.to(DEV) for t in (p, g, m, v)]
    ref = R.clip_adam(*d, 2.5e-4, (0.9, 0.999), 1e-5, wd, mx, gs, step)
    ratios = {k: R.ratio_to_bar(got[k], ref[k], ref["bar_" + k]) for k in ("params", "exp_avg", "exp_avg_sq", "norm")}
    guards = {}
    for pt in R.ADAM_PERTURBATIONS:
        pr = R.clip_adam(*d, 2.5e-4, (0.9, 0.999), 1e-5, wd, mx, gs, step, perturb=pt)
        if pr is not None and not torch.equal(pr["params"], ref["params"]):
            guards[pt] = R.ratio_to_bar(pr["params"], ref["params"], ref["bar_params"])
    assert max(ratios.values()) <= 1.0, ratios
    assert guards["eps_in_sqrt"] >= 10.0
    if step <= 10:
        assert guards["bias_step"] >= 10.0
    if "scale_after_norm" in guards:
        assert guards["scale_after_norm"] >= 10.0
    return ratios, guards


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 1_081_343, 1_081_344, 1_081_345, 8_481_125])
def test_clip_adam_sizes(hb, n):
    """tails of 1-3 elements, one grid-stride pass exactly (132 * 8 * 256 * 4 = 1,081,344) and either side of it"""
    ratios, guards = _check_adam(hb, n, 0.2, 0.0, 1.0, 1, False)
    print(f"  adam n{n}: kernel / bar {ratios}; perturbed / bar {guards}")


ADAM_OPTS = [(mx, wd, gs, st) for mx in (0.0, 0.2, 1e9) for wd in (0.0, 0.01) for gs in (1.0, 0.5, 1 / 3)
             for st in (1, 2, 10, 10_000)]


@pytest.mark.parametrize("hyper", [False, True], ids=["lr_arg", "lr_device"])
@pytest.mark.parametrize("mx,wd,gs,step", ADAM_OPTS, ids=[f"mx{a}-wd{b}-gs{c:.3g}-s{d}" for a, b, c, d in ADAM_OPTS])
def test_clip_adam_options(hb, mx, wd, gs, step, hyper):
    _check_adam(hb, 1023, mx, wd, gs, step, hyper)


def test_grad_sqnorm(hb):
    """hb200_grad_sqnorm alone: the fp64 sum of the fp32 scaled squares, within 16 u of it"""
    from habitat_lab_b200 import _lib

    for n in (1, 5, 1_081_345):
        g = torch.randn(n, generator=torch.Generator().manual_seed(n), device="cpu").to(DEV)
        out = torch.zeros(1, device=DEV)
        ws = torch.empty(_lib.load().hb200_clip_adam_workspace_bytes(n), dtype=torch.uint8, device=DEV)
        _lib.call("hb200_grad_sqnorm", _lib.ptr(g), n, 0.5, _lib.ptr(out), _lib.ptr(ws))
        torch.cuda.synchronize()
        ref = ((g * 0.5).double() ** 2).sum().item()
        assert abs(out.item() - ref) <= R.K * R.U * ref


# ---------------------------------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,A", [(512, 0), (512, 9), (96, 4), (1024, 4)])
def test_ppo_loss_refuses_unsupported_shapes(hb, H, A):
    from habitat_lab_b200 import _lib, ops

    B = 16
    f = lambda *sh: torch.randn(*sh, device=DEV)  # noqa: E731
    out = _loss_out(B, H, max(A, 1))
    with pytest.raises(_lib.Hb200Error, match="ppo_loss: (n_actions|hidden)"):
        _lib.call("hb200_ppo_loss", *(_lib.ptr(t) for t in (f(B, H), f(max(A, 1), H), f(max(A, 1)), f(H), f(1),
                                                             torch.zeros(B, dtype=torch.int64, device=DEV), f(B),
                                                             f(B), f(B), f(B))), None, B, H, A, 0.2, 0.5, 0.01, 1, 1,
                  *(_lib.ptr(out[k]) for k in ("values", "log_probs", "entropy") + R.GRADS + ("metrics",)),
                  _lib.ptr(ops.ppo_loss_workspace(B, H, max(A, 1), DEV)))
