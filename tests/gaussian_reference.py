"""Float64 restatement of the Gaussian action head (GaussianNet + CustomNormal, HB/utils/common.py:99-175), of Policy.act's
tail for it (HB/rl/ppo/policy.py:330-342) and of PPO's loss over it (HB/rl/ppo/ppo.py:195-250), with gradients, the
per-element error bars the fp32 kernels (csrc/rl_kernels.cu: gaussian_act / gaussian_ppo_loss) are judged by, and the
perturbed restatements that show the bars are tight.  Shared by tests/test_gpu_gaussian.py and
tests/test_gaussian_reference_cpu.py.  u = 2^-24.

The restatement is the reference's own op sequence evaluated by torch autograd in the dtype asked for (float64 for the
reference, float32 for the CPU check that fp32 stays within the bars), so its gradients follow torch's conventions at
every edge the kernels must match: clamp passes the gradient at its bounds, softplus switches to the identity above 20,
torch.min sends the gradient to both operands when one is NaN.

Bars: first-order propagation of the roundings the kernels make, per frame and action dimension a
-------------------------------------------------------------------------------------------------
Every fp32 operation rounds once (<= u/2; libm / CUDA exp, log, tanh, log1p within 2 ulp).  A length-n dot product or
sum carries K u sqrt(n) (sum of |terms|) -- independent roundings add like a random walk.  K = 16 throughout.
  z   = x . w + b (each mu_maybe_std row, the critic):  bar(z) = K u sqrt(H) (|x| . |w| + |b|)
  mu  = tanh(mu_pre) or mu_pre:                          bar(mu) = T bar(z_mu) + 4 u |mu|,   T = 1 - mu^2 (tanh) or 1
  std = softplus(exp(clamp(s0))) (steps by flag):        bar(std) = |J| bar(z_s) + 8 u std,  J = d std / d s0
        (J = 0 where the clamp is active; s0 is the std parameter itself -- no rounding -- with use_std_param)
  d = x - mu, q = d^2 / std^2:                           bar(d) = bar(mu) + 2 u (|x| + |mu|)
  lp_a = -q/2 - log std - log sqrt(2 pi):                bar(lp_a) = |d| / std^2 bar(d) + (q + 1) / std bar(std)
                                                                     + K u (q / 2 + |log std| + 1)
  lp = sum_a lp_a, H = sum_a (0.5 + log sqrt(2 pi) + log std_a):
        bar(lp) = sum_a bar(lp_a) + K u sum_a |lp_a|,    bar(H) = sum_a bar(std_a) / std_a + K u sum_a |H_a|
  ratio = exp(lp - old_lp):                             bar(ratio) = ratio (bar(lp) + K u (1 + |lp - old_lp|))
Gradients, with c = min(is_coeff, 1), g_lp = -adv ratio c / B (0 on the clipped branch), g_h = -c_e c / B:
  dmu     = g_lp d / std^2            bar = bar(g_lp) |d| / std^2 + |g_lp| (bar(d) / std^2 + 2 |d| / std^3 bar(std))
                                             + K u |dmu|,   bar(g_lp) = |adv| c / B bar(ratio) + K u |g_lp|
  dmu_pre = T dmu                     bar = T bar(dmu) + 2 |mu dmu| bar(mu) [tanh] + 4 u |dmu_pre|
  dstd    = g_lp (q - 1) / std + g_h / std
          bar = bar(g_lp) |q - 1| / std + |g_lp| (2 |d| / std^2 bar(d) + (3 q + 1) / std^2 bar(std)) + |g_h| bar(std) / std^2
                + K u (|g_lp| (q + 1) + |g_h|) / std
  ds0     = J dstd                    bar = |J| bar(dstd) + |J dstd| (K u + (2 + |s2|) bar(z_s))
          (s2 = std before softplus: the log-derivative of J with respect to s0 is at most 2 + |s2| for every flag mix)
  g_v     = c_v c (v_used - ret) / B  bar = c_v c / B (bar(v) + K u (|v| + |old_v| + |ret|)) + K u |g_v|
Contractions over the head rows o (R = L + 1 of them) and over the B frames:
  d_features = sum_o dl_o W_o        bar = sum_o bar(dl_o) |W_o| + K u sqrt(R) sum_o |dl_o| |W_o|
  d_W[o] = sum_b dl_bo x_b           bar = sqrt(sum_b bar(dl_bo)^2 x_b^2) + K u sqrt(B) max(|d_W|, sqrt(sum_b dl_bo^2 x_b^2))
  (biases and d_std: x = 1).  Loss means of per-frame terms t_b: (sum_b bar(t_b) + K u sqrt(B) sum_b |t_b|) / B.
The two branch decisions (ratio against 1 +- clip, |v - old_v| against clip) are kept away from their boundaries by
make_case (old_log_probs / old_values are placed at least 100 bars from them), so both sides take the same branch.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
K = 16.0
LOG_STD, SOFTPLUS, STD_PARAM, CLAMP_STD, TANH = 1, 2, 4, 8, 16
HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)
PERTURBATIONS = ("no_tanh_grad", "clamp_grad_everywhere", "clamp_grad_blocked_at_bounds", "entropy_not_summed",
                 "log_prob_not_summed")


def bounds(cfg):
    """(flags, min, max) GaussianNet derives from an ActionDistributionConfig-like dict (utils/common.py:126-142)"""
    c = dict(use_log_std=True, use_softplus=False, use_std_param=False, clamp_std=True, min_std=1e-6, max_std=1,
             min_log_std=-5, max_log_std=2, action_activation="tanh", log_std_init=0.0)
    c.update(cfg)
    if c["use_log_std"]:
        lo, hi = c["min_log_std"], c["max_log_std"]
    elif c["use_softplus"]:
        inv = lambda x: math.log(math.exp(x) - 1)  # noqa: E731
        lo, hi = inv(c["min_std"]), inv(c["max_std"])
    else:
        lo, hi = c["min_std"], c["max_std"]
    flags = ((LOG_STD if c["use_log_std"] else 0) | (SOFTPLUS if c["use_softplus"] else 0) |
             (STD_PARAM if c["use_std_param"] else 0) | (CLAMP_STD if c["clamp_std"] else 0) |
             (TANH if c["action_activation"] == "tanh" else 0))
    return flags, float(lo), float(hi)


def _f32(v):
    """a hyper-parameter as the fp32 value the C ABI receives"""
    return float(torch.tensor(v, dtype=torch.float32))


def head(x, w_mu, b_mu, std_p, w_val, b_val, flags, lo, hi, perturb=None):
    """GaussianNet.forward + CriticHead in the tensors' dtype, differentiable: (mu, std, value, pieces)"""
    A = w_mu.shape[0] if flags & STD_PARAM else w_mu.shape[0] // 2
    z = x @ w_mu.T + b_mu
    if flags & STD_PARAM:
        mu_pre, s0 = z, std_p.expand(x.shape[0], A)
    else:
        mu_pre, s0 = z[:, :A], z[:, A:]
    mu = mu_pre
    if flags & TANH:
        mu = torch.tanh(mu_pre)
        if perturb == "no_tanh_grad":
            mu = mu_pre + (mu - mu_pre).detach()
    s = s0
    if flags & CLAMP_STD:
        s = torch.clamp(s0, _f32(lo), _f32(hi))
        if perturb == "clamp_grad_everywhere":
            s = s0 + (s - s0).detach()
        elif perturb == "clamp_grad_blocked_at_bounds":
            inside = (s0 > _f32(lo)) & (s0 < _f32(hi))
            s = torch.where(inside, s0, s.detach())
    if flags & LOG_STD:
        s = torch.exp(s)
    s2 = s
    if flags & SOFTPLUS:
        s = torch.nn.functional.softplus(s)
    v = (x @ w_val.T + b_val).squeeze(-1)
    return mu, s, v, dict(mu_pre=mu_pre, s0=s0, s2=s2)


def log_prob_entropy(mu, std, actions, perturb=None):
    """CustomNormal.log_probs / entropy: Normal's, summed over the action dimension"""
    d = torch.distributions.Normal(mu, std, validate_args=False)
    lp_a, ent_a = d.log_prob(actions), d.entropy()
    lp = lp_a.mean(-1) if perturb == "log_prob_not_summed" else lp_a.sum(-1)
    ent = ent_a.mean(-1) if perturb == "entropy_not_summed" else ent_a.sum(-1)
    return lp, ent


def loss(params, x, case, flags, lo, hi, perturb=None, dtype=torch.float64):
    """PPO._update_from_batch's loss over the Gaussian head (ppo.py:195-250) by autograd in `dtype`: every output the
    kernel writes, gradients included."""
    P = {k: (None if v is None else v.detach().to(dtype).requires_grad_(True)) for k, v in params.items()}
    xf = x.detach().to(dtype).requires_grad_(True)
    t = {k: (None if v is None else v.to(dtype)) for k, v in case.items() if isinstance(v, torch.Tensor)}
    clip, c_v, c_e = (torch.tensor(_f32(case[k]), dtype=dtype) for k in ("clip", "c_v", "c_e"))
    mu, std, v, _ = head(xf, P["w_mu"], P["b_mu"], P["std"], P["w_val"], P["b_val"], flags, lo, hi, perturb)
    lp, ent = log_prob_entropy(mu, std, t["actions"], perturb)
    ratio = torch.exp(lp - t["old_lp"])
    s1 = ratio * t["adv"]
    s2 = torch.clamp(ratio, 1.0 - clip, 1.0 + clip) * t["adv"]
    a_loss = -torch.min(s1, s2)
    if case["use_clipped_value_loss"]:
        delta = (v - t["old_v"]).detach()
        v_used = torch.where(delta.abs() < clip, v, t["old_v"] + torch.clamp(delta, -clip, clip))
    else:
        v_used = v
    v_loss = 0.5 * (v_used - t["ret"]) ** 2
    w = torch.ones_like(v) if t.get("is_coeffs") is None else torch.clamp(t["is_coeffs"], max=1.0)
    B = x.shape[0]
    vl, al, el = (w * v_loss).mean(), (w * a_loss).mean(), (w * ent).mean()
    total = c_v * vl + al - c_e * el
    total.backward()
    metrics = torch.stack([vl, al, el, v.min(), v.mean(), v.max(), ratio.min(), ratio.mean(), ratio.max(),
                           ((ratio > 1.0 + clip).float().sum() + (ratio < 1.0 - clip).float().sum()) / B, total])
    out = dict(values=v.detach(), log_probs=lp.detach(), entropy=ent.detach(), metrics=metrics.detach(),
               d_features=xf.grad, d_w_mu=P["w_mu"].grad, d_b_mu=P["b_mu"].grad, d_w_val=P["w_val"].grad,
               d_b_val=P["b_val"].grad, ratio=ratio.detach(), v_loss=v_loss.detach(), a_loss=a_loss.detach(),
               mu=mu.detach(), std=std.detach())
    if P["std"] is not None:
        out["d_std"] = P["std"].grad
    return out


def _chain(s0, flags, lo, hi):
    """std and J = d std / d s0 in float64, closed form (the autograd conventions of head())"""
    s = s0.clamp(lo, hi) if flags & CLAMP_STD else s0
    J = ((s0 >= lo) & (s0 <= hi)).double() if flags & CLAMP_STD else torch.ones_like(s0)
    if flags & LOG_STD:
        s = torch.exp(s)
        J = J * s
    s2 = s
    if flags & SOFTPLUS:
        J = torch.where(s2 > 20, J, J * torch.sigmoid(s2))
        s = torch.nn.functional.softplus(s2)
    return s, J, s2


def bars(params, x, case, flags, lo, hi, ref):
    """per-element bars of every kernel output (see the module docstring)"""
    d64 = lambda t: None if t is None else t.detach().double()  # noqa: E731
    P = {k: d64(v) for k, v in params.items()}
    x = d64(x)
    B, H = x.shape
    A = P["w_mu"].shape[0] if flags & STD_PARAM else P["w_mu"].shape[0] // 2
    u = U
    ax = x.abs()
    bz = K * u * math.sqrt(H) * (ax @ P["w_mu"].abs().T + P["b_mu"].abs())
    bz_mu = bz[:, :A]
    bz_s = torch.zeros(B, A, dtype=torch.float64) if flags & STD_PARAM else bz[:, A:]
    z = x @ P["w_mu"].T + P["b_mu"]
    s0 = P["std"].expand(B, A) if flags & STD_PARAM else z[:, A:]
    mu = torch.tanh(z[:, :A]) if flags & TANH else z[:, :A]
    T = (1 - mu * mu) if flags & TANH else torch.ones_like(mu)
    std, J, s2 = _chain(s0, flags, lo, hi)
    bmu = T * bz_mu + 4 * u * mu.abs()
    bstd = J.abs() * bz_s + 8 * u * std
    xa = case["actions"].double()
    d = xa - mu
    var = std * std
    q = d * d / var
    bd = bmu + 2 * u * (xa.abs() + mu.abs())
    lp_a = -q / 2 - torch.log(std) - HALF_LOG_2PI
    blp_a = d.abs() / var * bd + (q + 1) / std * bstd + K * u * (q / 2 + torch.log(std).abs() + 1)
    blp = blp_a.sum(-1) + K * u * lp_a.abs().sum(-1)
    ent_a = 0.5 + HALF_LOG_2PI + torch.log(std)
    bent = (bstd / std).sum(-1) + K * u * ent_a.abs().sum(-1)
    bv = K * u * math.sqrt(H) * (ax @ P["w_val"].abs().T + P["b_val"].abs()).squeeze(-1)
    old_lp = case["old_lp"].double()
    ratio = ref["ratio"]
    lp = ref["log_probs"]
    br = ratio * (blp + K * u * (1 + (lp - old_lp).abs()))
    clip, c_v, c_e = (_f32(case[k]) for k in ("clip", "c_v", "c_e"))
    adv = case["adv"].double()
    c = torch.ones(B, dtype=torch.float64) if case.get("is_coeffs") is None else case["is_coeffs"].double().clamp(max=1)
    s1, s2r = adv * ratio, adv * ratio.clamp(1 - clip, 1 + clip)
    live = ~(s1 > s2r)
    g_lp = torch.where(live, -adv * ratio * c / B, torch.zeros_like(adv))
    bg_lp = torch.where(live, adv.abs() * c / B * br + K * u * g_lp.abs(), torch.zeros_like(adv))
    g_h = -c_e * c / B
    v = ref["values"]
    ov, ret = case["old_v"].double(), case["ret"].double()
    if case["use_clipped_value_loss"]:
        v_live = (v - ov).abs() < clip
        v_used = torch.where(v_live, v, ov + (v - ov).clamp(-clip, clip))
    else:
        v_live, v_used = torch.ones_like(v, dtype=torch.bool), v
    g_v = torch.where(v_live, c_v * c * (v_used - ret) / B, torch.zeros_like(v))
    bg_v = torch.where(v_live, c_v * c / B * (bv + K * u * (v.abs() + ov.abs() + ret.abs())) + K * u * g_v.abs(),
                       torch.zeros_like(v))
    gl, bgl, gh = g_lp[:, None], bg_lp[:, None], g_h[:, None] if torch.is_tensor(g_h) else g_h
    dmu = gl * d / var
    bdmu = bgl * d.abs() / var + gl.abs() * (bd / var + 2 * d.abs() / (var * std) * bstd) + K * u * dmu.abs()
    dmu_pre = T * dmu
    bdmu_pre = T * bdmu + (2 * (mu * dmu).abs() * bmu if flags & TANH else 0) + 4 * u * dmu_pre.abs()
    dstd = gl * (q - 1) / std + gh / std
    bdstd = (bgl * (q - 1).abs() / std + gl.abs() * (2 * d.abs() / var * bd + (3 * q + 1) / var * bstd)
             + abs(gh) * bstd / var + K * u * (gl.abs() * (q + 1) + abs(gh)) / std)
    ds0 = J * dstd
    bds0 = J.abs() * bdstd + (J * dstd).abs() * (K * u + (2 + s2.abs()) * bz_s)
    # dl columns as the kernel lays them out: mu_maybe_std rows, then the critic
    if flags & STD_PARAM:
        dl, bdl, W = torch.cat([dmu_pre, g_v[:, None]], 1), torch.cat([bdmu_pre, bg_v[:, None]], 1), \
            torch.cat([P["w_mu"], P["w_val"]], 0)
    else:
        dl = torch.cat([dmu_pre, ds0, g_v[:, None]], 1)
        bdl = torch.cat([bdmu_pre, bds0, bg_v[:, None]], 1)
        W = torch.cat([P["w_mu"], P["w_val"]], 0)
    R = W.shape[0]
    out = {}
    out["d_features"] = bdl @ W.abs() + K * u * math.sqrt(R) * (dl.abs() @ W.abs())

    def wsum(g, bg, xx):   # [B, n] x [B, m] -> bar of g^T xx
        tot = g.T @ xx
        rss = torch.sqrt((g * g).T @ (xx * xx))
        return torch.sqrt((bg * bg).T @ (xx * xx)) + K * u * math.sqrt(B) * torch.maximum(tot.abs(), rss)

    one = torch.ones(B, 1, dtype=torch.float64)
    L = R - 1
    out["d_w_mu"] = wsum(dl[:, :L], bdl[:, :L], x)
    out["d_w_val"] = wsum(dl[:, L:], bdl[:, L:], x)
    out["d_b_mu"] = wsum(dl[:, :L], bdl[:, :L], one).squeeze(-1)
    out["d_b_val"] = wsum(dl[:, L:], bdl[:, L:], one).squeeze(-1)
    if flags & STD_PARAM:
        out["d_std"] = wsum(ds0, bds0, one).squeeze(-1)
    out["values"], out["log_probs"], out["entropy"] = bv, blp, bent
    mean_bar = lambda tb, tv: (tb.sum() + K * u * math.sqrt(B) * tv.abs().sum()) / B  # noqa: E731
    dv = (v_used - ret).abs()
    b_vl = c * dv * (torch.where(v_live, bv, torch.zeros_like(bv)) + K * u * (v.abs() + ov.abs() + ret.abs()))
    b_al = c * adv.abs() * br
    b_en = c * bent
    vl, al, el = mean_bar(b_vl, c * ref["v_loss"]), mean_bar(b_al, c * ref["a_loss"]), mean_bar(b_en, c * ref["entropy"])
    m = torch.zeros(11, dtype=torch.float64)
    m[0], m[1], m[2] = vl, al, el
    m[3], m[5] = bv.max(), bv.max()
    m[4] = mean_bar(bv, v)
    m[6], m[8] = br.max(), br.max()
    m[7] = mean_bar(br, ratio)
    m[9] = 0.0
    m[10] = c_v * vl + al + c_e * el + K * u * (c_v * ref["metrics"][0].abs() + ref["metrics"][1].abs()
                                                  + c_e * ref["metrics"][2].abs())
    out["metrics"] = m
    # the act tail: mean, sample mu + eps std, its log-probability
    out["mu"], out["std"], out["bz_s"], out["J"] = bmu, bstd, bz_s, J
    return out


def act_bars(params, x, flags, lo, hi, eps):
    """bars of gaussian_act's actions and log-probabilities (eps None: the mean), and the float64 values"""
    P = {k: None if v is None else v.detach().double() for k, v in params.items()}
    x64 = x.detach().double()
    with torch.no_grad():
        mu, std, v, _ = head(x64, P["w_mu"], P["b_mu"], P["std"], P["w_val"], P["b_val"], flags, lo, hi)
    a = mu if eps is None else mu + eps.double() * std
    lp, _ = log_prob_entropy(mu, std, a)
    case = dict(actions=a, old_lp=lp, adv=torch.zeros_like(v), old_v=v, ret=v, clip=0.2, c_v=0.5, c_e=0.0,
                use_clipped_value_loss=False)
    ref = dict(ratio=torch.ones_like(v), log_probs=lp, values=v, v_loss=torch.zeros_like(v),
               a_loss=torch.zeros_like(v), entropy=torch.zeros_like(v), metrics=torch.zeros(11, dtype=torch.float64))
    b = bars(params, x, case, flags, lo, hi, ref)
    ba = b["mu"] if eps is None else b["mu"] + eps.double().abs() * b["std"] + 4 * U * a.abs()
    # lp is computed from the kernel's own mu: d = a - mu = eps std up to the rounding of a, so mu's error cancels
    d = a - mu
    q = d * d / (std * std)
    e = torch.zeros_like(a) if eps is None else eps.double().abs()
    bd = e * b["std"] + 2 * U * (a.abs() + mu.abs())
    blp = d.abs() / (std * std) * bd + (q + 1) / std * b["std"] + K * U * (q / 2 + torch.log(std).abs() + 1)
    blp = blp.sum(-1) + K * U * lp.abs().sum(-1)
    return dict(actions=a, log_probs=lp, values=v), dict(actions=ba, log_probs=blp, values=b["values"])


def make_case(B, H, A, cfg, seed, std_at_bounds=False, dtype=torch.float32):
    """fp32 parameters, features and a minibatch for one flag mix; old_log_probs / old_values are placed away from the
    clip boundaries (see the module docstring).  std_at_bounds: some raw std values sit exactly on the clamp bounds."""
    flags, lo, hi = bounds(cfg)
    g = torch.Generator().manual_seed(seed)
    L = A if flags & STD_PARAM else 2 * A
    x = torch.randn(B, H, generator=g) * 0.5
    w_mu = torch.randn(L, H, generator=g) / math.sqrt(H)
    b_mu = torch.randn(L, generator=g) * 0.1
    std = None
    if flags & STD_PARAM:
        # centred one below the upper bound: a std of order 1 (the midpoint is a std of 1e-3 for the softplus bounds)
        std = torch.randn(A, generator=g) * 0.5 + ((hi - 1.0) if flags & CLAMP_STD else 0.0)
        if not flags & (LOG_STD | SOFTPLUS):
            std = std.abs() + 0.2
        if std_at_bounds and flags & CLAMP_STD:
            std[0] = _f32(hi)
            if A >= 2 and flags & LOG_STD:   # the other lower bounds are a std of 1e-6: below fp32's resolution of mu
                std[1] = _f32(lo)
    else:
        if not flags & (LOG_STD | SOFTPLUS):   # raw std must stay positive without a transform
            b_mu[A:] = 1.0
            w_mu[A:] *= 0.1
        if std_at_bounds and flags & CLAMP_STD:
            w_mu[A:, :] = 0.0   # the raw std is exactly the bias: the upper bound for dimension 0, the lower for 1
            b_mu[A] = _f32(hi)
            if A >= 2 and flags & LOG_STD:
                b_mu[A + 1] = _f32(lo)
    w_val = torch.randn(1, H, generator=g) / math.sqrt(H)
    b_val = torch.randn(1, generator=g) * 0.1
    params = dict(w_mu=w_mu, b_mu=b_mu, std=std, w_val=w_val, b_val=b_val)
    with torch.no_grad():
        mu, sd, v, _ = head(x.double(), w_mu.double(), b_mu.double(), None if std is None else std.double(),
                            w_val.double(), b_val.double(), flags, lo, hi)
    actions = (mu + sd * torch.randn(B, A, generator=g, dtype=torch.float64)).float()
    lp, _ = log_prob_entropy(mu, sd, actions.double())
    clip = 0.2
    # target ratios uniform in [0.6, 1.4] away from 1 +- clip; old values away from v +- clip
    r = 0.6 + 0.8 * torch.rand(B, generator=g, dtype=torch.float64)
    r = torch.where((r - 0.8).abs() < 0.02, r + 0.05, r)
    r = torch.where((r - 1.2).abs() < 0.02, r + 0.05, r)
    old_lp = (lp - torch.log(r)).float()
    dv = 0.4 * torch.rand(B, generator=g, dtype=torch.float64) - 0.2
    dv = torch.where((dv.abs() - clip).abs() < 0.02, dv * 0.5, dv)
    dv = torch.where(torch.rand(B, generator=g) < 0.3, dv * 3.0, dv)
    dv = torch.where((dv.abs() - clip).abs() < 0.02, dv * 0.5, dv)
    old_v = (v - dv).float()
    case = dict(actions=actions, old_lp=old_lp, adv=torch.randn(B, generator=g), old_v=old_v,
                ret=torch.randn(B, generator=g), is_coeffs=None, clip=clip, c_v=0.5, c_e=0.01,
                use_clipped_value_loss=True)
    return params, x, case, (flags, lo, hi)


def ratio_to_bar(got, ref, bar):
    """max |got - ref| / bar over elements (NaN positions must agree; they are excluded)"""
    got, ref, bar = got.double(), ref.double(), bar.double()
    nan = torch.isnan(ref)
    if not torch.equal(nan, torch.isnan(got)):
        return math.inf
    keep = ~nan
    if not keep.any():
        return 0.0
    return float(((got - ref).abs()[keep] / bar[keep].clamp(min=1e-300)).max())


COMPARED = ("values", "log_probs", "entropy", "d_features", "d_w_mu", "d_b_mu", "d_w_val", "d_b_val", "d_std")
