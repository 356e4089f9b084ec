"""Plain float64 references of the PPO tail kernels (csrc/rl_kernels.cu: GAE, advantage normalisation, PPO loss,
clip + Adam; csrc/elementwise.cu: heads_fwd / heads_act), their error bars, and the perturbed references that show
each bar is tight.  Shared by tests/test_gpu_ppo_tail.py and tests/test_ppo_reference_cpu.py.

Every reference starts from the kernels' own fp32 operands, hyper-parameters included (gamma, gamma * tau, clip, lr,
betas, eps, ... are the fp32 values the C ABI receives), and runs in float64 (or, for the CPU restatement, in the dtype
asked for).  u = 2^-24.

Bars: running error bounds
--------------------------
A bar is per element.  It evaluates the same contraction or recurrence on absolute values in float64 and takes
K * u * (that) * sqrt(length): independent roundings add like a random walk, so the sqrt(length) growth is what a sum
of `length` rounded terms shows, and stating the bar on absolute values keeps it tight under cancellation and large |z|.

GAE (use_gae).  delta_t = r_t + gamma V_{t+1} m_{t+1} - V_t, gae_t = delta_t + gt m_{t+1} gae_{t+1}, R_t = gae_t + V_t.
  Every step rounds each of its four operations once, and an error made at step s reaches step t scaled by the
  product of the gt m factors in between (<= 1).  The warp kernel folds each lane's chunk into an affine map
  g -> A + B g, composes the maps across lanes in a 5-level shuffle scan, and replays its chunk from the composed
  incoming value; composing affine maps of absolute values gives back the same recurrence, so one bound covers both
  variants:  G_t = |r_t| + |gamma V_{t+1}| m_{t+1} + |V_t| + gt m_{t+1} G_{t+1}, and
      bar(R_t) = bar(adv_t) = K u sqrt(T) (G_t + |V_t|),   K = 16.
  With gamma = tau = 1 nothing damps: G_t then sums every later term, which is exactly the size the accumulated
  rounding errors scale with, so the bar holds without damping.  Rows t >= T (bootstrap and stale rows) are one fp32
  subtraction of the buffers and are compared bit for bit.  Without GAE the return scan is R_t = r_t + gamma m R_{t+1}
  with the same bound on G_t = |r_t| + gamma m G_{t+1}.
Advantage statistics.  Each finite fp32 advantage is exact in float64, so the kernel's float64 sums differ from any
  other order by at most n 2^-53 sum|a| (and n 2^-53 sum a^2); the count is exact.
adv_normalize.  mean and var are rounded to fp32 (u/2 each), var + eps, sqrtf and 1 / x are IEEE round-to-nearest
  (u/2 each), then a - mean and the product (u/2 each): |err| <= 3 u (|a| + |mean|) / sqrt(var + eps).
      bar = K u (|a| + |mean|) / sqrt(var + eps),   K = 4.
Heads.  z = x . w + b is a length-H fp32 dot product: bar(z) = 16 u sqrt(H) (|x| . |w| + |b|), the same for v.  With
  lse = max + log(sum exp(z - max)), each log-probability carries its own z error, the largest z error through lse,
  and the rounding of the subtractions, exp and log (heads_act uses __expf / __logf: a few u of |z| and of log A):
      bar(logp_a) = bar(z_a) + max_a bar(z_a) + 16 u (|z_a| + |lse| + A)
      bar(H)      = sum_a p_a (1 + |logp_a|) bar(logp_a) + 16 u A sum_a p_a |logp_a|.
PPO loss.  The ratio carries the log-probability error and the rounding of lp - old_lp and expf:
  bar(ratio) = ratio (bar(lp) + 16 u (1 + |lp - old_lp|)).  Per frame, with the branch the reference takes,
  g_lp = d total / d lp = -adv ratio c / B (or 0 when clipped), g_h = -c_e c / B, c = min(is_coeffs, 1), and
      dz_a = g_lp (1[a = act] - p_a) - g_h p_a (logp_a + H)         (d total / d logit a)
      bar(dz_a) = bar(g_lp) |1[a = act] - p_a| + |g_lp| bar(p_a) + |g_h| (bar(p_a) |logp_a + H| + p_a (bar(logp_a) +
                  bar(H))) + 16 u (|g_lp| (1 + p_a) + |g_h| p_a (|logp_a| + H)),   bar(p_a) = p_a (bar(logp_a) + 16 u)
  and for the value, dv = v_used - ret: bar(g_v) = c_v c / B (bar(v) + 16 u (|v| + |old_v| + |ret|)) + 16 u |g_v|.
  d_features = dz W (+ g_v w_val), length A + 1; d_w / d_b are sums over the B frames:
      bar(d_features) = bar(dz) |W| + 16 u sqrt(A + 1) |dz| |W|
      bar(d_w_act)    = sqrt(sum_b bar(dz_b)^2 x_b^2) + 16 u sqrt(B) max(|sum_b dz_b x_b|, sqrt(sum_b dz_b^2 x_b^2))
  (d_b: x = 1; the value head alike).  Each frame's error comes from that frame's own roundings, so across the B
  frames they add like a random walk: the root of the sum of squares, not the sum.  Likewise the partial sums the
  kernel rounds (fma chains per frame slice, 8 slices, up to 32 slabs) are about max(|total|, root of the sum of
  squared terms) in size, not sum |terms|, which is what lets a sum missing one frame slab show.
  The losses are means of per-frame terms t_b, each with its own bar from the above:
      bar(mean t) = (sum_b bar(t_b) + 16 u sqrt(B) sum_b |t_b|) / B.
  The two branch decisions (ratio against 1 +- clip, where it changes min(s1, s2); |v - old_v| against clip) can go
  either way in fp32 for a frame within the bar of the boundary.  For such a frame the d_features row may match any
  combination of the two branches' float64 gradients.  The weight gradients are compared with the reference built
  from the branch each row shows (branch_choice), so their bars do not grow with the number of such frames; only a
  frame whose row fits two choices within the bar adds its |difference| (times |x|).  fraction_clipped may differ by
  one frame per ambiguous frame.  Every loss case without |z| ~ 1e3 frames (see make_loss_case) also requires zeroed
  weight gradients, and sums missing the last frame slab of ppo_heads_wgrad_kernel, to miss the weight-gradient bars
  by at least 10x (weight_grad_guards).
clip + Adam.  The gradient norm is an fp64 sum of fp32-rounded g * grad_scale, rounded to fp32 and square-rooted:
  bar(norm) = 16 u norm.  The update is a fixed chain of about 12 roundings per element; with the absolute values
  M = |m| + (1 - b1) (|g'| + |m|), g' = g grad_scale coef + wd p, the bars are
      bar(m') = 16 u M,  bar(v') = 16 u v',  bar(p') = 16 u (|p| + 3 lr / bc1 M / denom).

Margins.  On the CPU, fp32 restatements of every reference (another evaluation order, other exp / log) stay inside
every bar (tests/test_ppo_reference_cpu.py prints the ratios): at most 0.07 of the bar for GAE, 0.42 for
adv_normalize, 0.27 for the loss outputs (frames within 1e-5 of a clip boundary left out: torch's autograd splits the
gradient between tied surrogates there) and 0.22 for Adam.

Values.  oracle.torch_oracle.ppo_loss casts the values to fp32 (the reference's values.float()), so the float64
reference runs its value path on fp32-rounded values; the value bars' 16 u |v| term covers that rounding.

Perturbed references.  Each must miss its bar by at least 10x wherever it changes the exact result:
  GAE        zero_chunk_in (the incoming value at the first warp-chunk boundary zeroed), mask_at_t (m_t read instead
             of m_{t+1}), gamma_for_gt (gamma in place of gamma * tau)
  normalize  biased_var (divides by n; changes the result by 1 / (2 n) relative, so it is asserted where n <= 2^14),
             eps_outside (1 / (sqrt(var) + eps))
  loss       straight_through_v (the value gradient flows while clipped), grad_through_clip (the surrogate's gradient
             flows through the clamp), entropy_no_h (d H / d z without the + H term), is_unclamped (is_coeffs not
             clamped at 1)
  Adam       eps_in_sqrt (sqrt(v / bc2 + eps)), bias_step (bias corrections of step + 1; at step 10^4 both are 1 to
             within 5e-5 and the change is below the bar, so it is asserted for step <= 10), scale_after_norm
             (norm of the unscaled gradient; changes the result only while clipping is active and grad_scale != 1)
"""
import math

import torch
import torch.nn.functional as F

from oracle import torch_oracle as O

U = 2.0 ** -24
K = 16.0
K_NORM = 4.0
EPS_PPO = 1e-5
f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))  # noqa: E731  (a hyper-parameter as the C ABI sees it)

GAE_PERTURBATIONS = ("zero_chunk_in", "mask_at_t", "gamma_for_gt")
NORM_PERTURBATIONS = ("biased_var", "eps_outside")
LOSS_PERTURBATIONS = ("straight_through_v", "grad_through_clip", "entropy_no_h", "is_unclamped")
ADAM_PERTURBATIONS = ("eps_in_sqrt", "bias_step", "scale_after_norm")


def ratio_to_bar(got, ref, bar):
    """max |got - ref| / bar over the elements; non-finite elements must agree exactly (same inf, NaN with NaN)"""
    got, ref, bar = got.double(), ref.double().to(got.device), bar.double().to(got.device)
    fin = torch.isfinite(ref)
    bad = ~fin & ~((got == ref) | (torch.isnan(got) & torch.isnan(ref)))
    if bool(bad.any()):
        return math.inf
    if not bool(fin.any()):
        return 0.0
    return ((got - ref).abs()[fin] / bar[fin].clamp_min(1e-300)).max().item()


# ---------------------------------------------------------------------------------------------------------------------
# GAE
# ---------------------------------------------------------------------------------------------------------------------
def gae_discounts(gamma, tau):
    """the fp32 gamma and gamma * tau the kernel runs with"""
    g = f32(gamma)
    return g, f32(g * f32(tau))


def gae(rewards, values, masks, next_value, returns_buf, t_cur, gamma, tau, use_gae=True, perturb=None,
        dtype=torch.float64):
    """rewards / values / returns_buf fp32 [Ta, N] (values before the bootstrap write, returns_buf what the returns
    buffer holds), masks bool [Ta, N], next_value [N].  Returns dict(returns, adv, values [Ta, N] as the kernel leaves
    them, bar [Ta, N]; rows >= t_cur of returns / adv are fp32 and exact), or None when the perturbation cannot change
    this case (no warp-chunk boundary)."""
    Ta, N = rewards.shape
    T = t_cur
    g32, gt32 = gae_discounts(gamma, tau)
    dev = rewards.device
    m = masks.to(dtype=dtype)
    r, V = rewards.to(dtype), values.to(dtype).clone()
    values_out = values.clone()
    ret = returns_buf.clone().to(dtype)
    bar = torch.zeros(Ta, N, dtype=torch.float64, device=dev)
    L = (T + 31) // 32
    tb = L - 1 if T > L else None    # lane 0's last step receives the first chunk boundary's incoming value
    if perturb == "zero_chunk_in" and tb is None:
        return None
    c_gt = g32 if perturb == "gamma_for_gt" else gt32
    sq = math.sqrt(max(T, 1))
    if use_gae:
        values_out[T] = next_value
        V[T] = next_value.to(dtype)
        g = torch.zeros(N, dtype=dtype, device=dev)
        G = torch.zeros(N, dtype=torch.float64, device=dev)
        for t in reversed(range(T)):
            mt = m[t] if perturb == "mask_at_t" else m[t + 1]
            delta = r[t] + g32 * V[t + 1] * mt - V[t]
            g_in = torch.zeros_like(g) if (perturb == "zero_chunk_in" and t == tb) else g
            g = delta + c_gt * mt * g_in
            ret[t] = g + V[t]
            G = (r[t].abs() + abs(g32) * V[t + 1].abs() * mt + V[t].abs()).double() + gt32 * mt.double() * G
            bar[t] = K * U * sq * (G + V[t].abs().double())
        adv = ret - V
        rows = slice(T, Ta)
        adv[rows] = (returns_buf[rows] - values_out[rows]).to(dtype)   # one fp32 subtraction: exact rows
    else:
        ret[T] = next_value.to(dtype)
        G = next_value.abs().double()
        for t in reversed(range(T)):
            mt = m[t] if perturb == "mask_at_t" else m[t + 1]
            ret[t] = g32 * ret[t + 1] * mt + r[t]
            G = r[t].abs().double() + abs(g32) * mt.double() * G
            bar[t] = K * U * sq * (G + V[t].abs().double())
        ret32 = ret.float()
        ret32[T + 1:] = returns_buf[T + 1:]
        ret[T + 1:] = returns_buf[T + 1:].to(dtype)
        adv = (ret - V)
        adv[T:] = (ret32[T:] - values_out[T:]).to(dtype)
    return dict(returns=ret, adv=adv, values=values_out, bar=bar)


def adv_stats(adv):
    """(sum, sum of squares, count) of the finite entries in float64, and the bars of the two sums"""
    a = adv.double()
    a = a[torch.isfinite(a)]
    n = a.numel()
    s, ss = a.sum().item(), (a * a).sum().item()
    e = n * 2.0 ** -53
    return dict(sum=s, sumsq=ss, count=n, bar_sum=e * a.abs().sum().item(), bar_sumsq=e * ss)


def adv_normalize(adv, mean_var=None, perturb=None, dtype=torch.float64):
    """mode 0 (mean_var None): unbiased var_mean over the finite entries of the fp32 advantages; mode 1: the fp32
    (mean, var) given.  Returns (normalised advantages, bar)."""
    a = adv.to(dtype)
    if mean_var is None:
        fin = a[torch.isfinite(a)]
        var, mean = torch.var_mean(fin, correction=0 if perturb == "biased_var" else 1)
        var, mean = var.item(), mean.item()
    else:
        mean, var = float(mean_var[0]), float(mean_var[1])
    if perturb == "eps_outside":
        inv = 1.0 / (math.sqrt(var) + EPS_PPO)
    else:
        inv = 1.0 / math.sqrt(var + f32(EPS_PPO))
    out = (a - mean) * inv
    bar = K_NORM * U * (a.double().abs() + abs(mean)) / math.sqrt(var + EPS_PPO)
    return out, bar


# ---------------------------------------------------------------------------------------------------------------------
# heads
# ---------------------------------------------------------------------------------------------------------------------
def heads(feat, w_act, b_act, w_val, b_val, dtype=torch.float64):
    """logits, values, log-softmax, entropy of fp32 operands, and their bars"""
    x, Wa, ba, Wv, bv = (t.to(dtype) for t in (feat, w_act, b_act, w_val.reshape(1, -1), b_val.reshape(1)))
    H, A = x.shape[1], Wa.shape[0]
    z = F.linear(x, Wa, ba)
    v = F.linear(x, Wv, bv).view(-1)
    logp = torch.log_softmax(z, -1)
    p = logp.exp()
    ent = -(p * logp).sum(-1)
    xa = x.double().abs()
    sq = K * U * math.sqrt(H)
    zbar = sq * (xa @ Wa.double().abs().t() + ba.double().abs())
    vbar = sq * (xa @ Wv.double().abs().t() + bv.double().abs()).view(-1)
    lse = torch.logsumexp(z.double(), -1, keepdim=True)
    lpbar = zbar + zbar.max(-1, keepdim=True).values + K * U * (z.double().abs() + lse.abs() + A)
    pd, lpd = p.double(), logp.double()
    entbar = (pd * (1 + lpd.abs()) * lpbar).sum(-1) + K * U * A * (pd * lpd.abs()).sum(-1)
    return dict(logits=z, values=v, logp=logp, entropy=ent, logits_bar=zbar, values_bar=vbar, logp_bar=lpbar,
                entropy_bar=entbar)


# ---------------------------------------------------------------------------------------------------------------------
# PPO loss
# ---------------------------------------------------------------------------------------------------------------------
METRICS = ("value_loss", "action_loss", "dist_entropy", "value_pred_min", "value_pred_mean", "value_pred_max",
           "prob_ratio_min", "prob_ratio_mean", "prob_ratio_max", "ppo_fraction_clipped", "total_loss")
GRADS = ("d_features", "d_w_act", "d_b_act", "d_w_val", "d_b_val")


def ppo_loss(feat, w_act, b_act, w_val, b_val, actions, old_lp, adv, old_v, ret, is_coeffs, clip, c_v, c_e, use_clip_v,
             dtype=torch.float64):
    """Forward and backward of heads + oracle.torch_oracle.ppo_loss by autograd in `dtype` on fp32 operands (clip,
    c_v, c_e as the fp32 values the kernel gets).  An action outside [0, A) has log-probability NaN.  Returns the
    per-frame outputs (values, log_probs, entropy), the 11 metrics, the gradients, every bar, the branch-ambiguous
    frames and what perturb_grads() needs."""
    clip, c_v, c_e = f32(clip), f32(c_v), f32(c_e)
    B, H = feat.shape
    A = w_act.shape[0]
    hd = heads(feat, w_act, b_act, w_val, b_val)   # bars (float64)
    leaves = [t.to(dtype).detach().requires_grad_(True) for t in (feat, w_act, b_act, w_val.reshape(1, -1),
                                                                   b_val.reshape(1))]
    x, Wa, ba, Wv, bv = leaves
    z = F.linear(x, Wa, ba)
    z.retain_grad()
    v = F.linear(x, Wv, bv)
    v.retain_grad()
    logp = torch.log_softmax(z, -1)
    act = actions.view(-1).long()
    valid = (act >= 0) & (act < A)
    nan = torch.tensor(float("nan"), dtype=dtype, device=x.device)
    lp = logp.gather(1, act.clamp(0, A - 1).view(-1, 1)) + torch.where(valid, 0.0, nan).view(-1, 1)
    lp.retain_grad()
    ent = -(logp.exp() * logp).sum(-1, keepdim=True)
    ent.retain_grad()
    col = lambda t: t.to(dtype).view(-1, 1)  # noqa: E731
    # O.ppo_loss casts the values to fp32 (the reference's values.float()); without value clipping nothing promotes
    # them back, and the returns must then be fp32 as well (they are fp32 operands: no rounding)
    batch = dict(action_log_probs=col(old_lp), advantages=col(adv), value_preds=col(old_v),
                 returns=col(ret) if use_clip_v else ret.float().view(-1, 1))
    if is_coeffs is not None:
        batch["is_coeffs"] = col(is_coeffs)
    out = O.ppo_loss(v, lp, ent, batch, clip, c_v, c_e, use_clip_v)
    out["total_loss"].backward()
    dz, dv = z.grad.detach(), v.grad.detach().view(-1)
    ref = dict(values=v.detach().view(-1), log_probs=lp.detach().view(-1), entropy=ent.detach().view(-1))
    ref.update({k: out[k].detach() for k in METRICS})
    ref.update(d_features=x.grad, d_w_act=Wa.grad, d_b_act=ba.grad, d_w_val=Wv.grad.view(-1), d_b_val=bv.grad)

    # ---- bars (float64), per frame first
    d = lambda t: t.detach().double().view(-1)  # noqa: E731
    xd, Wad, Wvd = x.detach().double(), Wa.detach().double(), Wv.detach().double().view(-1)
    lpv, olp, advd, ovd, retd = d(lp), d(col(old_lp)), d(col(adv)), d(col(old_v)), d(col(ret))
    vv, entv = d(v), d(ent)
    cf = d(col(is_coeffs)).clamp(max=1.0) if is_coeffs is not None else torch.ones_like(vv)
    ratio = torch.exp(lpv - olp)
    ac = act.clamp(0, A - 1).view(-1, 1)
    lpbar_act = hd["logp_bar"].gather(1, ac).view(-1)
    rbar = ratio * (lpbar_act + K * U * (1 + (lpv - olp).abs()))
    g_lp, g_h = d(lp.grad), d(ent.grad)
    g_u = -advd * ratio * cf / B                          # the unclipped branch's d total / d lp
    lo, hi = 1.0 - clip, 1.0 + clip
    win = rbar + U * hi
    amb_r = ((advd > 0) & ((ratio - hi).abs() <= win)) | ((advd < 0) & ((ratio - lo).abs() <= win))
    live_r = (g_lp != 0) | amb_r                          # frames whose action gradient either branch may carry
    glpbar = torch.where(live_r, (advd.abs() * cf / B) * rbar + K * U * g_u.abs(), torch.zeros_like(g_u))
    pd, lpd = logp.detach().double().exp(), logp.detach().double()
    lpbar, entbar = hd["logp_bar"], hd["entropy_bar"]
    onehot = F.one_hot(ac.view(-1), A).double()
    pbar = pd * (lpbar + K * U)
    gl, gh = torch.where(amb_r, g_lp.abs().maximum(g_u.abs()), g_lp).view(-1, 1), g_h.view(-1, 1)
    dzbar = (glpbar.view(-1, 1) * (onehot - pd).abs() + gl.abs() * pbar
             + gh.abs() * (pbar * (lpd + entv.view(-1, 1)).abs() + pd * (lpbar + entbar.view(-1, 1)))
             + K * U * (gl.abs() * (1 + pd) + gh.abs() * pd * (lpd.abs() + entv.view(-1, 1).abs())))
    vbar = hd["values_bar"]
    vf = vv.float().double()   # O.ppo_loss runs the value path on values.float(), as the reference does
    delta = vf - ovd
    # (not |delta| < clip, as torch.where reads it: a NaN delta takes the clipped branch)
    clipped_v = ~(delta.abs() < clip) if use_clip_v else torch.zeros_like(vv, dtype=torch.bool)
    v_used = torch.where(clipped_v, ovd + delta.clamp(-clip, clip), vf)
    dvv = v_used - retd
    dvbar = vbar + K * U * (vv.abs() + ovd.abs() + retd.abs())

    # ---- branch-ambiguous frames and the other branch's gradients
    g_lp_alt = torch.where(g_lp == 0, g_u, torch.zeros_like(g_u))
    amb_v = torch.zeros_like(amb_r)
    if use_clip_v:
        amb_v = ((delta.abs() - clip).abs() <= vbar + K * U * (vv.abs() + ovd.abs() + clip))
    dv_alt = torch.where(clipped_v, c_v * (vf - retd) * cf / B, torch.zeros_like(vv))
    dz_alt = torch.where(amb_r.view(-1, 1), dz.double() + (g_lp_alt - g_lp).view(-1, 1) * (onehot - pd), dz.double())
    dv_alt = torch.where(amb_v, dv_alt, d(dv))
    gv_max = torch.where(amb_v, d(dv).abs().maximum(dv_alt.abs()), d(dv).abs())
    gvbar = torch.where(clipped_v & ~amb_v, 0.0, c_v * cf / B * dvbar + K * U * gv_max)

    Wfull = torch.cat([Wad, Wvd.view(1, -1)], 0).abs()
    dzfull = torch.cat([dz.double().abs().maximum(dz_alt.abs()), d(dv).abs().maximum(dv_alt.abs()).view(-1, 1)], 1)
    dzbarfull = torch.cat([dzbar, gvbar.view(-1, 1)], 1)
    xa = xd.abs()
    sB = K * U * math.sqrt(B)
    bars = dict(values=vbar, log_probs=lpbar_act, entropy=entbar)
    bars["d_features"] = (dzbarfull @ Wfull + K * U * math.sqrt(A + 1) * (dzfull @ Wfull)).expand(B, H)
    # the weight-gradient bars hold for the branches the kernel took: loss_ratios() reads them off its d_features
    # rows and adds only the differences it cannot tell apart
    # per-frame errors come from each frame's own roundings: they add like a random walk across the frames; the
    # partial sums the kernel rounds are about max(|sum t|, sqrt(sum t^2)) in size
    dzs = torch.cat([dz.double(), d(dv).view(-1, 1)], 1)
    wbar = ((dzbarfull ** 2).t() @ xa ** 2).sqrt() + sB * ((dzs.t() @ xd).abs()).maximum(((dzfull ** 2).t() @ xa ** 2).sqrt())
    bbar = (dzbarfull ** 2).sum(0).sqrt() + sB * dzs.sum(0).abs().maximum((dzfull ** 2).sum(0).sqrt())
    bars.update(d_w_act=wbar[:A], d_b_act=bbar[:A], d_w_val=wbar[A], d_b_val=bbar[A:])

    def mean_bar(t, tbar):
        return ((tbar.sum() + sB * t.abs().sum()) / B).view(())

    s1, s2 = advd * ratio, advd * ratio.clamp(lo, hi)
    t_v = cf * 0.5 * dvv ** 2
    t_a = -cf * torch.minimum(s1, s2)
    t_e = cf * entv
    bars["value_loss"] = mean_bar(t_v, cf * dvv.abs() * dvbar + K * U * t_v.abs())
    bars["action_loss"] = mean_bar(t_a, cf * advd.abs() * rbar + K * U * t_a.abs())
    bars["dist_entropy"] = mean_bar(t_e, cf * entbar + K * U * t_e.abs())
    bars["value_pred_min"] = bars["value_pred_max"] = vbar.max().view(())
    bars["value_pred_mean"] = mean_bar(vv, vbar)
    bars["prob_ratio_min"] = bars["prob_ratio_max"] = rbar.max().view(())
    bars["prob_ratio_mean"] = mean_bar(ratio, rbar)
    n_amb = int(amb_r.sum())
    ambf = (((ratio - hi).abs() <= win) | ((ratio - lo).abs() <= win)).sum().item()   # count decisions, both signs
    bars["ppo_fraction_clipped"] = torch.tensor((ambf + 0.5) / B, dtype=torch.float64)
    mv, ma, me = (ref[k].double().abs() for k in ("value_loss", "action_loss", "dist_entropy"))
    bars["total_loss"] = (c_v * bars["value_loss"] + bars["action_loss"] + c_e * bars["dist_entropy"]
                          + K * U * (c_v * mv + ma + c_e * me))
    ref["bars"] = bars
    ref["amb_r"], ref["amb_v"], ref["n_amb"] = amb_r, amb_v, n_amb
    ref["_state"] = dict(dz=dz.double(), dv=d(dv), dz_alt=dz_alt, dv_alt=dv_alt, x=xd, Wa=Wad, Wv=Wvd,
                         g_lp=g_lp, g_u=g_u, g_h=g_h, p=pd, ent=entv, onehot=onehot, clipped_v=clipped_v,
                         v_used=v_used, ret=retd, cf=cf, c_v=c_v, B=B,
                         coeffs=d(col(is_coeffs)) if is_coeffs is not None else None)
    return ref


def _grads_from(st, dz, dv):
    x, Wa, Wv = st["x"], st["Wa"], st["Wv"]
    return dict(d_features=dz @ Wa + dv.view(-1, 1) * Wv.view(1, -1), d_w_act=dz.t() @ x, d_b_act=dz.sum(0),
                d_w_val=dv @ x, d_b_val=dv.sum().view(1))


def alternate_grads(ref, flip="rv"):
    """the gradients with every branch-ambiguous frame on its other ratio branch ('r' in flip) and / or value branch
    ('v' in flip)"""
    st = ref["_state"]
    return _grads_from(st, st["dz_alt"] if "r" in flip else st["dz"], st["dv_alt"] if "v" in flip else st["dv"])


WGRADS = ("d_w_act", "d_b_act", "d_w_val", "d_b_val")


def branch_choice(got_d_features, ref):
    """The branch each frame of a loss call took, read off its d_features row: of the reference and the three
    alternatives (ratio branch flipped, value branch flipped, both; they differ only on branch-ambiguous frames) the
    one nearest in units of the bar, per row.  Returns the weight gradients of those choices, their bars, and the
    d_features error / bar of each row under its choice.  Where another choice also fits a row within the bar the
    weight-gradient bars grow by that frame's |difference| (times |x|); rows that can be told apart add nothing."""
    st = ref["_state"]
    A = st["Wa"].shape[0]
    dzs = (st["dz"], st["dz_alt"], st["dz"], st["dz_alt"])
    dvs = (st["dv"], st["dv"], st["dv_alt"], st["dv_alt"])
    bar = ref["bars"]["d_features"]
    g = got_d_features.double().to(bar.device).view(bar.shape)
    es = []
    for i, (a, b) in enumerate(zip(dzs, dvs)):
        df = ref["d_features"] if i == 0 else _grads_from(st, a, b)["d_features"]
        e = ((g - df).abs() / bar).max(-1).values
        es.append(torch.nan_to_num(e, nan=math.inf))
    es = torch.stack(es)                                       # [4, B]
    choice = es.argmin(0)
    rows = torch.arange(es.shape[1], device=es.device)
    r_flip, v_flip = ((choice == 1) | (choice == 3)).view(-1, 1), (choice >= 2)
    dz_c, dv_c = torch.where(r_flip, st["dz_alt"], st["dz"]), torch.where(v_flip, st["dv_alt"], st["dv"])
    full_c = torch.cat([dz_c, dv_c.view(-1, 1)], 1)
    allow = torch.zeros_like(full_c)
    for i, (a, b) in enumerate(zip(dzs, dvs)):
        diff = (torch.cat([a, b.view(-1, 1)], 1) - full_c).abs()
        allow = torch.maximum(allow, torch.where((es[i] <= 1.0).view(-1, 1), diff, torch.zeros_like(diff)))
    xa = st["x"].abs()
    grads = _grads_from(st, dz_c, dv_c)
    bars = {k: ref["bars"][k] for k in WGRADS}
    wx, ws = allow.t() @ xa, allow.sum(0)
    bars.update(d_w_act=bars["d_w_act"] + wx[:A], d_b_act=bars["d_b_act"] + ws[:A], d_w_val=bars["d_w_val"] + wx[A],
                d_b_val=bars["d_b_val"] + ws[A:])
    return dict(grads={k: grads[k] for k in WGRADS}, bars=bars, dz=dz_c, dv=dv_c, row_ratio=es[choice, rows])


def loss_ratios(got, ref, keys=None):
    """{output: max error / bar} of a loss call's outputs.  A d_features row may match either branch of a
    branch-ambiguous frame; the weight gradients are held to the reference built from the branches the rows show
    (branch_choice)."""
    ch = branch_choice(got["d_features"], ref)
    ref["_choice"] = ch
    out = {}
    for k in keys or ("values", "log_probs", "entropy") + METRICS + GRADS:
        g = got[k].double().to(ref[k].device).view(ref[k].shape)
        if k in WGRADS:
            r = ratio_to_bar(g, ch["grads"][k].view(g.shape), ch["bars"][k].view(g.shape))
        else:
            r = ratio_to_bar(g, ref[k], ref["bars"][k])
        if k == "d_features" and r > 0 and bool(torch.isfinite(g).all()):
            r = ch["row_ratio"].max().item()
        out[k] = r
    return out


def weight_grad_guards(ref):
    """{(fault, head): how many bars it misses by} for two faults of the weight-gradient path, against the reference
    of the branches loss_ratios() found: every weight gradient zeroed, and the last frame slab of
    ppo_heads_wgrad_kernel (blockIdx.y = min(32, cdiv(B, 64)) - 1) left out of the sums.  Per head (action: d_w_act
    and d_b_act; value: d_w_val and d_b_val) the larger miss counts: both come from the same slab partials, and a
    bias is one sum that can cancel by chance (26 value gradients of ~1e-3 summing to 4e-7 in one case).  Heads a
    fault leaves unchanged are not listed."""
    st, ch = ref["_state"], ref["_choice"]
    B = st["B"]
    gy = min(32, -(-B // 64))
    b0 = (gy - 1) * (-(-B // gy))
    keep = (torch.arange(B, device=ch["dv"].device) < b0)
    slab = _grads_from(st, ch["dz"] * keep.view(-1, 1), ch["dv"] * keep)
    out = {}
    for head, keys in (("action", ("d_w_act", "d_b_act")), ("value", ("d_w_val", "d_b_val"))):
        for name in ("zeroed", "last_slab_dropped"):
            miss = [ratio_to_bar(got, ch["grads"][k], ch["bars"][k]) for k in keys
                    for got in [torch.zeros_like(ch["grads"][k]) if name == "zeroed" else slab[k]]
                    if not torch.equal(got, ch["grads"][k])]
            if miss:
                out[(name, head)] = max(miss)
    return out


def perturb_grads(ref, perturb):
    """the gradients of a perturbed loss (see LOSS_PERTURBATIONS), or None where it cannot change this case"""
    st = ref["_state"]
    dz, dv, B = st["dz"].clone(), st["dv"].clone(), st["B"]
    if perturb == "straight_through_v":
        cv = st["clipped_v"]
        if not bool(cv.any()):
            return None
        dv = torch.where(cv, st["c_v"] * (st["v_used"] - st["ret"]) * st["cf"] / B, dv)
    elif perturb == "grad_through_clip":
        dz = dz + (st["g_u"] - st["g_lp"]).view(-1, 1) * (st["onehot"] - st["p"])
    elif perturb == "entropy_no_h":
        dz = dz + (st["g_h"] * st["ent"]).view(-1, 1) * st["p"]
    elif perturb == "is_unclamped":
        c = st["coeffs"]
        if c is None or not bool((c > 1).any()):
            return None
        s = torch.where(c > 1, c / st["cf"], torch.ones_like(c))
        dz, dv = dz * s.view(-1, 1), dv * s
    out = _grads_from(st, dz, dv)
    if all(torch.equal(out[k], g) for k, g in _grads_from(st, st["dz"], st["dv"]).items()):
        return None
    return out


REGIME_FRAMES = 2


def make_loss_case(B, H, A, seed=0, is_mode="none", b_act_zero=False, clip=0.2, large_logits=True):
    """CPU fp32 operands of one loss call.  REGIME_FRAMES frames, spread over the batch, of each regime: 0 logits =
    b_act (uniform with b_act = 0), 1 |z| ~ 1e3 (probabilities that underflow to 0), 2-4 ratio on and one ulp either
    side of 1 + clip, 5-7 the same at 1 - clip, 8-9 |v - old_v| on the value-clip boundary.  The rest are a random mix
    of clipped / unclipped ratios and advantage signs, frame 0 clipped.  The regime frames are few on purpose, so the
    weight-gradient sums stay dominated by ordinary frames.  large_logits = False leaves regime 1 out: its features
    are ~1e3 times larger than the others, and their legitimate fp32 error (u |z| per logit, times |x|) then sets the
    weight-gradient bars, too large to see a missing frame slab.  is_mode: none, rand (in [0, 1.6]) or ones."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    x = rn(B, H)
    Wa, ba = rn(A, H) * (0.5 / math.sqrt(H)), (torch.zeros(A) if b_act_zero else rn(A) * 0.1)
    Wv, bv = rn(1, H) * (0.5 / math.sqrt(H)), rn(1)
    kind = torch.full((B,), 10)
    for j in range(10 * REGIME_FRAMES):   # REGIME_FRAMES frames of each regime 0-9, spread over the batch
        kind[((j + 1) * B) // (10 * REGIME_FRAMES + 1)] = j % 10
    if not large_logits:
        kind[kind == 1] = 10
    x[kind == 0] = 0.0
    z0 = x[kind == 1] @ Wa.t()
    if A > 1 and z0.numel():
        x[kind == 1] *= 1e3 / z0.abs().amax(-1, keepdim=True).clamp_min(1e-3)
    actions = torch.randint(0, A, (B,), generator=g)
    with torch.no_grad():
        hd = heads(x, Wa, ba, Wv, bv)
    lp = hd["logp"].gather(1, actions.view(-1, 1)).view(-1)
    v = hd["values"]
    clip32 = f32(clip)
    olp = lp + 0.3 * rn(B).double()
    adv = rn(B)
    hi, lo = torch.tensor(1.0, dtype=torch.float32) + clip32, torch.tensor(1.0, dtype=torch.float32) - clip32
    up, dn = torch.tensor(math.inf), torch.tensor(-math.inf)
    targets = {2: hi, 3: torch.nextafter(hi, up), 4: torch.nextafter(hi, dn),
               5: lo, 6: torch.nextafter(lo, up), 7: torch.nextafter(lo, dn)}
    for k, tg in targets.items():
        sel = kind == k
        olp[sel] = lp[sel] - math.log(float(tg))
    ov = v + 0.3 * rn(B).double()
    for k, sgn in ((8, 1.0), (9, -1.0)):
        sel = kind == k
        ov[sel] = v[sel] - sgn * clip32
    olp[0], adv[0] = lp[0] - math.log(1.5), 1.0   # frame 0 always clipped (ratio 1.5, adv > 0)
    ret = v + rn(B).double()
    isc = {"none": None, "rand": torch.rand(B, generator=g) * 1.6, "ones": torch.ones(B)}[is_mode]
    return dict(feat=x, w_act=Wa, b_act=ba, w_val=Wv, b_val=bv, actions=actions, old_lp=olp.float(), adv=adv,
                old_v=ov.float(), ret=ret.float(), is_coeffs=isc)


# ---------------------------------------------------------------------------------------------------------------------
# clip + Adam
# ---------------------------------------------------------------------------------------------------------------------
def clip_adam(p, g, m, v, lr, betas, eps, weight_decay, max_norm, grad_scale, step, perturb=None,
              dtype=torch.float64):
    """clip_grad_norm_(max_norm) of g * grad_scale + one torch.optim.Adam step (weight_decay folded into the gradient,
    as Adam does) on fp32 operands, all hyper-parameters as fp32 values.  max_norm <= 0: no clipping.  Returns
    dict(params, exp_avg, exp_avg_sq, norm) and their bars, or None where the perturbation cannot change the case."""
    lr, b1, b2, eps, wd, mx, gs = (f32(t) for t in (lr, betas[0], betas[1], eps, weight_decay, max_norm, grad_scale))
    if perturb == "scale_after_norm" and (gs == 1.0 or mx <= 0):
        return None
    p, g, m, v = (t.to(dtype) for t in (p, g, m, v))
    gsc = g * gs
    norm = torch.sqrt(((g if perturb == "scale_after_norm" else gsc).double() ** 2).sum()).to(dtype)
    coef = torch.clamp(mx / (norm + 1e-6), max=1.0) if mx > 0 else torch.ones((), dtype=dtype, device=g.device)
    gg = gsc * coef
    if wd != 0:
        gg = gg + wd * p
    st = step + 1 if perturb == "bias_step" else step
    bc1, bc2 = 1 - b1 ** st, 1 - b2 ** st
    m2 = m.lerp(gg, 1 - b1)
    v2 = v * b2 + (1 - b2) * gg * gg
    if perturb == "eps_in_sqrt":
        denom = (v2 / bc2 + eps).sqrt()
    else:
        denom = v2.sqrt() / math.sqrt(bc2) + eps
    p2 = p - (lr / bc1) * m2 / denom
    ga = (gsc * coef).double().abs() + abs(wd) * p.double().abs()
    M = m.double().abs() + (1 - b1) * (ga + m.double().abs())
    return dict(params=p2, exp_avg=m2, exp_avg_sq=v2, norm=norm,
                bar_params=K * U * (p.double().abs() + 3 * (lr / bc1) * M / denom.double()),
                bar_exp_avg=K * U * M, bar_exp_avg_sq=K * U * v2.double().abs(), bar_norm=K * U * norm.double())
