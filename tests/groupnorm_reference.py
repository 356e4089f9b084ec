"""Plain float64 references of the GroupNorm, max-pool and observation-prep kernels in csrc/elementwise.cu, their
per-element error bars, and the host dispatch rules that pick a kernel for a shape.  Shared by
tests/test_gpu_groupnorm.py and tests/test_groupnorm_reference_cpu.py.

Layouts are the kernels' own: activations NHWC flattened to [B, HW, C], statistics [B, G, 2] float64 (sum, sum of
squares over the group's HW * C/G values, as the conv epilogues produce them).  Every reference takes the kernels'
rounded operands (fp16 y / act / res, bf16 g / dpool, fp32 gamma / beta) and runs in float64, in frame chunks of at
most CHUNK frames; GroupNorm is per frame, so chunking is exact, and dgamma / dbeta are accumulated across chunks in
float64.

Bars (u = 2^-24; uh = 2^-11 and ub = 2^-8 are the fp16 / bf16 unit roundoffs)
-----------------------------------------------------------------------------
Forward.  The kernels evaluate z = gamma (x - mu) rstd + beta either as fmaf((x - mu) rs, gamma, beta) (two-pass /
  fused backward, generic pool) or as fmaf(x, rs gamma, beta - mu rs gamma) (gn_apply, gn_residual_relu, slab pool,
  cluster backward).  mu and rstd come from the float64 sums rounded to fp32, rsqrtf is within 2 ulp.  Each formula
  rounds a handful of times on terms no larger than |x sc|, |mu sc| and |beta| (sc = rstd gamma), so
      e(z) = K u (|x sc| + |mu sc| + |beta|) + K d_rs |x - mu| |sc|,   K = 8,
  where d_rs = u (mu^2 + var) / (var + eps) is the relative rstd error of E[x^2] * inv_m rounded through an fp32
  inv_m; it is 0 when C/G * HW is a power of two (inv_m exact).  The residual sum adds the residual's own e(z) and
  one rounding.  ReLU and max are 1-Lipschitz, so the pooled value's bar is the window's largest e(z).  A stored
  output adds its format's half ulp: uh |z| + 2^-25 (fp16, with subnormals), ub |z| (bf16), 0 (fp32).
ReLU ambiguity band.  Where |z| <= e(z) the fp32 sign may differ from float64's.  The backward's mask there can go
  either way: those elements are excluded from per-element checks (band()), counted, and their |g| (|g x_hat|) is
  added to the sums' bars below.
Backward sums.  A = sum gz, Bx = sum gz x_hat per (frame, channel) are fp32 sums over HW pixels in blocks of at most
  256 serial terms followed by trees; the rounding errors of D serial steps add like a random walk, at most
  sqrt(D) <= 16 times one rounding of the sum of |terms|:
      e(A) = KS u sum|gz| + sum_band |g|,   KS = 16,
      e(Bx) = KS u sum|gz x_hat| + K u |mu rstd| |A| + K d_rs |Bx| + sum_band |g x_hat|,
  where the middle terms are x_hat's fp32 rounding of mu and of rstd, common to every pixel of a group.
  S1 = sum_{c in group} gamma_c A_c and S2 likewise carry sum |gamma_c| e(.) + KS u sum |gamma_c .|, and
      e(dy) = K u rstd (|gamma gz| + (|S1| + (|x_hat| + 2 |mu| rstd) |S2|) / m) + rstd (e(S1) + |x_hat| e(S2)) / m
              + 2 K d_rs |dy| + ub |dy|.
  dgamma / dbeta sum the per-frame rows over B frames in a fixed order (32 chunks, then the chunk totals):
      e(dgamma) = sum_b e(Bx_b) + KS u sum_b |Bx_b|, and dbeta alike.
Prep.  The pooled value is four fp32 products and adds on non-negative terms: 4 u |x|; the RunningMeanAndVar merge
  runs on fp32-accumulated float64 sums and in fp32: e(mean) = KS u (rms(x) + |mean|), e(var) = KS u (E[x^2] + var +
  (new_mean - mean)^2) per update.  The output is fmaf(x, inv, -mean inv): e = K u (|x inv| + |mean inv|).
"""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
UH = 2.0 ** -11
UB = 2.0 ** -8
K = 8.0
KS = 16.0
CHUNK = 256
F16_SUB = 2.0 ** -25   # half the fp16 subnormal spacing


# ---------------------------------------------------------------------------------------------------------------
# host dispatch rules (restated from csrc/elementwise.cu; pure arithmetic on the shape)
# ---------------------------------------------------------------------------------------------------------------
def gn_bwd_path(C, G, hw, mask_mode):
    """hb200_gn_bwd: ('cluster', cluster size, pixels per CTA) or ('fused', None, None)"""
    cv = C // 8
    if cv <= 32:
        ntens = 3 if mask_mode == 2 else 2
        cs = 1
        while True:
            ppc = (hw + cs - 1) // cs
            slice_ = ntens * ppc * C * 2
            if slice_ <= 48 * 1024 or cs == 8:
                break
            cs *= 2
        if slice_ + 4 * (20 * C + 2 * G) <= 200 * 1024:
            return ("cluster", cs, ppc)
    return ("fused", None, None)


def gn_pool_fwd_path(C, h, w):
    """hb200_gn_relu_maxpool: ('slab', rows) or ('generic', None)"""
    cv = C // 8
    if h % 2 == 0 and w % 2 == 0:
        rows = 0
        for r in (8, 6, 4, 2):
            if h % r == 0 and (r + 1) * w * C * 2 <= 64 * 1024:
                rows = r
                break
        if rows and cv <= 32 and 256 % cv == 0:
            return ("slab", rows)
    return ("generic", None)


def gn_pool_bwd_plan(h, w, C, G):
    """gn_pool_bwd_plan: (cluster size, rows per CTA), or None where hb200_gn_relu_maxpool_bwd is unsupported"""
    cv = C // 8
    if C % 8 or cv < 1 or cv > 32 or 256 % cv or h % 2 or w % 2:
        return None
    for cs in (1, 2, 4, 8):
        if h % (2 * cs):
            continue
        rows = h // cs
        nbytes = rows * w * C * 2 + (rows // 2 + 1) * (w // 2) * C * 3 + 4 * (20 * C + 2 * G)
        if nbytes <= 50 * 1024 or (cs == 8 and nbytes <= 200 * 1024):
            return cs, rows
    return None


# ---------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------
def stats_of(y, G):
    """[B, HW, C] -> float64 [B, G, 2] (sum, sum of squares per group)"""
    B, hw, C = y.shape
    out = torch.empty(B, G, 2, dtype=torch.float64, device=y.device)
    for b0 in range(0, B, CHUNK):
        yg = y[b0:b0 + CHUNK].double().reshape(-1, hw, G, C // G).transpose(1, 2).reshape(-1, G, hw * C // G)
        out[b0:b0 + CHUNK, :, 0] = yg.sum(-1)
        out[b0:b0 + CHUNK, :, 1] = (yg * yg).sum(-1)
    return out


def _inv_m_exact(C, G, hw):
    n = (C // G) * hw
    return n & (n - 1) == 0


def coeffs(stats, C, G, hw, eps):
    """per-channel mean, rstd [B, C] and the relative rstd error d_rs [B, C] of an fp32 inv_m (see the bars)"""
    m = (C // G) * hw
    mean = stats[..., 0] / m
    var = (stats[..., 1] / m - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + eps)
    d_rs = torch.zeros_like(var) if _inv_m_exact(C, G, hw) else U * (mean * mean + var) / (var + eps)
    rep = lambda t: t.repeat_interleave(C // G, dim=1)  # noqa: E731
    return rep(mean), rep(rstd), rep(d_rs)


def _gn_z(x, mean, rstd, d_rs, gamma, beta):
    """z = gamma x_hat + beta and its fp32 bar e(z); x [b, HW, C], per-channel [b, 1, C]"""
    sc = rstd * gamma
    z = (x - mean) * sc + beta
    e = K * U * ((x * sc).abs() + (mean * sc).abs() + beta.abs()) + K * d_rs * ((x - mean) * sc).abs()
    return z, e


def out_bar(ref, fmt):
    a = ref.abs()
    if fmt == "f16":
        return UH * a + F16_SUB
    if fmt == "bf16":
        return UB * a
    return torch.zeros_like(a)


def gn_forward(y, stats, gamma, beta, G, eps=1e-5, relu=True, res=None, res_stats=None, res_gamma=None,
               res_beta=None):
    """relu?(GN(y)) or relu(GN(y) + res) or relu(GN(y) + GN_d(res)); returns (value, fp32 bar before the output
    rounding, band mask |z| <= e(z)).  y / res [B, HW, C], any float dtype."""
    B, hw, C = y.shape
    dev = y.device
    ga, be = gamma.double().view(1, 1, C).to(dev), beta.double().view(1, 1, C).to(dev)
    mean, rstd, d_rs = coeffs(stats.to(dev), C, G, hw, eps)
    if res_stats is not None:
        rmean, rrstd, rd = coeffs(res_stats.to(dev), C, G, hw, eps)
        rga, rbe = res_gamma.double().view(1, 1, C).to(dev), res_beta.double().view(1, 1, C).to(dev)
    val = torch.empty(B, hw, C, dtype=torch.float64, device=dev)
    bar = torch.empty_like(val)
    band = torch.empty(B, hw, C, dtype=torch.bool, device=dev)
    for b0 in range(0, B, CHUNK):
        s = slice(b0, b0 + CHUNK)
        z, e = _gn_z(y[s].double(), mean[s, None], rstd[s, None], d_rs[s, None], ga, be)
        if res is not None:
            r = res[s].double()
            if res_stats is not None:
                r, er = _gn_z(r, rmean[s, None], rrstd[s, None], rd[s, None], rga, rbe)
                e = e + er
            e = e + U * (z.abs() + r.abs())
            z = z + r
        band[s] = z.abs() <= e
        val[s] = z.clamp_min(0.0) if (relu or res is not None) else z
        bar[s] = e
    return val, bar, band


def band(y, stats, gamma, beta, G, eps=1e-5):
    """elements whose float64 pre-ReLU value lies within the fp32 error of zero"""
    return gn_forward(y, stats, gamma, beta, G, eps, relu=False)[2]


def gn_backward(g, y, stats, gamma, beta, G, mask_mode, act=None, eps=1e-5):
    """exact float64 gradient of [relu](group_norm(y)) seeded with g (mask_mode 0: none, 1: z > 0, 2: act > 0), the
    statistics being the sums of y itself.  Returns dict dy, gz, dgamma, dbeta, the per-frame rows A / Bx [B, C], the
    bars e_dy (per element), e_A / e_Bx (per frame row), e_dgamma / e_dbeta, and the band mask (mode 1 only)."""
    B, hw, C = y.shape
    dev = y.device
    cpg = C // G
    m = cpg * hw
    ga = gamma.double().to(dev)
    mean, rstd, d_rs = coeffs(stats.to(dev), C, G, hw, eps)
    out = {k: torch.empty(B, hw, C, dtype=torch.float64, device=dev) for k in ("dy", "gz", "e_dy")}
    out["band"] = torch.zeros(B, hw, C, dtype=torch.bool, device=dev)
    for k in ("A", "Bx", "e_A", "e_Bx"):
        out[k] = torch.empty(B, C, dtype=torch.float64, device=dev)
    gsum = lambda t: t.view(t.shape[0], G, cpg).sum(-1).repeat_interleave(cpg, dim=1)  # noqa: E731  per group
    for b0 in range(0, B, CHUNK):
        s = slice(b0, b0 + CHUNK)
        x, gg = y[s].double(), g[s].double()
        mu, rs = mean[s, None], rstd[s, None]
        xh = (x - mu) * rs
        if mask_mode == 1:
            z, e = _gn_z(x, mu, rs, d_rs[s, None], ga, beta.double().to(dev))
            bd = z.abs() <= e
            out["band"][s] = bd
            gz = gg * (z > 0)
        elif mask_mode == 2:
            bd = None
            gz = gg * (act[s].double() > 0)
        else:
            bd = None
            gz = gg
        A, Bx = gz.sum(1), (gz * xh).sum(1)
        # x_hat carries the fp32 rounding of mu (the same for every pixel of the group) and of rstd
        eA = KS * U * gz.abs().sum(1)
        eB = KS * U * (gz * xh).abs().sum(1) + K * U * (mu * rs).abs()[:, 0] * A.abs() + K * d_rs[s] * Bx.abs()
        if bd is not None:
            eA = eA + (gg.abs() * bd).sum(1)
            eB = eB + ((gg * xh).abs() * bd).sum(1)
        S1, S2 = gsum(ga * A), gsum(ga * Bx)
        eS1 = gsum(ga.abs() * eA) + KS * U * gsum((ga * A).abs())
        eS2 = gsum(ga.abs() * eB) + KS * U * gsum((ga * Bx).abs())
        dy = rs * (ga * gz - (S1[:, None] + xh * S2[:, None]) / m)
        e_dy = (K * U * rs * ((ga * gz).abs() + (S1.abs()[:, None] + (xh.abs() + 2 * mu.abs() * rs) * S2.abs()[:, None]) / m)
                + rs * (eS1[:, None] + xh.abs() * eS2[:, None]) / m + 2 * K * d_rs[s, None] * dy.abs())
        out["dy"][s], out["gz"][s], out["e_dy"][s] = dy, gz, e_dy
        out["A"][s], out["Bx"][s], out["e_A"][s], out["e_Bx"][s] = A, Bx, eA, eB
    out["dbeta"], out["dgamma"] = out["A"].sum(0), out["Bx"].sum(0)
    out["e_dbeta"] = out["e_A"].sum(0) + KS * U * out["A"].abs().sum(0)
    out["e_dgamma"] = out["e_Bx"].sum(0) + KS * U * out["Bx"].abs().sum(0)
    return out


# ---------------------------------------------------------------------------------------------------------------
# MaxPool2d(3, 2, 1) after GroupNorm + ReLU
# ---------------------------------------------------------------------------------------------------------------
def pool_out_hw(h, w):
    return (h + 1) // 2, (w + 1) // 2


def _taps(t, h, w, fill):
    """[b, h*w, C] -> [9, b, Ho, Wo, C]: the 3x3 stride-2 pad-1 windows, tap r*3+s, padding = fill"""
    b, _, C = t.shape
    Ho, Wo = pool_out_hw(h, w)
    p = torch.full((b, 2 * Ho + 1, 2 * Wo + 1, C), fill, dtype=t.dtype, device=t.device)
    p[:, 1:h + 1, 1:w + 1] = t.view(b, h, w, C)
    return torch.stack([p[:, r:r + 2 * Ho:2, s:s + 2 * Wo:2] for r in range(3) for s in range(3)])


def first_max(vals):
    """max over dim 0 and the first index reaching it (torch's max_pool2d rule: a later tap wins only if greater)"""
    mx = vals.max(0).values
    idx = torch.arange(vals.shape[0], device=vals.device).view(-1, *([1] * (vals.dim() - 1)))
    return mx, torch.where(vals == mx, idx, vals.shape[0]).min(0).values


def gn_relu_maxpool(y, stats, gamma, beta, G, h, w, eps=1e-5):
    """pooled relu(GN(y)) [B, Ho*Wo, C], its fp32 bar, the argmax tap codes (uint8) by the first-maximum rule,
    `ambiguous`: windows where a tap other than the winner, with a different float64 z, lies within the two taps'
    bars of the maximum (fp32 may pick either), or whose maximum is within its bar of 0, and `dead`: windows whose
    every tap has z < -e(z), so their pooled value is 0 in any evaluation and no gradient passes the ReLU."""
    B, _, C = y.shape
    Ho, Wo = pool_out_hw(h, w)
    val = torch.empty(B, Ho * Wo, C, dtype=torch.float64, device=y.device)
    bar = torch.empty_like(val)
    code = torch.empty(B, Ho * Wo, C, dtype=torch.uint8, device=y.device)
    amb = torch.empty(B, Ho * Wo, C, dtype=torch.bool, device=y.device)
    dead = torch.empty_like(amb)
    z_all, e_all, _ = gn_forward(y, stats, gamma, beta, G, eps, relu=False)
    for b0 in range(0, B, CHUNK):
        s = slice(b0, b0 + CHUNK)
        zpre = _taps(z_all[s], h, w, -math.inf)
        et = _taps(e_all[s], h, w, 0.0)
        zt = zpre.clamp_min(0.0)
        zt[zpre == -math.inf] = -math.inf
        mx, arg = first_max(zt)
        ew = et.gather(0, arg[None])[0]
        near = (zt < mx) & (zt >= mx - ew - et)
        val[s] = mx.reshape(-1, Ho * Wo, C)
        bar[s] = et.max(0).values.reshape(-1, Ho * Wo, C)
        code[s] = arg.to(torch.uint8).reshape(-1, Ho * Wo, C)
        amb[s] = (near.any(0) | (mx <= ew)).reshape(-1, Ho * Wo, C)
        dead[s] = (zpre < -et).all(0).reshape(-1, Ho * Wo, C)
    return val, bar, code, amb, dead


def maxpool_route(dpool, code, h, w):
    """MaxPool2d(3, 2, 1) backward given the argmax tap codes: [B, Ho*Wo, C] -> [B, h*w, C] float64"""
    B, _, C = dpool.shape
    Ho, Wo = pool_out_hw(h, w)
    dz = torch.zeros(B, 2 * Ho + 1, 2 * Wo + 1, C, dtype=torch.float64, device=dpool.device)
    dp = dpool.double().view(B, Ho, Wo, C)
    cd = code.view(B, Ho, Wo, C)
    for r in range(3):
        for s in range(3):
            dz[:, r:r + 2 * Ho:2, s:s + 2 * Wo:2] += dp * (cd == r * 3 + s)
    return dz[:, 1:h + 1, 1:w + 1].reshape(B, h * w, C)


def gn_relu_maxpool_bwd(dpool, code, y, stats, gamma, beta, G, h, w, eps=1e-5):
    """backward of pool, ReLU and GroupNorm together (what gn_relu_maxpool_bwd fuses): gn_backward mode 1 seeded with
    the routed pooled gradient"""
    return gn_backward(maxpool_route(dpool, code, h, w), y, stats, gamma, beta, G, 1, eps=eps)


# ---------------------------------------------------------------------------------------------------------------
# observation prep (ResNetEncoder.forward up to the backbone)
# ---------------------------------------------------------------------------------------------------------------
def prep_pooled(rgb, depth, frame_rows, dtype=torch.float64):
    """avg_pool2d(cat(rgb * (1/255), depth), 2) of the gathered frames, NHWC [B, H/2, W/2, C]"""
    rows = frame_rows.long()
    xs = []
    if rgb is not None:
        xs.append(rgb[rows].to(dtype) * (1.0 / 255.0))
    if depth is not None:
        xs.append(depth[rows].to(dtype))
    x = torch.cat(xs, -1)
    B, H, W, C = x.shape
    return x.view(B, H // 2, 2, W // 2, 2, C).sum((2, 4)) * 0.25


def running_merge(x_sum, x_sqsum, n_el, frames, mean, var, count):
    """RunningMeanAndVar's merge of one batch (float64): per-channel sums over the batch's n_el values per channel"""
    new_mean = x_sum / n_el
    new_var = (x_sqsum / n_el - new_mean * new_mean).clamp_min(0.0)
    new_count = float(frames)
    m2 = var * count + new_var * new_count + (new_mean - mean) ** 2 * count * new_count / (count + new_count)
    tot = count + new_count
    return (count * mean + new_count * new_mean) / tot, m2 / tot, tot


def running_merge_bars(x_sum, x_sqsum, n_el, mean, var):
    new_mean = x_sum / n_el
    ex2 = x_sqsum / n_el
    e_mean = KS * U * (ex2.sqrt() + mean.abs())
    e_var = KS * U * (ex2 + var + (new_mean - mean) ** 2)
    return e_mean, e_var


def prep_normalise(x, mean, var):
    """(x - mean) / sqrt(max(var, 1e-2)) and its fp32 bar; x [..., C], mean / var [C]"""
    inv = 1.0 / torch.sqrt(var.double().clamp_min(1e-2))
    mean = mean.double()
    return (x - mean) * inv, K * U * ((x * inv).abs() + (mean * inv).abs())


def nhwc8(x):
    """[B, Hp, Wp, C<=4] -> the kernels' 8-channel zero-padded layout"""
    return F.pad(x, (0, 8 - x.shape[-1]))


def s2d(x):
    """[B, Hp, Wp, C<=4] -> [B, Hp/2, Wp/2, 16] with channel (dy * 2 + dx) * 4 + c"""
    B, Hp, Wp, C = x.shape
    x4 = F.pad(x, (0, 4 - C))
    return x4.view(B, Hp // 2, 2, Wp // 2, 2, 4).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp // 2, Wp // 2, 16)
