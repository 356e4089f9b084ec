"""Plain reference of the masked LSTM / GRU recurrence in csrc/rnn.cu, its error bars, and the perturbed references that
show each bar is tight.  Shared by tests/test_gpu_recurrence.py and tests/test_recurrence_reference_cpu.py.

The reference starts from the kernels' own operands (xproj, W_hh, b_hh, h0, c0, masks), so the input-projection GEMM is
not part of any comparison:

  LSTM  h_in = h_{t-1} m_t,  c_in = c_{t-1} m_t,  (i, f, g, o) = (sig, sig, tanh, sig)(xproj_t + h_in W_hh^T + b_hh)
        c_t = f c_in + i g,   h_t = o tanh(c_t)
  GRU   h_in = h_{t-1} m_t,  gh = h_in W_hh^T + b_hh,  r = sig(x_r + gh_r),  z = sig(x_z + gh_z)
        n = tanh(x_n + r gh_n),  h_t = (1 - z) n + z h_in

The backward is autograd through that loop seeded with dh_out = dL/dhs (the kernels take no separate gradient of the
final state): dgates / dgx = dL/dxproj and, for the GRU, dgh = dL/dgh, whose n part is dL/dn_pre * r (hb200.h).

Error bars (max-abs error over the reference's max, one bar per output)
----------------------------------------------------------------------
u = 2^-24.  A step's pre-activation is an fp32 dot product of length H (fma chains plus a shuffle tree) and two adds;
with |h| <= 1 and the unit-norm columns of an orthogonal W_hh its rounding error is about u * sqrt(H) (independent
roundings add like a random walk; the worst-case bound H u is never approached).  expf / tanhf add at most two ulp, the
cell update a few u of |c|.  The step contracts its state (sigmoid' <= 1/4, f < 1, ||W_hh|| = 1): an error made at
step t is damped at every later step, so the error does not grow with T and stays at the one-step size.  The
backward runs the same contraction in reverse on operands that carry the forward's error, with one 4H-long (GRU: 3H)
dot product per unit and step.  So every bar is

    K * u * sqrt(H),   K = 16            (hs, cs, gates, saved, dgates, dgx, dgh)

The fp32 recurrence on the CPU (a third summation order, with its own expf / tanhf) measures at most 1.1 u sqrt(H) on
every output over the shapes, mask patterns and saturated cases of the GPU tests, with no trend in T from 1 to 128
(tests/test_recurrence_reference_cpu.py checks it at smaller shapes).  K = 16 leaves a factor of ~15 over that for
the kernels' different reduction trees and GPU math functions.  The bar is 2.2e-5 of the output's max at H = 512.
Every perturbed reference changes an output by 1e-3 of its max or more, hundreds of times the bar; the tests require
at least 10x case by case, and skip a perturbation only where it does not change the exact result at all (a reset
ignored where there is none, a stale h behind a reset, a carry cut where every sequence resets anyway).
"""
import math

import torch

U = 2.0 ** -24
K = 16.0

FWD_PERTURBATIONS = ("stale_h", "ignore_reset", "drop_b_hh")
GRU_FWD_PERTURBATIONS = FWD_PERTURBATIONS + ("bhn_outside_r",)
LSTM_BWD_PERTURBATIONS = ("drop_dh", "unmask_dc", "cut_carry")
GRU_BWD_PERTURBATIONS = ("drop_dh", "dgh_without_r")


def bar(H):
    """atol of every output, as a fraction of the reference's max"""
    return K * U * math.sqrt(H)


def _last_reset(m):
    """(t, n - 1) of the latest reset of the last sequence, or None"""
    ts = (m[:, -1] == 0).nonzero().flatten()
    return None if ts.numel() == 0 else int(ts[-1])


def recurrence(kind, xproj, w_hh, b_hh, h0, c0, masks, dh_out=None, perturb=None, dtype=torch.float64):
    """kind 'lstm' / 'gru'; xproj [T, n, G*H], masks [T, n] (nonzero = no reset), h0 / c0 [n, H] (c0 ignored for the
    GRU), dh_out [T, n, H] or None.  perturb names one deliberate fault (see FWD_ / *_BWD_PERTURBATIONS):
      stale_h        the last 4 hidden units (the last CTA) read h_{t-2} instead of h_{t-1} at the last step
                     (h_{-1} = 0: a buffer no step has written)
      ignore_reset   the latest reset of the last sequence is ignored
      drop_b_hh      b_hh left out
      bhn_outside_r  (GRU) n = tanh(x_n + r (W_hn h) + b_hn)
      drop_dh        no gradient through h_in W_hh^T at the last step
      unmask_dc      (LSTM) dc flows through the latest reset (t >= 1) of the last sequence
      cut_carry      (LSTM) no gradient into h_{t-1}, c_{t-1} at t = T / 2 (a zeroed carry at a chunk boundary)
      dgh_without_r  (GRU) the n part of dgh is dL/dn_pre, not dL/dn_pre * r
    Returns a dict of hs, cs (LSTM), gates (LSTM: i, f, g, o) / saved (GRU: r, z, n, W_hn h + b_hn) and, with dh_out,
    dgates (LSTM) / dgx, dgh (GRU); or None when the perturbation does not apply to this case."""
    lstm = kind == "lstm"
    T, n, GH = xproj.shape
    H = GH // (4 if lstm else 3)
    m = (masks.reshape(T, n) != 0).to(dtype=dtype, device=xproj.device)
    if perturb == "ignore_reset" or perturb == "unmask_dc":
        tr = _last_reset(m)
        if tr is None or (perturb == "unmask_dc" and tr == 0):
            return None
    if perturb in ("stale_h", "drop_dh", "cut_carry") and T < 2:
        return None
    if perturb == "ignore_reset":
        m = m.clone()
        m[tr, -1] = 1.0
    grad = dh_out is not None
    x = xproj.to(dtype).detach().requires_grad_(grad)
    w = w_hh.to(dtype)
    b = torch.zeros(GH, dtype=dtype, device=w.device) if b_hh is None or perturb == "drop_b_hh" else b_hh.to(dtype)
    h, c = h0.to(dtype), (c0.to(dtype) if lstm else None)
    hs, cs, acts, ghs = [], [], [], []
    for t in range(T):
        mt = m[t].unsqueeze(1)
        hp, cp = h, c
        if perturb == "cut_carry" and t == T // 2:
            hp, cp = hp.detach(), (cp.detach() if lstm else None)
        h_in = hp * mt
        h_rec = h_in.detach() if perturb == "drop_dh" and t == T - 1 else h_in
        gh = h_rec @ w.t() + b
        if perturb == "stale_h" and t == T - 1:
            stale = (hs[t - 2] if t >= 2 else torch.zeros_like(h)) * mt
            cols = torch.zeros(GH, dtype=torch.bool, device=w.device)
            cols.view(-1, H)[:, H - 4:] = True
            gh = torch.where(cols, stale @ w.t() + b, gh)
        xt = x[t]
        if lstm:
            c_in = cp * mt
            if perturb == "unmask_dc" and t == tr:
                keep = torch.zeros_like(mt)
                keep[-1] = 1.0
                c_in = c_in + keep * (cp - cp.detach())    # same value, gradient no longer masked
            pre = xt + gh
            i_, f_, o_ = (torch.sigmoid(pre[:, k * H:(k + 1) * H]) for k in (0, 1, 3))
            g_ = torch.tanh(pre[:, 2 * H:3 * H])
            c = f_ * c_in + i_ * g_
            h = o_ * torch.tanh(c)
            acts.append(torch.cat([i_, f_, g_, o_], 1))
            cs.append(c)
        else:
            if grad:   # a zero leaf per step: its gradient is dL/dgh_t (h0 does not require grad at t = 0)
                probe = torch.zeros_like(gh, requires_grad=True)
                ghs.append(probe)
                gh = gh + probe
            r_ = torch.sigmoid(xt[:, :H] + gh[:, :H])
            z_ = torch.sigmoid(xt[:, H:2 * H] + gh[:, H:2 * H])
            if perturb == "bhn_outside_r":
                n_ = torch.tanh(xt[:, 2 * H:] + r_ * (gh[:, 2 * H:] - b[2 * H:]) + b[2 * H:])
            else:
                n_ = torch.tanh(xt[:, 2 * H:] + r_ * gh[:, 2 * H:])
            h = (1 - z_) * n_ + z_ * h_in
            acts.append(torch.cat([r_, z_, n_, gh[:, 2 * H:]], 1))
        hs.append(h)
    out = {"hs": torch.stack(hs)}
    if lstm:
        out.update(cs=torch.stack(cs), gates=torch.stack(acts))
    else:
        out["saved"] = torch.stack(acts)
    if grad:
        (out["hs"] * dh_out.to(dtype)).sum().backward()
        if lstm:
            out["dgates"] = x.grad
        else:
            out["dgx"] = x.grad
            dgh = torch.stack([g.grad for g in ghs])
            if perturb == "dgh_without_r":
                dgh = torch.cat([dgh[..., :2 * H], x.grad[..., 2 * H:]], -1)
            out["dgh"] = dgh
    return {k: v.detach() for k, v in out.items()}


MASK_PATTERNS = ("random", "all_true", "all_false", "reset_t0", "reset_last", "chunk_bounds")


def make_masks(pattern, T, n, gen, chunks=4):
    """[T, n] bool, True = no reset.  random: 4 % resets, plus one in the last sequence at t = T - 2 when T >= 3 (so
    the reset perturbations apply); reset_t0: every sequence resets at t = 0; reset_last: every other sequence resets
    at t = T - 1; chunk_bounds: every sequence resets at the first step of each of `chunks` time chunks but the
    first"""
    m = torch.ones(T, n, dtype=torch.bool)
    if pattern == "random":
        m = torch.rand(T, n, generator=gen) > 0.04
        if T >= 3:
            m[T - 2, n - 1] = False
    elif pattern == "all_false":
        m[:] = False
    elif pattern == "reset_t0":
        m[0] = False
    elif pattern == "reset_last":
        m[T - 1, ::2] = False
    elif pattern == "chunk_bounds":
        for c in range(1, chunks):
            m[c * T // chunks] = False
    return m


def make_case(kind, T, n, H, masks="random", pre_scale=1.0, seed=0):
    """CPU float32 operands of one recurrence: xproj (times pre_scale: 30 saturates every gate), W_hh with orthonormal
    columns as the policies initialise it, b_hh, h0 in (-1, 1), c0, masks and dh_out"""
    gen = torch.Generator().manual_seed(seed)
    G = 4 if kind == "lstm" else 3
    rn = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    q, _ = torch.linalg.qr(rn(G * H, H))
    return dict(xproj=rn(T, n, G * H) * pre_scale, w_hh=q.contiguous(), b_hh=0.1 * rn(G * H), h0=torch.tanh(rn(n, H)),
                c0=rn(n, H), masks=make_masks(masks, T, n, gen), dh_out=rn(T, n, H))


FWD_KEYS = {"lstm": ("hs", "cs", "gates"), "gru": ("hs", "saved")}
BWD_KEYS = {"lstm": ("dgates",), "gru": ("dgx", "dgh")}


def err_ratio(got, ref, H):
    """max |got - ref| / (bar(H) * max |ref|): <= 1 passes"""
    scale = max(ref.abs().max().item(), 1e-30)
    return (got.double() - ref.double()).abs().max().item() / (bar(H) * scale)


def guard_ratios(kind, ops, ref, H):
    """{perturbation: how many bars its reference misses by (max over the outputs it is meant to change)} for every
    perturbation that changes the exact result of this case; ops are recurrence()'s operands"""
    out = {}
    bwd = "dh_out" in ops and ops["dh_out"] is not None
    names = (GRU_FWD_PERTURBATIONS if kind == "gru" else FWD_PERTURBATIONS) + \
        ((GRU_BWD_PERTURBATIONS if kind == "gru" else LSTM_BWD_PERTURBATIONS) if bwd else ())
    for p in names:
        keys = FWD_KEYS[kind] if p in GRU_FWD_PERTURBATIONS else BWD_KEYS[kind]
        pr = recurrence(kind, **ops, perturb=p)
        if pr is None or all(torch.equal(pr[k], ref[k]) for k in keys):
            continue
        out[p] = max(err_ratio(pr[k], ref[k], H) for k in keys)
    return out
