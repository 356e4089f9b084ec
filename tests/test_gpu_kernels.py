"""GPU parity tests, kernel by kernel, through the C ABI (libhb200.so) against the CPU oracle
(oracle/torch_oracle.py) or a plain fp32 torch restatement of the same op.

Tolerances (stated per test): GAE variant 1 is bit-exact; fp32 kernels 1e-5..1e-4; the tensor-core
convolutions are compared against an fp32 convolution of the SAME rounded operands (forward values fp16 = hf(),
gradients bf16 = bf()), so only accumulation order + the final rounding of the output differ (2^-11 rel for the
fp16 forward outputs, 2^-8 for the bf16 data gradients).
"""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

from oracle import torch_oracle as O  # noqa: E402  (checker only)

DEV = "cuda"


def bf(x):   # gradient storage type
    return x.to(torch.bfloat16)


def hf(x):   # forward-value storage type (activations, forward weight images)
    return x.to(torch.float16)


def nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


def nchw(x_nhwc):
    return x_nhwc.permute(0, 3, 1, 2).contiguous()


# ---------------------------------------------------------------------------------------------
# GAE / advantages
# ---------------------------------------------------------------------------------------------
def _rollout_scalars(T, N, seed, p_done=1 / 25):
    g = torch.Generator().manual_seed(seed)
    rewards = torch.randn(T + 1, N, 1, generator=g) * 0.1
    masks = torch.rand(T + 1, N, 1, generator=g) > p_done
    rewards = rewards + 2.5 * (~masks).float()
    values = torch.randn(T + 1, N, 1, generator=g)
    returns_stale = torch.randn(T + 1, N, 1, generator=g)
    next_value = torch.randn(N, 1, generator=g)
    return rewards, values, masks, returns_stale, next_value


@pytest.mark.parametrize("T,N,t_cur", [(128, 64, 128), (16, 8, 16), (128, 64, 37), (5, 3, 5), (1, 1, 1),
                                       (33, 129, 33), (128, 2048, 128)])
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("use_gae", [True, False])
def test_gae_adv(hb, T, N, t_cur, variant, use_gae):
    from habitat_lab_b200 import ops

    rewards, values, masks, stale, next_value = _rollout_scalars(T, N, 7 * T + N)
    v_ref = values.clone()
    ret_ref = O.compute_returns(rewards, v_ref, masks, next_value, t_cur, use_gae, 0.99, 0.95)
    # rows the reference does not write keep whatever the buffer held
    keep = torch.ones(T + 1, dtype=torch.bool)
    keep[: t_cur + (0 if use_gae else 1)] = False
    ret_full = torch.where(keep.view(-1, 1, 1), stale, ret_ref)
    adv_ref = O.get_advantages(ret_full, v_ref, normalize=False)

    d = lambda t: t.to(DEV).contiguous()  # noqa: E731
    r, v, m, nv = d(rewards), d(values), d(masks), d(next_value)
    ret = d(stale)
    adv = torch.empty_like(ret)
    stats = torch.zeros(4, dtype=torch.float64, device=DEV)
    ops.gae_adv(r, v, m, nv, ret, adv, stats, t_cur, 0.99, 0.95, use_gae, variant)
    torch.cuda.synchronize()
    if variant == 1 or not use_gae:
        assert torch.equal(ret.cpu(), ret_full), "serial GAE must be bit-exact with the reference order"
        assert torch.equal(adv.cpu(), adv_ref)
    else:
        torch.testing.assert_close(ret.cpu(), ret_full, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(adv.cpu(), adv_ref, rtol=1e-5, atol=2e-5)
    assert torch.equal(v.cpu(), v_ref)  # bootstrap row written like the reference
    # normalisation (single-process unbiased var_mean, ppo.py:151-157)
    adv_n_ref = O.get_advantages(ret_full, v_ref, normalize=True)
    ops.adv_normalize(adv, stats=stats)
    torch.testing.assert_close(adv.cpu(), adv_n_ref, rtol=1e-4, atol=1e-5)
    # distributed statistics path (ddppo.py:59-84) with explicit mean/var
    adv2 = d(adv_ref)
    var, mean = O.distributed_var_mean([adv_ref, adv_ref * 0.5 + 0.1])
    ops.adv_normalize(adv2, mean_var=torch.tensor([mean, var], device=DEV))
    torch.testing.assert_close(adv2.cpu(), O.get_advantages(ret_full, v_ref, True, (var, mean)), rtol=1e-5, atol=1e-6)


def test_gae_nonfinite_excluded_from_stats(hb):
    from habitat_lab_b200 import ops

    T, N = 8, 4
    rewards, values, masks, stale, next_value = _rollout_scalars(T, N, 3)
    stale[T, 1, 0] = float("inf")  # stale/bootstrap rows can be non-finite; ppo.py:146 filters them
    d = lambda t: t.to(DEV).contiguous()  # noqa: E731
    ret, adv = d(stale), torch.empty(T + 1, N, 1, device=DEV)
    stats = torch.zeros(4, dtype=torch.float64, device=DEV)
    ops.gae_adv(d(rewards), d(values), d(masks), d(next_value), ret, adv, stats, T, 0.99, 0.95, True, 1)
    assert stats[2].item() == (T + 1) * N - 1


# ---------------------------------------------------------------------------------------------
# heads + PPO loss
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,A", [(4096, 512, 4), (257, 512, 4), (64, 128, 6), (7, 32, 2)])
@pytest.mark.parametrize("use_clip_v", [True, False])
@pytest.mark.parametrize("perturb", [0.0, 0.5])
def test_ppo_loss(hb, B, H, A, use_clip_v, perturb):
    from habitat_lab_b200 import ops

    g = torch.Generator().manual_seed(B + H + A)
    feats = torch.randn(B, H, generator=g)
    w_act = torch.randn(A, H, generator=g) * (0.01 + perturb * 0.1)
    b_act = torch.randn(A, generator=g) * 0.1
    w_val = torch.randn(1, H, generator=g) * 0.05
    b_val = torch.randn(1, generator=g)
    actions = torch.randint(0, A, (B, 1), generator=g)
    with torch.no_grad():
        v0, lp0, _ = O.heads(feats, w_act, b_act, w_val, b_val, actions)
    batch = dict(
        action_log_probs=lp0 + perturb * torch.randn(B, 1, generator=g) * 0.3,
        advantages=torch.randn(B, 1, generator=g),
        value_preds=v0 + perturb * torch.randn(B, 1, generator=g),
        returns=v0 + torch.randn(B, 1, generator=g),
    )
    clip, c_v, c_e = 0.2, 0.5, 0.01
    req = [t.clone().requires_grad_(True) for t in (feats, w_act, b_act, w_val, b_val)]
    v, lp, ent = O.heads(*req, actions)
    ref = O.ppo_loss(v, lp, ent, batch, clip, c_v, c_e, use_clip_v)
    ref["total_loss"].backward()

    d = lambda t: t.to(DEV).contiguous()  # noqa: E731
    out = dict(values=torch.empty(B, device=DEV), log_probs=torch.empty(B, device=DEV),
               entropy=torch.empty(B, device=DEV), d_features=torch.empty(B, H, device=DEV),
               d_w_act=torch.empty(A, H, device=DEV), d_b_act=torch.empty(A, device=DEV),
               d_w_val=torch.empty(H, device=DEV), d_b_val=torch.empty(1, device=DEV),
               metrics=torch.empty(ops.N_METRICS, device=DEV))
    ws = ops.ppo_loss_workspace(B, H, A, DEV)
    ops.ppo_loss(d(feats), d(w_act), d(b_act), d(w_val), d(b_val), d(actions.view(-1)),
                 d(batch["action_log_probs"].view(-1)), d(batch["advantages"].view(-1)),
                 d(batch["value_preds"].view(-1)), d(batch["returns"].view(-1)), clip, c_v, c_e, use_clip_v, True,
                 out, ws)
    torch.cuda.synchronize()
    mt = out["metrics"].cpu()
    for i, k in enumerate(ops.METRIC_KEYS):
        torch.testing.assert_close(mt[i], ref[k].detach().float().reshape(()), rtol=2e-4, atol=2e-6, msg=lambda s, k=k: f"{k}: {s}")
    torch.testing.assert_close(out["values"].cpu(), v.detach().view(-1), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out["log_probs"].cpu(), lp.detach().view(-1), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out["entropy"].cpu(), ent.detach().view(-1), rtol=1e-4, atol=1e-5)
    gscale = max(1.0 / B, 1e-6)
    torch.testing.assert_close(out["d_features"].cpu(), req[0].grad, rtol=1e-3, atol=1e-3 * gscale)
    torch.testing.assert_close(out["d_w_act"].cpu(), req[1].grad, rtol=1e-3, atol=2e-5)
    torch.testing.assert_close(out["d_b_act"].cpu(), req[2].grad, rtol=1e-3, atol=2e-5)
    torch.testing.assert_close(out["d_w_val"].cpu(), req[3].grad.view(-1), rtol=1e-3, atol=2e-5)
    torch.testing.assert_close(out["d_b_val"].cpu(), req[4].grad, rtol=1e-3, atol=2e-5)


# ---------------------------------------------------------------------------------------------
# clip + Adam
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [8_481_125, 1003, 4])
@pytest.mark.parametrize("max_norm", [0.2, 1e9])
def test_clip_adam(hb, n, max_norm):
    from habitat_lab_b200 import ops

    g = torch.Generator().manual_seed(n)
    n_pad = (n + 3) // 4 * 4
    p0 = torch.randn(n, generator=g)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref_p], lr=2.5e-4, eps=1e-5)
    flat = torch.zeros(4, n_pad, device=DEV)  # params, grads, m, v share one allocation (16B aligned rows)
    flat[0, :n] = p0.to(DEV)
    ws = ops.clip_adam_workspace(n, DEV)
    gn = torch.zeros(1, device=DEV)
    for step in range(1, 4):
        grad = torch.randn(n, generator=g) * (0.01 * step)
        ref_p.grad = grad.clone()
        true_norm = grad.double().norm().item()
        ref_norm = torch.nn.utils.clip_grad_norm_([ref_p], max_norm)
        opt.step()
        flat[1, :n] = grad.to(DEV)
        ops.clip_adam(flat[0, :n], flat[1, :n], flat[2, :n], flat[3, :n], 2.5e-4, (0.9, 0.999), 1e-5, 0.0,
                      max_norm, 1.0, step, gn, ws)
        torch.cuda.synchronize()
        # torch's fp32 CPU norm of 8.5M elements is itself off by ~3e-4 relative; the kernel
        # accumulates in fp64 and must match the exact norm tightly, the reference loosely
        assert gn.item() == pytest.approx(true_norm, rel=1e-5)
        torch.testing.assert_close(gn.cpu()[0], ref_norm, rtol=1e-3, atol=1e-7)
        torch.testing.assert_close(flat[0, :n].cpu(), ref_p.detach(), rtol=1e-5, atol=2e-7)
    st = opt.state[ref_p]
    # with clipping active the moments inherit the reference's ~3e-4 fp32 norm error (see above)
    torch.testing.assert_close(flat[2, :n].cpu(), st["exp_avg"], rtol=1e-3, atol=1e-8)
    torch.testing.assert_close(flat[3, :n].cpu(), st["exp_avg_sq"], rtol=2e-3, atol=1e-10)


def test_ppo_loss_importance_coefficients(hb):
    """VER's importance-sampling weights (rl/ppo/ppo.py:226-232: every per-frame loss term is weighted by
    is_coeffs.clamp(max=1) before the mean) through the fused loss kernel, forward and backward."""
    from habitat_lab_b200 import ops

    B, H, A = 1000, 512, 4
    g = torch.Generator().manual_seed(9)
    feats = torch.randn(B, H, generator=g)
    w_act, b_act = torch.randn(A, H, generator=g) * 0.05, torch.randn(A, generator=g) * 0.1
    w_val, b_val = torch.randn(1, H, generator=g) * 0.05, torch.randn(1, generator=g)
    actions = torch.randint(0, A, (B, 1), generator=g)
    with torch.no_grad():
        v0, lp0, _ = O.heads(feats, w_act, b_act, w_val, b_val, actions)
    batch = dict(action_log_probs=lp0 + 0.1 * torch.randn(B, 1, generator=g), advantages=torch.randn(B, 1, generator=g),
                 value_preds=v0 + 0.3 * torch.randn(B, 1, generator=g), returns=v0 + torch.randn(B, 1, generator=g),
                 is_coeffs=torch.rand(B, 1, generator=g) * 1.6)   # ~40 % above 1: the clamp matters
    req = [t.clone().requires_grad_(True) for t in (feats, w_act, b_act, w_val, b_val)]
    v, lp, ent = O.heads(*req, actions)
    ref = O.ppo_loss(v, lp, ent, batch, 0.2, 0.5, 0.01, True)
    ref["total_loss"].backward()
    d = lambda t: t.to(DEV).contiguous()  # noqa: E731
    out = dict(values=torch.empty(B, device=DEV), log_probs=torch.empty(B, device=DEV), entropy=torch.empty(B, device=DEV),
               d_features=torch.empty(B, H, device=DEV), d_w_act=torch.empty(A, H, device=DEV),
               d_b_act=torch.empty(A, device=DEV), d_w_val=torch.empty(H, device=DEV), d_b_val=torch.empty(1, device=DEV),
               metrics=torch.empty(ops.N_METRICS, device=DEV))
    ops.ppo_loss(d(feats), d(w_act), d(b_act), d(w_val), d(b_val), d(actions.view(-1)), d(batch["action_log_probs"].view(-1)),
                 d(batch["advantages"].view(-1)), d(batch["value_preds"].view(-1)), d(batch["returns"].view(-1)), 0.2, 0.5,
                 0.01, True, True, out, ops.ppo_loss_workspace(B, H, A, DEV), is_coeffs=d(batch["is_coeffs"].view(-1)))
    torch.cuda.synchronize()
    mt = out["metrics"].cpu()
    for i, k in enumerate(("value_loss", "action_loss", "dist_entropy")):
        torch.testing.assert_close(mt[i], ref[k].float().reshape(()), rtol=2e-4, atol=2e-6, msg=lambda s, k=k: f"{k}: {s}")
    torch.testing.assert_close(mt[10], ref["total_loss"].detach().float().reshape(()), rtol=2e-4, atol=2e-6)
    torch.testing.assert_close(out["d_features"].cpu(), req[0].grad, rtol=1e-3, atol=1e-3 / B)
    torch.testing.assert_close(out["d_w_act"].cpu(), req[1].grad, rtol=1e-3, atol=1e-5)
    torch.testing.assert_close(out["d_w_val"].cpu().view(1, -1), req[3].grad, rtol=1e-3, atol=1e-5)
    # an action outside [0, A) poisons the loss instead of silently scoring log_prob = 0
    bad = d(actions.view(-1)).clone()
    bad[3] = A
    ops.ppo_loss(d(feats), d(w_act), d(b_act), d(w_val), d(b_val), bad, d(batch["action_log_probs"].view(-1)),
                 d(batch["advantages"].view(-1)), d(batch["value_preds"].view(-1)), d(batch["returns"].view(-1)), 0.2, 0.5,
                 0.01, True, True, out, ops.ppo_loss_workspace(B, H, A, DEV))
    torch.cuda.synchronize()
    assert torch.isnan(out["metrics"][1]).item()


# ---------------------------------------------------------------------------------------------
# wgmma descriptor probe + convolutions
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", [0, 2])
def test_umma_probe(hb, layout):
    from habitat_lab_b200 import ops

    m, n, k = 256, 64, 192
    a = bf(torch.randn(m, k, device=DEV))
    b = bf(torch.randn(n, k, device=DEV))
    d = torch.zeros(m, n, device=DEV)
    if layout == 2:
        ops.umma_gemm_probe(a.t().contiguous(), b.t().contiguous(), d, m, n, k, 2)
    else:
        ops.umma_gemm_probe(a, b, d, m, n, k, layout)
    torch.cuda.synchronize()
    torch.testing.assert_close(d, a.float() @ b.float().t(), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("layout", [0, 1, 2])
@pytest.mark.parametrize("a_f16,b_f16", [(True, True)])
def test_umma_probe_operand_formats(hb, layout, a_f16, b_f16):
    """fp16 x fp16 operands (the forward convolutions; gradients use bf16 x bf16, test_umma_probe).  Values carry > 8
    significant bits so a wrong operand type (fp16 bits read as bf16) cannot pass.  The tensor core has no MIXED
    fp16 x bf16 form -- the reason the weight-gradient kernels read a bf16 twin of the activations."""
    from habitat_lab_b200 import ops

    m, n, k = 256, 64, 192
    torch.manual_seed(layout * 4 + a_f16 * 2 + b_f16)
    a32, b32 = torch.randn(m, k, device=DEV), torch.randn(n, k, device=DEV)
    a = a32.half() if a_f16 else a32.bfloat16()
    b = b32.half() if b_f16 else b32.bfloat16()
    d = torch.zeros(m, n, device=DEV)
    flags = layout | (16 if a_f16 else 0) | (32 if b_f16 else 0)
    if layout == 2:
        ops.umma_gemm_probe(a.t().contiguous(), b.t().contiguous(), d, m, n, k, flags)
    else:
        ops.umma_gemm_probe(a, b, d, m, n, k, flags)
    torch.cuda.synchronize()
    torch.testing.assert_close(d, a.float() @ b.float().t(), rtol=1e-4, atol=1e-3)


CONV_CASES = [
    # B, H, W, Ci_real, Ci_pad, Co, k, stride, pad
    (2, 32, 32, 32, 32, 32, 3, 1, 1),     # layer1
    (3, 32, 32, 32, 32, 64, 3, 2, 1),     # layer2.0 conv a
    (3, 32, 32, 32, 32, 64, 1, 2, 0),     # layer2.0 downsample
    (2, 16, 16, 64, 64, 64, 3, 1, 1),
    (2, 8, 8, 128, 128, 128, 3, 1, 1),
    (4, 4, 4, 256, 256, 256, 3, 1, 1),    # layer4 (two frames per warp in the stats epilogue)
    (4, 4, 4, 256, 256, 128, 3, 1, 1),    # compression
    (2, 64, 64, 4, 8, 32, 7, 2, 3),       # stem, 4 real channels padded to 8
    (1, 31, 17, 32, 32, 32, 3, 1, 1),     # odd sizes, ragged tile tail
    (9, 8, 8, 64, 64, 128, 3, 2, 1),
    (2, 128, 128, 1, 8, 32, 8, 4, 0),     # SimpleCNN conv 1 (depth only), simple_cnn.py:84-96
    (2, 31, 31, 32, 32, 64, 4, 2, 0),     # SimpleCNN conv 2 (odd input, last row/col unused)
    (2, 14, 14, 64, 64, 32, 3, 1, 0),     # SimpleCNN conv 3 (no padding)
    # the cases above have < 132 row tiles: the gather kernel slices the packed N tile (32-wide CTAs, the actor's
    # launch shape); these two keep the full-width tiles of the learner's 4096-frame minibatches covered
    (1200, 4, 4, 256, 256, 256, 3, 1, 1),
    (300, 8, 8, 64, 64, 128, 3, 2, 1),
    (64, 4, 4, 256, 256, 256, 3, 1, 1),   # the actor's layer4 launch: 8 row tiles x 8 slices of 32 channels
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fwd_dgrad_wgrad(hb, case):
    from habitat_lab_b200 import ops

    B, H, W, ci_real, ci, co, k, stride, pad = case
    torch.manual_seed(sum(case))
    x = torch.randn(B, ci_real, H, W, device=DEV)
    w = torch.randn(co, ci_real, k, k, device=DEV) * (1.0 / math.sqrt(ci_real * k * k))
    xb, wb, wh_ = hf(x).float(), bf(w).float(), hf(w).float()   # forward: fp16 x fp16; dgrad image: bf16
    y_ref = F.conv2d(xb, wh_, stride=stride, padding=pad)
    s = ops.conv_shape(B, H, W, ci, co, k, k, stride, pad)
    x_nhwc = torch.zeros(B, H, W, ci, device=DEV, dtype=torch.float16)
    x_nhwc[..., :ci_real] = hf(nhwc(x))
    wp, wt = ops.pack_conv_weight(w, ci, want_t=ci >= 32)
    y = torch.empty(B, s.ho, s.wo, co, device=DEV, dtype=torch.float16)
    groups = 16 if co % 16 == 0 and co // 16 >= 2 else 1
    stats = torch.zeros(B, groups, 2, device=DEV, dtype=torch.float64)
    ops.conv_fwd(x_nhwc, wp, y, s, stats, groups)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(y.float()), y_ref, rtol=2e-3, atol=2e-3)
    # fused GroupNorm statistics: sum / sum of squares per (frame, group) of the fp32 accumulators
    yg = y_ref.view(B, groups, -1)
    torch.testing.assert_close(stats[..., 0].float(), yg.sum(-1), rtol=1e-3, atol=2e-2)
    torch.testing.assert_close(stats[..., 1].float(), (yg * yg).sum(-1), rtol=1e-3, atol=2e-2)

    dy = torch.randn_like(y_ref)
    dyb = bf(dy).float()
    dy_nhwc = bf(nhwc(dy))
    # weight gradient: bf16 twin of x (the forward kernels write it next to the fp16 activation) x bf16 dy
    dw_ref = torch.nn.grad.conv2d_weight(bf(x).float(), w.shape, dyb, stride=stride, padding=pad)
    x_nhwc_b = torch.zeros(B, H, W, ci, device=DEV, dtype=torch.bfloat16)
    x_nhwc_b[..., :ci_real] = bf(nhwc(x))
    acc = torch.zeros(k * k * ci, co, device=DEV)
    ops.conv_wgrad(x_nhwc_b, dy_nhwc, acc, s)
    dw = torch.empty_like(w)
    ops.unpack_conv_wgrad(acc, dw, ci)
    torch.cuda.synchronize()
    torch.testing.assert_close(dw, dw_ref, rtol=2e-3, atol=2e-3 * dw_ref.abs().max().item())
    # data gradient (+ fused residual-gradient add)
    if ci >= 32:
        dx_ref = torch.nn.grad.conv2d_input(xb.shape, wb, dyb, stride=stride, padding=pad)
        addend = bf(torch.randn(B, H, W, ci, device=DEV))
        dx = torch.empty(B, H, W, ci, device=DEV, dtype=torch.bfloat16)
        ops.conv_dgrad(dy_nhwc, wt, dx, s, addend=None)
        torch.cuda.synchronize()
        torch.testing.assert_close(nchw(dx.float()), dx_ref, rtol=1e-2, atol=1e-2 * max(1.0, dx_ref.abs().max().item()))
        ops.conv_dgrad(dy_nhwc, wt, dx, s, addend=addend)
        torch.cuda.synchronize()
        torch.testing.assert_close(nchw(dx.float()), dx_ref + nchw(addend.float()), rtol=1e-2,
                                   atol=2e-2 * max(1.0, dx_ref.abs().max().item()))


@pytest.fixture(params=[1, 0], ids=["ws_swizzled", "slabs"])
def s2_variant(hb, request):
    """forward / dgrad of the stride-2 block entry: warp-specialised swizzled pixel-row copies (default) or 16-byte slabs"""
    lib = hb.load()
    prev = lib.hb200_get_conv_s2_ws()
    lib.hb200_set_conv_s2_ws(request.param)
    yield request.param
    lib.hb200_set_conv_s2_ws(prev)


@pytest.mark.parametrize("B,H,W", [(3, 32, 32), (2, 64, 16), (160, 32, 32)])
def test_conv_s2_block_entry(hb, s2_variant, B, H, W):
    """conv_s2.cu: 3x3 stride-2 conv + 1x1 stride-2 downsample conv of one input in one launch (forward with both
    GroupNorm sums, and the summed data gradient) over the TMA space-to-depth view, vs torch convolutions."""
    from habitat_lab_b200 import ops

    C, NA, NB, G = 32, 64, 64, 16
    assert ops.conv_s2_supported(C, NA, NB, H, W)
    torch.manual_seed(B + H + W)
    x = torch.randn(B, C, H, W, device=DEV)
    wa = torch.randn(NA, C, 3, 3, device=DEV) / math.sqrt(9 * C)
    wd = torch.randn(NB, C, 1, 1, device=DEV) / math.sqrt(C)
    wcat = torch.zeros(NA + NB, C, 3, 3, device=DEV)
    wcat[:NA] = wa
    wcat[NA:, :, 1, 1] = wd[:, :, 0, 0]
    img = torch.empty(9 * C * (NA + NB), device=DEV, dtype=torch.float16)
    img_t = torch.empty(9 * C * (NA + NB), device=DEV, dtype=torch.bfloat16)
    ops.pack_halo_weight(wcat, img, C, NA + NB, 3, 0)
    ops.pack_halo_weight(wcat, img_t, NA + NB, C, 3, 1)
    x_nhwc = hf(nhwc(x))
    ya = torch.empty(B, H // 2, W // 2, NA, device=DEV, dtype=torch.float16)
    yb = torch.empty(B, H // 2, W // 2, NB, device=DEV, dtype=torch.float16)
    sa = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
    sb = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
    ops.conv_s2_fwd(x_nhwc, img, ya, yb, B, H, W, C, NA, NB, stats_a=sa, groups_a=G, stats_b=sb, groups_b=G)
    torch.cuda.synchronize()
    xh = hf(x).float()
    ya_ref = F.conv2d(xh, hf(wa).float(), stride=2, padding=1)
    yb_ref = F.conv2d(xh, hf(wd).float(), stride=2)
    torch.testing.assert_close(nchw(ya.float()), ya_ref, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(nchw(yb.float()), yb_ref, rtol=2e-3, atol=2e-3)
    for st, ref in ((sa, ya_ref), (sb, yb_ref)):
        yg = ref.reshape(B, G, -1)
        torch.testing.assert_close(st[..., 0].float(), yg.sum(-1), rtol=1e-3, atol=2e-2)
        torch.testing.assert_close(st[..., 1].float(), (yg * yg).sum(-1), rtol=1e-3, atol=2e-2)
    # data gradient of both branches, summed (+ optional addend)
    dya = torch.randn_like(ya_ref)
    dyb = torch.randn_like(yb_ref)
    dx_ref = (torch.nn.grad.conv2d_input(x.shape, bf(wa).float(), bf(dya).float(), stride=2, padding=1) +
              torch.nn.grad.conv2d_input(x.shape, bf(wd).float(), bf(dyb).float(), stride=2))
    dx = torch.empty(B, H, W, C, device=DEV, dtype=torch.bfloat16)
    ops.conv_s2_dgrad(bf(nhwc(dya)), bf(nhwc(dyb)), img_t, dx, B, H, W, C, NA, NB)
    torch.cuda.synchronize()
    tol = 1e-2 * max(1.0, dx_ref.abs().max().item())
    torch.testing.assert_close(nchw(dx.float()), dx_ref, rtol=1e-2, atol=tol)
    addend = bf(torch.randn(B, H, W, C, device=DEV))
    ops.conv_s2_dgrad(bf(nhwc(dya)), bf(nhwc(dyb)), img_t, dx, B, H, W, C, NA, NB, addend=addend)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(dx.float()), dx_ref + nchw(addend.float()), rtol=1e-2, atol=2 * tol)
    # weight gradient of the 3x3 branch over the same view (x halo by one 5-D TMA box per tile)
    assert ops.conv_s2_wgrad_supported(C, NA, H, W)
    acc = torch.zeros(16 * C, NA, device=DEV)
    ops.conv_s2_wgrad(bf(nhwc(x)), bf(nhwc(dya)), acc, B, H, W, C, NA)
    dw = torch.empty_like(wa)
    ops.unpack_s2_wgrad(acc, dw)
    torch.cuda.synchronize()
    dw_ref = torch.nn.grad.conv2d_weight(bf(x).float(), wa.shape, bf(dya).float(), stride=2, padding=1)
    torch.testing.assert_close(dw, dw_ref, rtol=2e-3, atol=2e-3 * dw_ref.abs().max().item())
    # the 7 structurally-zero sub-taps of the 2x2 x 2x2 accumulator are never unpacked; the 9 real ones cover dw


HALO_CASES = [(3, 32, 32, 32, 32), (2, 16, 16, 64, 64), (5, 16, 8, 32, 32), (600, 32, 32, 32, 32)]


@pytest.fixture(params=[1, 0, 2, 3, 4, 5],
                ids=["default", "cp_async", "tma_swizzled", "tma_warp_specialised", "tma_ws_swizzled", "tma_slabs"])
def halo_loader(hb, request):
    """the halo load paths of the forward / dgrad halo kernels: the per-layer default, the cp.async gather, TMA copies of
    whole pixel rows into the swizzled K-major layout (three pre-shifted copies per tile), the warp-specialised pipeline
    (slabs / swizzled rows) and plain TMA box copies of 16-byte channel slabs"""
    lib = hb.load()
    prev = lib.hb200_get_halo_tma()
    lib.hb200_set_halo_tma(request.param)
    yield request.param
    lib.hb200_set_halo_tma(prev)


@pytest.fixture(params=[0, 1], ids=["x_regs", "x_tma"])
def wgrad_x(hb, request):
    """x halo of the halo weight-gradient kernels: register staging / cp.async, or one 5-D TMA box per tile"""
    lib = hb.load()
    prev = lib.hb200_get_wgrad_xtma()
    lib.hb200_set_wgrad_xtma(request.param)
    yield request.param
    lib.hb200_set_wgrad_xtma(prev)


@pytest.mark.parametrize("B,H,W,C,N", HALO_CASES)
def test_conv_halo_3x3(hb, halo_loader, wgrad_x, B, H, W, C, N):
    """halo kernels (one input load per tile, taps by descriptor shift) vs fp32 conv of the same rounded operands"""
    from habitat_lab_b200 import ops

    assert ops.conv_halo_supported(C, N, 3, H, W)
    torch.manual_seed(B + H + C)
    x = torch.randn(B, C, H, W, device=DEV)
    w = torch.randn(N, C, 3, 3, device=DEV) / math.sqrt(9 * C)
    xb, wb = hf(x).float(), bf(w).float()
    y_ref = F.conv2d(xb, hf(w).float(), padding=1)
    x_nhwc = hf(nhwc(x))
    wh = torch.empty(9 * C * N, device=DEV, dtype=torch.float16)
    wht = torch.empty(9 * C * N, device=DEV, dtype=torch.bfloat16)
    ops.pack_halo_weight(w, wh, C, N, 3, 0)
    ops.pack_halo_weight(w, wht, N, C, 3, 1)
    y = torch.empty(B, H, W, N, device=DEV, dtype=torch.float16)
    G = 16
    stats = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
    ops.conv_halo(x_nhwc, wh, y, B, H, W, C, N, 3, 0, gn_stats=stats, gn_groups=G)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(y.float()), y_ref, rtol=2e-3, atol=2e-3)
    yg = y_ref.view(B, G, -1)
    torch.testing.assert_close(stats[..., 0].float(), yg.sum(-1), rtol=1e-3, atol=2e-2)
    torch.testing.assert_close(stats[..., 1].float(), (yg * yg).sum(-1), rtol=1e-3, atol=2e-2)
    dy = torch.randn_like(y_ref)
    dyb, dy_nhwc = bf(dy).float(), bf(nhwc(dy))
    dx_ref = torch.nn.grad.conv2d_input(xb.shape, wb, dyb, padding=1)
    addend = bf(torch.randn(B, H, W, C, device=DEV))
    dx = torch.empty(B, H, W, C, device=DEV, dtype=torch.bfloat16)
    ops.conv_halo(dy_nhwc, wht, dx, B, H, W, N, C, 3, 1, addend=addend)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(dx.float()), dx_ref + nchw(addend.float()), rtol=1e-2,
                               atol=2e-2 * max(1.0, dx_ref.abs().max().item()))
    dw_ref = torch.nn.grad.conv2d_weight(bf(x).float(), w.shape, dyb, padding=1)
    acc = torch.zeros(9 * C, N, device=DEV)
    ops.conv_halo_wgrad(bf(nhwc(x)), dy_nhwc, acc, B, H, W, C, N, 3)
    dw = torch.empty_like(w)
    ops.unpack_conv_wgrad(acc, dw, C)
    torch.cuda.synchronize()
    torch.testing.assert_close(dw, dw_ref, rtol=2e-3, atol=2e-3 * dw_ref.abs().max().item())


@pytest.mark.parametrize("B,HW,C,N", [(5, 8, 128, 128), (2, 8, 128, 128), (7, 4, 256, 256), (3, 4, 256, 128),
                                      (600, 8, 128, 128), (1, 4, 32, 128)])
def test_conv_halo_wgrad_small_images(hb, B, HW, C, N):
    """weight gradient of the 8x8 / 4x4 layers: tiles of 2 / 4 stacked images (own padding rows, virtual zero pixels for
    4x4), 32-channel x 128-column slices, vs fp32 conv2d_weight of the same rounded operands; odd B = ragged last tile"""
    from habitat_lab_b200 import ops

    assert ops.conv_halo_wgrad_supported(C, N, 3, HW, HW) and not ops.conv_halo_supported(C, N, 3, HW, HW)
    torch.manual_seed(B + HW + C)
    x = torch.randn(B, C, HW, HW, device=DEV)
    dy = torch.randn(B, N, HW, HW, device=DEV)
    xb, dyb = bf(x).float(), bf(dy).float()
    dw_ref = torch.nn.grad.conv2d_weight(xb, (N, C, 3, 3), dyb, padding=1)
    acc = torch.zeros(9 * C, N, device=DEV)
    ops.conv_halo_wgrad(bf(nhwc(x)), bf(nhwc(dy)), acc, B, HW, HW, C, N, 3)
    dw = torch.empty(N, C, 3, 3, device=DEV)
    ops.unpack_conv_wgrad(acc, dw, C)
    torch.cuda.synchronize()
    torch.testing.assert_close(dw, dw_ref, rtol=2e-3, atol=2e-3 * dw_ref.abs().max().item())
    # and it must agree with the gather kernel it replaces
    acc2 = torch.zeros(9 * C, N, device=DEV)
    ops.conv_wgrad(bf(nhwc(x)), bf(nhwc(dy)), acc2, ops.conv_shape(B, HW, HW, C, N, 3, 3, 1, 1))
    torch.cuda.synchronize()
    torch.testing.assert_close(acc, acc2, rtol=2e-3, atol=2e-3 * acc2.abs().max().item())


@pytest.mark.parametrize("B,Hp,Wp", [(2, 128, 128), (3, 64, 32)])
def test_conv_halo_stem_s2d(hb, halo_loader, wgrad_x, B, Hp, Wp):
    """7x7 stride-2 pad-3 stem == 4x4 stride-1 conv over the space-to-depth input"""
    from habitat_lab_b200 import ops

    torch.manual_seed(Hp)
    x = torch.randn(B, 4, Hp, Wp, device=DEV)
    w = torch.randn(32, 4, 7, 7, device=DEV) / math.sqrt(196)
    xb, wb = hf(x).float(), hf(w).float()
    y_ref = F.conv2d(xb, wb, stride=2, padding=3)
    Ho, Wo = Hp // 2, Wp // 2
    # s2d: [B, Ho, Wo, (dy, dx, c)]
    xs = hf(x).view(B, 4, Ho, 2, Wo, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, Ho, Wo, 16).contiguous()
    wh = torch.empty(16 * 16 * 32, device=DEV, dtype=torch.float16)
    ops.pack_halo_weight(w, wh, 16, 32, 4, 2)
    y = torch.empty(B, Ho, Wo, 32, device=DEV, dtype=torch.float16)
    stats = torch.zeros(B, 16, 2, device=DEV, dtype=torch.float64)
    ops.conv_halo(xs, wh, y, B, Ho, Wo, 16, 32, 4, 0, gn_stats=stats, gn_groups=16)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(y.float()), y_ref, rtol=2e-3, atol=2e-3)
    dy = torch.randn_like(y_ref)
    dw_ref = torch.nn.grad.conv2d_weight(bf(x).float(), w.shape, bf(dy).float(), stride=2, padding=3)
    acc = torch.zeros(256, 32, device=DEV)
    xs_b = bf(x).view(B, 4, Ho, 2, Wo, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, Ho, Wo, 16).contiguous()   # bf16 twin
    ops.conv_halo_wgrad(xs_b, bf(nhwc(dy)), acc, B, Ho, Wo, 16, 32, 4)
    dw = torch.empty_like(w)
    ops.unpack_stem_wgrad(acc, dw)
    torch.cuda.synchronize()
    torch.testing.assert_close(dw, dw_ref, rtol=2e-3, atol=2e-3 * dw_ref.abs().max().item())


# ---------------------------------------------------------------------------------------------
# input prep + running mean/var
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("has_rgb,has_depth", [(True, True), (False, True), (True, False)])
def test_prep(hb, has_rgb, has_depth):
    from habitat_lab_b200 import ops

    rows, B, H, W = 12, 5, 32, 48
    g = torch.Generator().manual_seed(11)
    rgb = torch.randint(0, 256, (rows, H, W, 3), generator=g, dtype=torch.uint8)
    depth = torch.rand(rows, H, W, 1, generator=g)
    frame_rows = torch.tensor([3, 0, 11, 7, 7], dtype=torch.int32)
    C = (3 if has_rgb else 0) + (1 if has_depth else 0)
    obs, keys = {}, []
    if has_rgb:
        obs["rgb"] = rgb[frame_rows.long()]
        keys.append("rgb")
    if has_depth:
        obs["depth"] = depth[frame_rows.long()]
        keys.append("depth")
    xs = []
    for kname in keys:
        o = obs[kname].permute(0, 3, 1, 2)
        xs.append(o.float() * (1.0 / 255.0) if o.dtype == torch.uint8 else o)
    x = F.avg_pool2d(torch.cat(xs, 1), 2)
    mean, var, count = torch.rand(1, C, 1, 1), torch.rand(1, C, 1, 1) + 0.01, torch.tensor(7.0)
    m2, v2, c2 = O.running_mean_var_update(x, mean, var, count)
    ref = O.running_mean_var_apply(x, m2, v2)

    d = lambda t: t.to(DEV).contiguous()  # noqa: E731
    drgb = d(rgb) if has_rgb else None
    ddepth = d(depth) if has_depth else None
    stats = torch.zeros(17, dtype=torch.float64, device=DEV)
    rm, rv, rc = d(mean.view(-1)), d(var.view(-1)), d(count.view(1))
    ss = torch.zeros(16, device=DEV)
    out = torch.empty(B, H // 2, W // 2, 8, device=DEV, dtype=torch.float16)
    fr = d(frame_rows)
    ops.prep_stats(drgb, ddepth, fr, H, W, stats)
    ops.prep_finalize(stats, rm, rv, rc, ss, C, (H // 2) * (W // 2), True)
    out_b = torch.empty_like(out, dtype=torch.bfloat16)
    ops.prep_apply(drgb, ddepth, fr, H, W, ss, out, out_bf16=out_b)
    torch.cuda.synchronize()
    torch.testing.assert_close(out_b.float(), out.float(), rtol=8e-3, atol=1e-3)
    torch.testing.assert_close(rm.cpu(), m2.view(-1), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(rv.cpu(), v2.view(-1), rtol=1e-4, atol=1e-6)
    assert rc.item() == c2.item()
    got = nchw(out.float().cpu())
    torch.testing.assert_close(got[:, :C], ref, rtol=2e-3, atol=2e-3)  # fp16 output
    assert (got[:, C:] == 0).all()
    # space-to-depth form used by the halo stem: [B, H/4, W/4, (dy, dx, c4)]
    out2 = torch.empty(B, H // 4, W // 4, 16, device=DEV, dtype=torch.float16)
    ops.prep_apply(drgb, ddepth, fr, H, W, ss, out2, s2d=True)
    exp = out[..., :4].view(B, H // 4, 2, W // 4, 2, 4).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 4, W // 4, 16)
    assert torch.equal(out2, exp)


# ---------------------------------------------------------------------------------------------
# GroupNorm passes
# ---------------------------------------------------------------------------------------------
def _stats_of(y_nchw, groups):
    B = y_nchw.shape[0]
    yg = y_nchw.reshape(B, groups, -1)
    yg = yg.double()
    return torch.stack([yg.sum(-1), (yg * yg).sum(-1)], -1).contiguous()   # f64 [B,G,2] like the conv epilogue


@pytest.mark.parametrize("B,C,H,W,G", [(3, 32, 16, 16, 16), (2, 64, 8, 8, 16), (2, 128, 4, 4, 1), (5, 256, 4, 4, 16),
                                       (2, 32, 64, 64, 16), (3, 32, 32, 32, 16), (3, 64, 16, 16, 16),
                                       (2, 32, 31, 17, 16)])  # clusters of 8 / 4 / 2 CTAs per frame, ragged slice
def test_groupnorm_passes(hb, B, C, H, W, G):
    from habitat_lab_b200 import ops

    torch.manual_seed(C + H)
    y = hf(torch.randn(B, C, H, W, device=DEV) * 1.5 + 0.3).float()
    res = hf(torch.randn(B, C, H, W, device=DEV)).float()
    gamma = torch.rand(C, device=DEV) + 0.5
    beta = torch.randn(C, device=DEV) * 0.2
    stats = _stats_of(y, G)
    yb, resb = hf(nhwc(y)), hf(nhwc(res))
    hw = H * W
    # --- forward: GN + ReLU
    out = torch.empty_like(yb)
    out_b = torch.empty_like(yb, dtype=torch.bfloat16)
    ops.gn_apply(yb, stats, gamma, beta, out, B, hw, C, G, relu=True, out_bf16=out_b)
    torch.testing.assert_close(out_b.float(), out.float(), rtol=8e-3, atol=1e-3)   # bf16 twin of the same values
    yr = y.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    z = F.group_norm(yr, G, gr, br, eps=1e-5)
    a = F.relu(z)
    torch.testing.assert_close(nchw(out.float()), a.detach(), rtol=2e-3, atol=2e-3)
    outf = torch.empty(B, H, W, C, device=DEV)
    ops.gn_apply(yb, stats, gamma, beta, outf, B, hw, C, G, relu=True)
    torch.testing.assert_close(nchw(outf), a.detach(), rtol=1e-4, atol=1e-4)
    # --- backward through GN + ReLU (mask_mode 1)
    g = bf(torch.randn(B, C, H, W, device=DEV)).float()
    a.backward(g)
    sums = torch.zeros(B, G, 2, device=DEV)
    dga, dbe = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    gb = bf(nhwc(g))
    ops.gn_bwd_reduce(gb, None, yb, stats, gamma, beta, sums, dga, dbe, B, hw, C, G, 1)
    dy = torch.empty_like(gb)
    ops.gn_bwd_apply(gb, None, yb, stats, gamma, beta, sums, dy, None, B, hw, C, G, 1)
    torch.cuda.synchronize()
    sc = yr.grad.abs().max().item()
    torch.testing.assert_close(nchw(dy.float()), yr.grad, rtol=2e-2, atol=1e-2 * sc)
    # fused single-launch variant must reproduce the two-pass result
    dga2, dbe2, dy2 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.empty_like(gb)
    ops.gn_bwd(gb, None, yb, stats, gamma, beta, dga2, dbe2, dy2, None, B, hw, C, G, 1)
    torch.cuda.synchronize()
    torch.testing.assert_close(dy2.float(), dy.float(), rtol=1e-2, atol=1e-2 * sc)
    torch.testing.assert_close(dga2, dga, rtol=1e-4, atol=1e-4 * dga.abs().max().item())
    torch.testing.assert_close(dbe2, dbe, rtol=1e-4, atol=1e-4 * dbe.abs().max().item())
    torch.testing.assert_close(dga, gr.grad, rtol=1e-3, atol=1e-3 * gr.grad.abs().max().item())
    torch.testing.assert_close(dbe, br.grad, rtol=1e-3, atol=1e-3 * br.grad.abs().max().item())
    # --- residual block output: relu(GN(y) + res), backward with mask from the block output
    blk = torch.empty_like(yb)
    blk_b = torch.empty_like(yb, dtype=torch.bfloat16)
    ops.gn_residual_relu(yb, stats, gamma, beta, resb, blk, B, hw, C, G, out_bf16=blk_b)
    torch.testing.assert_close(blk_b.float(), blk.float(), rtol=8e-3, atol=1e-3)
    assert ((blk_b > 0) == (blk > 0))[blk_b.float().abs() > 1e-6].all()   # same ReLU decisions above fp16's underflow
    yr2 = y.clone().requires_grad_(True)
    rr2 = res.clone().requires_grad_(True)
    o2 = F.relu(F.group_norm(yr2, G, gamma, beta, eps=1e-5) + rr2)
    torch.testing.assert_close(nchw(blk.float()), o2.detach(), rtol=2e-3, atol=4e-3)
    o2.backward(g)
    sums.zero_(); dga.zero_(); dbe.zero_()
    gz = torch.empty_like(gb)
    # mask from the exact fp32 block output (rounded copies of tiny positives could flip the mask)
    act = hf(nhwc(o2.detach()))
    ops.gn_bwd_reduce(gb, act, yb, stats, gamma, beta, sums, dga, dbe, B, hw, C, G, 2)
    ops.gn_bwd_apply(gb, act, yb, stats, gamma, beta, sums, dy, gz, B, hw, C, G, 2)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(gz.float()), rr2.grad, rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(nchw(dy.float()), yr2.grad, rtol=2e-2, atol=1e-2 * yr2.grad.abs().max().item())
    dga2.zero_(); dbe2.zero_()
    gz2 = torch.empty_like(gb)
    ops.gn_bwd(gb, act, yb, stats, gamma, beta, dga2, dbe2, dy2, gz2, B, hw, C, G, 2)
    torch.cuda.synchronize()
    assert torch.equal(gz2, gz)
    torch.testing.assert_close(dy2.float(), dy.float(), rtol=1e-2, atol=1e-2 * yr2.grad.abs().max().item())
    torch.testing.assert_close(dga2, dga, rtol=1e-4, atol=1e-4 * dga.abs().max().item())
    torch.testing.assert_close(dbe2, dbe, rtol=1e-4, atol=1e-4 * dbe.abs().max().item())
    # mask_mode 0 (downsample branch: GroupNorm without ReLU)
    sums.zero_(); dga.zero_(); dbe.zero_(); dga2.zero_(); dbe2.zero_()
    ops.gn_bwd_reduce(gb, None, yb, stats, gamma, beta, sums, dga, dbe, B, hw, C, G, 0)
    ops.gn_bwd_apply(gb, None, yb, stats, gamma, beta, sums, dy, None, B, hw, C, G, 0)
    ops.gn_bwd(gb, None, yb, stats, gamma, beta, dga2, dbe2, dy2, None, B, hw, C, G, 0)
    torch.cuda.synchronize()
    torch.testing.assert_close(dy2.float(), dy.float(), rtol=1e-2, atol=1e-2 * dy.float().abs().max().item())
    torch.testing.assert_close(dga2, dga, rtol=1e-4, atol=1e-4 * dga.abs().max().item())
    # --- downsample variant: relu(GN(y) + GN_d(yd))
    gd, bd = torch.rand(C, device=DEV) + 0.5, torch.randn(C, device=DEV) * 0.1
    rstats = _stats_of(res, G)
    ops.gn_residual_relu(yb, stats, gamma, beta, resb, blk, B, hw, C, G, rstats, gd, bd)
    o3 = F.relu(F.group_norm(y, G, gamma, beta, eps=1e-5) + F.group_norm(res, G, gd, bd, eps=1e-5))
    torch.testing.assert_close(nchw(blk.float()), o3, rtol=2e-3, atol=6e-3)


@pytest.mark.parametrize("B,C,H,W,G", [(3, 32, 16, 24, 16), (2, 32, 64, 64, 16), (2, 64, 32, 32, 16)])
def test_gn_relu_maxpool(hb, B, C, H, W, G):
    from habitat_lab_b200 import ops

    torch.manual_seed(5)
    y = hf(torch.randn(B, C, H, W, device=DEV)).float()
    gamma, beta = torch.rand(C, device=DEV) + 0.5, torch.randn(C, device=DEV) * 0.2
    stats = _stats_of(y, G)
    yb = hf(nhwc(y))
    out = torch.empty(B, H // 2, W // 2, C, device=DEV, dtype=torch.float16)
    arg = torch.empty(B, H // 2, W // 2, C, device=DEV, dtype=torch.uint8)
    out_b = torch.empty_like(out, dtype=torch.bfloat16)
    ops.gn_relu_maxpool(yb, stats, gamma, beta, out, arg, B, H, W, C, G, out_bf16=out_b)
    torch.testing.assert_close(out_b.float(), out.float(), rtol=8e-3, atol=1e-3)
    yr = y.clone().requires_grad_(True)
    zr = F.relu(F.group_norm(yr, G, gamma, beta, eps=1e-5))
    zr.retain_grad()
    pr = F.max_pool2d(zr, 3, 2, 1)
    torch.testing.assert_close(nchw(out.float()), pr.detach(), rtol=2e-3, atol=2e-3)
    g = bf(torch.randn_like(pr)).float()
    pr.backward(g)
    dz = torch.empty(B, H, W, C, device=DEV, dtype=torch.bfloat16)
    ops.maxpool_bwd(bf(nhwc(g)), arg, dz, B, H, W, C)
    torch.cuda.synchronize()
    # compare only where the max is unique & positive (ties among zeros carry no gradient after ReLU)
    ref = zr.grad
    got = nchw(dz.float())
    mask = zr.detach() > 1e-3
    torch.testing.assert_close(got[mask], ref[mask], rtol=1e-2, atol=1e-2)
    # fused stem backward (pool + ReLU + GroupNorm backward in one cluster kernel) vs the two-kernel path and autograd
    hw = H * W
    dga, dbe, dy = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.empty_like(dz)
    ops.gn_bwd(dz, None, yb, stats, gamma, beta, dga, dbe, dy, None, B, hw, C, G, 1)
    assert ops.gn_relu_maxpool_bwd_supported(H, W, C, G)
    dga2, dbe2, dy2 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.empty_like(dz)
    ops.gn_relu_maxpool_bwd(bf(nhwc(g)), arg, yb, stats, gamma, beta, dga2, dbe2, dy2, B, H, W, C, G)
    torch.cuda.synchronize()
    sc = dy.float().abs().max().item()
    torch.testing.assert_close(dy2.float(), dy.float(), rtol=2e-2, atol=1e-2 * sc)
    torch.testing.assert_close(dga2, dga, rtol=1e-2, atol=1e-2 * dga.abs().max().item())
    torch.testing.assert_close(dbe2, dbe, rtol=1e-2, atol=1e-2 * dbe.abs().max().item())
    assert (nchw(dy2.float()) - yr.grad).norm().item() < 2e-2 * yr.grad.norm().item()


# ---------------------------------------------------------------------------------------------
# sgemm, LSTM recurrence, embeddings
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(4096, 512, 2048), (300, 70, 50), (128, 2048, 576), (5, 7, 3)])
def test_sgemm_linear(hb, M, N, K):
    from habitat_lab_b200 import ops

    torch.manual_seed(M + N + K)
    x = torch.randn(M, K, device=DEV)
    w = torch.randn(N, K, device=DEV) / math.sqrt(K)
    b = torch.randn(N, device=DEV)
    out = torch.empty(M, N + 8, device=DEV)  # ldc > N
    ops.linear_fwd(x, w, b, out, relu=True)
    ref = F.relu(F.linear(x.double(), w.double(), b.double())).float()
    torch.testing.assert_close(out[:, :N], ref, rtol=1e-4, atol=1e-4)
    dy = torch.randn(M, N, device=DEV)
    dx = torch.empty(M, K, device=DEV)
    ops.linear_bwd_input(dy, w, dx)
    torch.testing.assert_close(dx, (dy.double() @ w.double()).float(), rtol=1e-4, atol=1e-4)
    dw = torch.empty(N, K, device=DEV)
    ops.linear_bwd_weight(dy, x, dw)
    ref_dw = (dy.double().t() @ x.double()).float()
    torch.testing.assert_close(dw, ref_dw, rtol=1e-4, atol=1e-4 * max(1.0, ref_dw.abs().max().item()))
    db = torch.empty(N, device=DEV)
    ops.colsum(dy, db)
    torch.testing.assert_close(db, dy.sum(0), rtol=1e-4, atol=1e-3)


@pytest.fixture(params=[1, 0], ids=["tma", "cp_async"])
def tgemm_feed(hb, request):
    """both operand feeds of hb200_tgemm: TMA box loads (default) and the 16-byte cp.async gather"""
    lib = hb.load()
    prev = lib.hb200_get_tgemm_tma()
    lib.hb200_set_tgemm_tma(request.param)
    yield request.param
    lib.hb200_set_tgemm_tma(prev)


@pytest.mark.parametrize("M,N,K", [(4096, 512, 2048), (4096, 2048, 576), (128, 64, 64), (260, 36, 100),
                                   # one row tile (the actor's batches): deterministic split-K through the workspace
                                   (64, 512, 2048), (64, 2048, 576), (64, 2048, 512), (3, 36, 260), (128, 512, 4096)])
def test_tgemm_tf32(hb, tgemm_feed, M, N, K):
    """wgmma tf32 dense layers: forward (K-major x K-major), data gradient (K-major x N-major) and
    split-K weight gradient (M-major x N-major) vs fp64; tolerance = TF32 operand rounding (2^-11 relative)."""
    from habitat_lab_b200 import ops

    torch.manual_seed(M + N + K)
    x = torch.randn(M, K, device=DEV)
    w = torch.randn(N, K, device=DEV) / math.sqrt(K)
    b = torch.randn(N, device=DEV)
    out = torch.empty(M, N + 8, device=DEV)
    ops.linear_fwd(x, w, b, out, relu=True, tf32=True)
    ref = F.relu(F.linear(x.double(), w.double(), b.double())).float()
    torch.testing.assert_close(out[:, :N], ref, rtol=2e-3, atol=4e-3)
    dy = torch.randn(M, N, device=DEV)
    dx = torch.empty(M, K, device=DEV)
    ops.linear_bwd_input(dy, w, dx, tf32=True)
    ref_dx = (dy.double() @ w.double()).float()
    torch.testing.assert_close(dx, ref_dx, rtol=2e-3, atol=4e-3 * ref_dx.abs().max().item())
    dw = torch.zeros(N, K, device=DEV)
    ops.linear_bwd_weight(dy, x, dw, accumulate=True, tf32=True)
    ref_dw = (dy.double().t() @ x.double()).float()
    torch.testing.assert_close(dw, ref_dw, rtol=2e-3, atol=2e-3 * ref_dw.abs().max().item())


@pytest.mark.parametrize("T,n,H,D", [(16, 8, 512, 576), (7, 3, 32, 32), (33, 33, 128, 64), (9, 35, 512, 64)])
def test_lstm_masked_recurrence(hb, T, n, H, D):
    """The logic of test/test_rnn_state_encoder.py:72-94: flat (T*N) batch + masks must equal the
    step-by-step loop h = where(mask, h, 0); rnn(x_t, h), norm of the difference < 1e-3."""
    from habitat_lab_b200 import ops

    torch.manual_seed(T * n + H)
    lstm = torch.nn.LSTM(D, H, num_layers=1)
    for name, p in lstm.named_parameters():
        if "weight" in name:
            torch.nn.init.orthogonal_(p)
        else:
            torch.nn.init.normal_(p, std=0.1)
    sd = {"rnn." + k: v.detach() for k, v in lstm.state_dict().items()}
    x = torch.randn(T * n, D)
    masks = torch.rand(T * n, 1) > (1 / 25)
    hidden = torch.randn(n, 2, H)
    xr = x.clone().requires_grad_(True)
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    out_ref, hid_ref = O.rnn_seq_forward(xr, hidden, masks, sdr, "rnn.", "LSTM", 1, n)
    gout = torch.randn(T * n, H)
    (out_ref * gout).sum().backward()

    d = lambda t: t.to(DEV).contiguous()  # noqa: E731
    w_ih, w_hh = d(sd["rnn.weight_ih_l0"]), d(sd["rnn.weight_hh_l0"])
    bias = d(sd["rnn.bias_ih_l0"] + sd["rnn.bias_hh_l0"])
    xd, md = d(x), d(masks.view(-1)).view(torch.uint8)
    xproj = torch.empty(T * n, 4 * H, device=DEV)
    ops.linear_fwd(xd, w_ih, bias, xproj)
    h0, c0 = d(hidden[:, 0]), d(hidden[:, 1])
    hs = torch.empty(T, n, H, device=DEV)
    cs = torch.empty(T, n, H, device=DEV)
    gates = torch.empty(T, n, 4 * H, device=DEV)
    for t in range(T):
        ops.lstm_step_fwd(xproj[t * n:(t + 1) * n], w_hh, md[t * n:(t + 1) * n], h0 if t == 0 else hs[t - 1],
                          c0 if t == 0 else cs[t - 1], hs[t], cs[t], gates[t], n, H)
    torch.cuda.synchronize()
    diff = (hs.view(T * n, H).cpu() - out_ref.detach()).norm().item()
    assert diff < 1e-3, diff
    torch.testing.assert_close(hs[-1].cpu(), hid_ref[:, 0].detach(), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(cs[-1].cpu(), hid_ref[:, 1].detach(), rtol=1e-4, atol=1e-5)
    # persistent whole-sequence kernel (different reduction tree) must agree with the per-step kernel
    ws = torch.zeros(64, dtype=torch.uint8, device=DEV)
    hs2, cs2, gates2 = torch.empty_like(hs), torch.empty_like(cs), torch.empty_like(gates)
    ops.lstm_seq_fwd(xproj, w_hh, None, md, h0, c0, hs2, cs2, gates2, T, n, H, ws)
    torch.cuda.synchronize()
    for a_, b_ in ((hs2, hs), (cs2, cs), (gates2, gates)):
        torch.testing.assert_close(a_, b_, rtol=1e-5, atol=1e-6)
    dg2 = torch.empty(T, n, 4 * H, device=DEV)
    ops.lstm_seq_bwd(d(gout).view(T, n, H), gates, cs, c0, w_hh, md, dg2, T, n, H, ws)
    # backward through time
    dg = torch.empty(T, n, 4 * H, device=DEV)
    dh = [torch.zeros(n, H, device=DEV) for _ in range(2)]
    dc = [torch.zeros(n, H, device=DEV) for _ in range(2)]
    gd = d(gout).view(T, n, H)
    for t in reversed(range(T)):
        last = t == T - 1
        ops.lstm_step_bwd(gd[t], None if last else dh[(t + 1) % 2], None if last else dc[(t + 1) % 2], gates[t],
                          cs[t], c0 if t == 0 else cs[t - 1], w_hh, md[t * n:(t + 1) * n], dg[t], dh[t % 2],
                          dc[t % 2], n, H)
    torch.cuda.synchronize()
    torch.testing.assert_close(dg2, dg, rtol=1e-4, atol=1e-6)
    dgf = dg.view(T * n, 4 * H)
    dx = torch.empty(T * n, D, device=DEV)
    ops.linear_bwd_input(dgf, w_ih, dx)
    dw_ih = torch.empty_like(w_ih)
    ops.linear_bwd_weight(dgf, xd, dw_ih)
    hin = torch.empty(T, n, H, device=DEV)
    ops.rnn_shift_mask(hs, h0, md, hin, T, n, H)
    dw_hh = torch.empty_like(w_hh)
    ops.linear_bwd_weight(dgf, hin.view(T * n, H), dw_hh)
    db = torch.empty(4 * H, device=DEV)
    ops.colsum(dgf, db)
    torch.cuda.synchronize()
    tol = dict(rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(dx.cpu(), xr.grad, **tol)
    torch.testing.assert_close(dw_ih.cpu(), sdr["rnn.weight_ih_l0"].grad, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(dw_hh.cpu(), sdr["rnn.weight_hh_l0"].grad, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(db.cpu(), sdr["rnn.bias_ih_l0"].grad, rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("T,n,H,D", [(16, 8, 512, 514), (9, 3, 32, 16)])
def test_gru_masked_recurrence(hb, T, n, H, D):
    """persistent GRU kernels vs the masked step loop of the oracle (same contract as the LSTM test)"""
    from habitat_lab_b200 import ops

    torch.manual_seed(T + H)
    gru = torch.nn.GRU(D, H, num_layers=1)
    for name, p in gru.named_parameters():
        torch.nn.init.orthogonal_(p) if "weight" in name else torch.nn.init.normal_(p, std=0.1)
    sd = {"rnn." + k: v.detach() for k, v in gru.state_dict().items()}
    x = torch.randn(T * n, D)
    masks = torch.rand(T * n, 1) > (1 / 25)
    hidden = torch.randn(n, 1, H)
    xr = x.clone().requires_grad_(True)
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    out_ref, hid_ref = O.rnn_seq_forward(xr, hidden, masks, sdr, "rnn.", "GRU", 1, n)
    gout = torch.randn(T * n, H)
    (out_ref * gout).sum().backward()
    d = lambda t: t.to(DEV).contiguous()  # noqa: E731
    w_ih, w_hh, b_ih, b_hh = (d(sd["rnn." + k]) for k in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"))
    xd, md = d(x), d(masks.view(-1)).view(torch.uint8)
    xproj = torch.empty(T * n, 3 * H, device=DEV)
    ops.linear_fwd(xd, w_ih, b_ih, xproj)
    h0 = d(hidden[:, 0])
    hs, saved = torch.empty(T, n, H, device=DEV), torch.empty(T, n, 4 * H, device=DEV)
    ws = torch.zeros(64, dtype=torch.uint8, device=DEV)
    ops.gru_seq_fwd(xproj, w_hh, b_hh, md, h0, hs, saved, T, n, H, ws)
    torch.cuda.synchronize()
    assert (hs.view(T * n, H).cpu() - out_ref.detach()).norm().item() < 1e-3
    dgx, dgh = torch.empty(T, n, 3 * H, device=DEV), torch.empty(T, n, 3 * H, device=DEV)
    ops.gru_seq_bwd(d(gout).view(T, n, H), saved, hs, h0, w_hh, md, dgx, dgh, T, n, H, ws)
    dgxf, dghf = dgx.view(T * n, 3 * H), dgh.view(T * n, 3 * H)
    dx = torch.empty(T * n, D, device=DEV)
    ops.linear_bwd_input(dgxf, w_ih, dx)
    dw_ih, dw_hh = torch.empty_like(w_ih), torch.empty_like(w_hh)
    ops.linear_bwd_weight(dgxf, xd, dw_ih)
    hin = torch.empty(T, n, H, device=DEV)
    ops.rnn_shift_mask(hs, h0, md, hin, T, n, H)
    ops.linear_bwd_weight(dghf, hin.view(T * n, H), dw_hh)
    db_ih, db_hh = torch.empty(3 * H, device=DEV), torch.empty(3 * H, device=DEV)
    ops.colsum(dgxf, db_ih)
    ops.colsum(dghf, db_hh)
    torch.cuda.synchronize()
    torch.testing.assert_close(dx.cpu(), xr.grad, rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(dw_ih.cpu(), sdr["rnn.weight_ih_l0"].grad, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(dw_hh.cpu(), sdr["rnn.weight_hh_l0"].grad, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(db_ih.cpu(), sdr["rnn.bias_ih_l0"].grad, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(db_hh.cpu(), sdr["rnn.bias_hh_l0"].grad, rtol=1e-3, atol=1e-3)


def test_tgemm_skinny_split_k_is_deterministic_and_accumulates(hb, tgemm_feed):
    """The one-row-tile path reduces its K splits in split order (no atomics): repeated launches are bit-identical, and
    accumulate / ReLU / bias run once, in the reducing CTA."""
    from habitat_lab_b200 import ops

    torch.manual_seed(3)
    M, N, K = 64, 512, 2048
    x = torch.randn(M, K, device=DEV)
    w = torch.randn(N, K, device=DEV) / math.sqrt(K)
    b = torch.randn(N, device=DEV)
    outs = []
    for _ in range(3):
        o = torch.full((M, N), 7.0, device=DEV)
        ops.linear_fwd(x, w, b, o, relu=True, tf32=True)
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    ref = F.relu(F.linear(x.double(), w.double(), b.double())).float()
    torch.testing.assert_close(outs[0], ref, rtol=2e-3, atol=4e-3)
    # on a side stream (its own workspace), interleaved with the main stream
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    o_main = torch.empty(M, N, device=DEV)
    o_side = torch.empty(M, N, device=DEV)
    for _ in range(4):
        ops.linear_fwd(x, w, b, o_main, relu=False, tf32=True)
        with torch.cuda.stream(side):
            ops.linear_fwd(x, w, None, o_side, relu=False, tf32=True)
    torch.cuda.synchronize()
    torch.testing.assert_close(o_main - b, o_side, rtol=0, atol=1e-5)


@pytest.mark.parametrize("B,H,A", [(64, 512, 4), (7, 32, 6), (300, 128, 2)])
def test_heads_act(hb, B, H, A):
    """Fused tail of Policy.act: heads + log-softmax + draw / mode + log_probs(action) vs torch."""
    from habitat_lab_b200 import ops

    torch.manual_seed(B + A)
    feat = torch.randn(B, H, device=DEV)
    wa = torch.randn(A, H, device=DEV) * 0.2
    ba = torch.randn(A, device=DEV)
    wv = torch.randn(1, H, device=DEV) * 0.1
    bv = torch.randn(1, device=DEV)
    ref_lp = torch.log_softmax(F.linear(feat.double(), wa.double(), ba.double()), -1)
    ref_v = F.linear(feat.double(), wv.double(), bv.double())
    for u in (None, torch.rand(B, device=DEV), torch.zeros(B, device=DEV), torch.full((B,), 1.0 - 2 ** -24, device=DEV)):
        lp = torch.empty(B, A, device=DEV)
        val = torch.empty(B, 1, device=DEV)
        act = torch.full((B, 1), -1, device=DEV, dtype=torch.int64)
        alp = torch.empty(B, 1, device=DEV)
        ops.heads_act(feat, wa, ba, wv, bv, u, lp, val, act, alp)
        torch.cuda.synchronize()
        torch.testing.assert_close(lp.double(), ref_lp, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(val.double(), ref_v, rtol=1e-4, atol=1e-4)
        assert int(act.min()) >= 0 and int(act.max()) < A
        torch.testing.assert_close(alp, lp.gather(1, act), rtol=0, atol=0)
        if u is None:
            assert torch.equal(act.view(-1), lp.argmax(-1))
        else:
            # inverse CDF: the first action whose cumulative probability exceeds u (boundaries: within fp32 rounding)
            cdf = ref_lp.exp().cumsum(-1)
            lo = (cdf < (u.double().view(-1, 1) - 1e-5)).sum(-1).clamp(max=A - 1)
            hi = (cdf < (u.double().view(-1, 1) + 1e-5)).sum(-1).clamp(max=A - 1)
            a = act.view(-1)
            assert bool(((a >= lo) & (a <= hi)).all())
    # the draw follows the distribution: 20000 uniform numbers against one frame's probabilities
    n = 20000
    f1 = feat[:1].expand(n, H).contiguous()
    lp = torch.empty(n, A, device=DEV)
    val = torch.empty(n, 1, device=DEV)
    act = torch.empty(n, 1, device=DEV, dtype=torch.int64)
    alp = torch.empty(n, 1, device=DEV)
    ops.heads_act(f1, wa, ba, wv, bv, torch.rand(n, device=DEV), lp, val, act, alp)
    freq = torch.bincount(act.view(-1), minlength=A).double() / n
    assert (freq - ref_lp[0].exp()).abs().max().item() < 0.02


def test_embeddings(hb):
    from habitat_lab_b200 import ops

    rows, B, A = 40, 17, 4
    g = torch.Generator().manual_seed(2)
    goal = torch.rand(rows, 2, generator=g) * torch.tensor([10.0, 6.28]) - torch.tensor([0.0, 3.14])
    pa = torch.randint(0, A, (rows, 1), generator=g)
    masks = torch.rand(rows, 1, generator=g) > 0.3
    fr = torch.randint(0, rows, (B,), generator=g).int()
    w = torch.randn(32, 3, generator=g, requires_grad=True)
    b = torch.randn(32, generator=g, requires_grad=True)
    emb = torch.randn(A + 1, 32, generator=g, requires_grad=True)
    gsel = goal[fr.long()]
    gi = torch.stack([gsel[:, 0], torch.cos(-gsel[:, 1]), torch.sin(-gsel[:, 1])], -1)
    ref_t = F.linear(gi, w, b)
    idx = torch.where(masks[fr.long()].view(-1), pa[fr.long()].view(-1) + 1, torch.zeros(B, dtype=torch.long))
    ref_e = F.embedding(idx, emb)
    d = lambda t: t.detach().to(DEV).contiguous()  # noqa: E731
    out = torch.zeros(B, 576, device=DEV)
    pa_f, m_f = pa[fr.long()].view(-1), masks[fr.long()].view(-1)  # per-frame (gathered) like the minibatch
    ops.embed_fwd(d(goal), d(pa_f), d(m_f), d(fr), d(w), d(b), d(emb), out, 512)
    torch.testing.assert_close(out[:, 512:544].cpu(), ref_t.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(out[:, 544:576].cpu(), ref_e.detach(), rtol=0, atol=0)
    dout = torch.randn(B, 576, generator=g)
    (ref_t * dout[:, 512:544]).sum().backward()
    (ref_e * dout[:, 544:576]).sum().backward()
    dw, db, de = torch.zeros(32, 3, device=DEV), torch.zeros(32, device=DEV), torch.zeros(A + 1, 32, device=DEV)
    ops.embed_bwd(d(goal), d(pa_f), d(m_f), d(fr), d(dout), 512, dw, db, de)
    torch.cuda.synchronize()
    torch.testing.assert_close(dw.cpu(), w.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(db.cpu(), b.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(de.cpu(), emb.grad, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("C,oh0,ow0", [(32, 0, 0), (32, 16, 24), (64, 0, 8), (32, 16, 0)])
def test_tma_halo_probe(hb, C, oh0, ow0):
    """TMA box copies with out-of-bounds zero fill reproduce the zero-padded halo of a 16x8 tile of a 3x3 conv."""
    from habitat_lab_b200 import ops

    B, H, W, pad, hh, hw_ = 3, 32, 32, 1, 18, 10
    torch.manual_seed(C + oh0 + ow0)
    x = bf(torch.randn(B, H, W, C, device=DEV))
    out = torch.empty(C // 8, hh, hw_, 8, device=DEV, dtype=torch.bfloat16)
    b = 1
    ops.tma_halo_probe(x, out, b, oh0, ow0, hh, hw_, pad)
    torch.cuda.synchronize()
    xp = F.pad(x[b].float().permute(2, 0, 1), (pad, hw_, pad, hh))[:, oh0: oh0 + hh, ow0: ow0 + hw_]   # [C, hh, hw]
    ref = xp.reshape(C // 8, 8, hh, hw_).permute(0, 2, 3, 1)
    assert torch.equal(out.float(), ref)
