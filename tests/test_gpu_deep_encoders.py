"""GPU parity of the ResNet50 / ResNeXt50 encoder layers (configs #3 / #4), kernel by kernel, and run-to-run identity of
every kernel that sums gradients across blocks.

Conventions of tests/test_gpu_kernels.py: convolutions are compared with an fp32 convolution of the SAME rounded operands
(forward fp16 = hf(), gradients bf16 = bf()) with TF32 off, so only accumulation order and the final rounding of the
output differ; absolute bars are scaled by the reference's max.  Each conv test also checks its own bar: the reference
with its last N tile zeroed (see zero_last_tile) and, for the forward and dgrad passes whose reduction runs over more than
64 channels, with the last 64-channel K chunk dropped, must miss the bar by at least 10x, so a kernel that loses a tile or
a K chunk cannot pass.  (The weight gradient reduces over pixels: one lost 128-pixel chunk out of up to a million is
within its bar, so only its N tiles are guarded.)
"""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

DEV = "cuda"

# Every unique conv layer EncoderEngine builds at 256x256 input with the generic input prep (allow_s2d=False).
# (ci_real, ci, co, k, stride, pad, in_hw, conv_groups, gn_groups, family); family is the kernel route:
#   stem    7x7 s2 gather conv over the 8-channel padded input, no dgrad
#   gather  conv_fwd / conv_dgrad / conv_wgrad (implicit GEMM, conv.cu)
#   halo    conv_halo forward and dgrad, conv_halo_wgrad (conv_halo.cu)
#   gather+halo_wgrad   gather forward / dgrad, small-image halo weight gradient
# tests/test_reduction_order.py rebuilds the engines on the CPU and fails if one produces a layer missing here.
LAYER_TABLE = [
    # ---- config #3, ObjectNav ResNet50 (rgb 3 + depth 1 + semantic 1 input channels)
    (5, 8, 32, 7, 2, 3, 128, 1, 16, "stem"),                 # stem, 5 real channels padded to 8
    (32, 32, 32, 3, 1, 1, 32, 1, 16, "halo"),                # layer1 3x3
    (32, 32, 32, 1, 1, 0, 32, 1, 16, "gather"),              # layer1.0 1x1 reduce
    (32, 32, 128, 1, 1, 0, 32, 1, 16, "gather"),             # layer1 1x1 expand / downsample
    (64, 64, 64, 3, 2, 1, 32, 1, 16, "gather"),              # layer2.0 3x3 s2
    (128, 128, 32, 1, 1, 0, 32, 1, 16, "gather"),            # layer1 1x1 reduce
    (128, 128, 64, 1, 1, 0, 32, 1, 16, "gather"),            # layer2.0 1x1 reduce
    (128, 128, 256, 1, 2, 0, 32, 1, 16, "gather"),           # layer2.0 downsample 1x1 s2
    (64, 64, 64, 3, 1, 1, 16, 1, 16, "halo"),                # layer2 3x3
    (64, 64, 256, 1, 1, 0, 16, 1, 16, "gather"),             # layer2 1x1 expand
    (128, 128, 128, 3, 2, 1, 16, 1, 16, "gather"),           # layer3.0 3x3 s2
    (256, 256, 64, 1, 1, 0, 16, 1, 16, "gather"),            # layer2 1x1 reduce
    (256, 256, 128, 1, 1, 0, 16, 1, 16, "gather"),           # layer3.0 1x1 reduce
    (256, 256, 512, 1, 2, 0, 16, 1, 16, "gather"),           # layer3.0 downsample 1x1 s2
    (128, 128, 128, 3, 1, 1, 8, 1, 16, "gather+halo_wgrad"),  # layer3 3x3
    (128, 128, 512, 1, 1, 0, 8, 1, 16, "gather"),            # layer3 1x1 expand (4 N tiles)
    (256, 256, 256, 3, 2, 1, 8, 1, 16, "gather"),            # layer4.0 3x3 s2
    (512, 512, 128, 1, 1, 0, 8, 1, 16, "gather"),            # layer3 1x1 reduce
    (512, 512, 256, 1, 1, 0, 8, 1, 16, "gather"),            # layer4.0 1x1 reduce
    (512, 512, 1024, 1, 2, 0, 8, 1, 16, "gather"),           # layer4.0 downsample 1x1 s2 (8 N tiles)
    (256, 256, 256, 3, 1, 1, 4, 1, 16, "gather+halo_wgrad"),  # layer4 3x3
    (256, 256, 1024, 1, 1, 0, 4, 1, 16, "gather"),           # layer4 1x1 expand (64 channels per GN group)
    (1024, 1024, 128, 3, 1, 1, 4, 1, 1, "gather+halo_wgrad"),  # compression, one GN group over 128 channels
    (1024, 1024, 256, 1, 1, 0, 4, 1, 16, "gather"),          # layer4 1x1 reduce (K = 1024)
    # ---- config #4, ImageNav ResNeXt50 (two rgb encoders; cardinality 16)
    (3, 8, 32, 7, 2, 3, 128, 1, 16, "stem"),                 # stem, 3 real channels padded to 8
    (32, 32, 64, 1, 1, 0, 32, 1, 16, "gather"),              # layer1.0 1x1 reduce
    (64, 64, 64, 3, 1, 1, 32, 16, 16, "halo"),               # layer1 grouped 3x3 (block-diagonal weight)
    (64, 64, 64, 3, 1, 1, 32, 1, 16, "halo"),                # 3x3 64 @32 dense
    (64, 64, 128, 1, 1, 0, 32, 1, 16, "gather"),             # layer1 1x1 expand
    (128, 128, 64, 1, 1, 0, 32, 1, 16, "gather"),            # layer1 1x1 reduce
    (128, 128, 128, 3, 2, 1, 32, 16, 16, "gather"),          # layer2.0 grouped 3x3 s2
    (128, 128, 128, 1, 1, 0, 32, 1, 16, "gather"),           # layer2.0 1x1 reduce
    (128, 128, 256, 1, 2, 0, 32, 1, 16, "gather"),           # layer2.0 downsample 1x1 s2
    (128, 128, 128, 3, 1, 1, 16, 1, 16, "gather"),           # 3x3 128 @16 dense
    (128, 128, 256, 1, 1, 0, 16, 1, 16, "gather"),           # layer2 1x1 expand
    (256, 256, 128, 1, 1, 0, 16, 1, 16, "gather"),           # layer2 1x1 reduce
    (256, 256, 256, 3, 2, 1, 16, 16, 16, "gather"),          # layer3.0 grouped 3x3 s2
    (256, 256, 256, 1, 1, 0, 16, 1, 16, "gather"),           # layer3.0 1x1 reduce
    (256, 256, 512, 1, 2, 0, 16, 1, 16, "gather"),           # layer3.0 downsample 1x1 s2
    (256, 256, 256, 3, 1, 1, 8, 1, 16, "gather+halo_wgrad"),  # 3x3 256 @8 (small-image halo wgrad)
    (256, 256, 512, 1, 1, 0, 8, 1, 16, "gather"),            # layer3 1x1 expand
    (512, 512, 256, 1, 1, 0, 8, 1, 16, "gather"),            # layer3 1x1 reduce
    (512, 512, 512, 1, 1, 0, 8, 1, 16, "gather"),            # layer4.0 1x1 reduce
    (512, 512, 512, 3, 2, 1, 8, 16, 16, "gather"),           # layer4.0 grouped 3x3 s2
    (512, 512, 1024, 1, 2, 0, 8, 1, 16, "gather"),           # layer4.0 downsample 1x1 s2
    (512, 512, 512, 3, 1, 1, 4, 1, 16, "gather+halo_wgrad"),  # 3x3 512 @4 (small-image halo wgrad)
    (512, 512, 1024, 1, 1, 0, 4, 1, 16, "gather"),           # layer4 1x1 expand
    (1024, 1024, 128, 3, 1, 1, 4, 1, 1, "gather+halo_wgrad"),  # compression (as config #3)
    (1024, 1024, 512, 1, 1, 0, 4, 1, 16, "gather"),          # layer4 1x1 reduce
    # ---- config #2, PointNav ResNet18 (its stride-2 block entry pair is covered by test_conv_s2_block_entry)
    (4, 8, 32, 7, 2, 3, 128, 1, 16, "stem"),
    (64, 64, 128, 3, 2, 1, 16, 1, 16, "gather"),
    (64, 64, 128, 1, 2, 0, 16, 1, 16, "gather"),
    (128, 128, 256, 1, 2, 0, 8, 1, 16, "gather"),
    (128, 128, 256, 3, 2, 1, 8, 1, 16, "gather"),
    (256, 256, 128, 3, 1, 1, 4, 1, 1, "gather+halo_wgrad"),
]
# the learner's minibatch of configs #3 / #4 (T * N / num_mini_batch = 64 * 32 / 2) and an actor-sized batch (fewer than
# 132 row tiles: the gather kernel's sliced-N-tile launch)
BATCHES = {"actor": 2, "learner": 1024}


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def bf(x):
    return x.to(torch.bfloat16)


def hf(x):
    return x.to(torch.float16)


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def bar_ratio(got, ref, rtol, atol):
    """max over elements of |got - ref| / (atol + rtol |ref|): <= 1 passes torch.testing.assert_close's bar"""
    return ((got.double() - ref.double()).abs() / (atol + rtol * ref.double().abs())).max().item()


def check(name, got, ref, rtol, atol_rel, perturbed=()):
    """got vs ref with atol = atol_rel * max|ref|; every perturbed reference must miss that bar by >= 10x"""
    atol = atol_rel * max(ref.abs().max().item(), 1e-30)
    r = bar_ratio(got, ref, rtol, atol)
    guards = [bar_ratio(p, ref, rtol, atol) for p in perturbed]
    print(f"  {name}: error / bar {r:.3f}; perturbed-tile error / bar {[round(g, 1) for g in guards]}")
    assert r <= 1.0, f"{name}: error {r:.3f}x the bar"
    for g in guards:
        assert g >= 10.0, f"{name}: a zeroed tile / dropped K chunk only misses the bar by {g:.2f}x"


def zero_last_tile(t, dim=1):
    """t with its last N tile along dim zeroed: 128 columns where the dimension spans more than one such tile, else the
    last 32 (the width of the actor launch's N slices) or, for dimensions of 32 and less, the last 8 channels (one
    vector) -- always a strict part of the dimension, so a lost slice is visible however narrow the layer"""
    n = t.shape[dim]
    tile = 128 if n > 128 else (32 if n > 32 else 8)
    out = t.clone()
    out.narrow(dim, ((n - 1) // tile) * tile, n - ((n - 1) // tile) * tile).zero_()
    return out


def _block_diag_conv(ci, co, k, stride, pad, cg, in_hw, G):
    from habitat_lab_b200.rl.resnet_policy import _Conv

    conv = nn.Conv2d(ci, co, k, stride, pad, groups=cg, bias=False).to(DEV)
    c = _Conv(conv, nn.GroupNorm(G, co).to(DEV), (in_hw, in_hw))
    if cg > 1:
        c._wd = torch.zeros(co, ci, k, k, device=DEV)
        c._gd = torch.empty_like(c._wd)
    conv.weight.grad = torch.zeros_like(conv.weight)
    return c


@pytest.mark.parametrize("batch", list(BATCHES), ids=list(BATCHES))
@pytest.mark.parametrize("layer", LAYER_TABLE, ids=lambda r: "{}-{}-{}k{}s{}@{}g{}G{}-{}".format(*r[:4], r[4], r[6], r[7],
                                                                                                r[8], r[9]))
def test_layer_parity(hb, layer, batch):
    from habitat_lab_b200 import ops

    ci_real, ci, co, k, stride, pad, hw, cg, G, family = layer
    B = BATCHES[batch]
    torch.manual_seed(sum(layer[:9]) + B)
    c = _block_diag_conv(ci_real, co, k, stride, pad, cg, hw, G)
    with torch.no_grad():
        c.w.normal_(0.0, 1.0 / math.sqrt(ci_real // cg * k * k))
    w_g = c.w.data                          # [co, ci / cg, k, k], the parameter
    w = c.dense_weight()                    # [co, ci, k, k], block-diagonal when grouped
    x = torch.randn(B, ci_real, hw, hw, device=DEV)
    ho = (hw + 2 * pad - k) // stride + 1
    halo = family == "halo"
    print(f"\n{layer} B={B}")

    # ---- forward + fused GroupNorm statistics
    xh = hf(x).float()
    y_ref = F.conv2d(xh, hf(w_g).float(), stride=stride, padding=pad, groups=cg)
    x_nhwc = torch.zeros(B, hw, hw, ci, device=DEV, dtype=torch.float16)
    x_nhwc[..., :ci_real] = hf(nhwc(x))
    y = torch.empty(B, ho, ho, co, device=DEV, dtype=torch.float16)
    stats = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
    if halo:
        wh = torch.empty(9 * ci * co, dtype=torch.float16, device=DEV)
        wht = torch.empty(9 * ci * co, dtype=torch.bfloat16, device=DEV)
        ops.pack_halo_weight(w, wh, ci, co, 3, 0)
        ops.pack_halo_weight(w, wht, co, ci, 3, 1)
        ops.conv_halo(x_nhwc, wh, y, B, hw, hw, ci, co, 3, 0, gn_stats=stats, gn_groups=G)
    else:
        s = ops.conv_shape(B, hw, hw, ci, co, k, k, stride, pad)
        wp, wt = ops.pack_conv_weight(w, ci, want_t=family != "stem")
        ops.conv_fwd(x_nhwc, wp, y, s, stats, G)
    torch.cuda.synchronize()
    pert = [zero_last_tile(y_ref)]
    if ci_real > 64:
        xk = xh.clone()
        xk[:, ci_real - 64:] = 0
        pert.append(F.conv2d(xk, hf(w_g).float(), stride=stride, padding=pad, groups=cg))
    check("forward", nchw(y.float()), y_ref, 2e-3, 2e-3, pert)
    del pert
    yg = y_ref.double().reshape(B, G, -1)
    for j, ref in enumerate((yg.sum(-1), (yg * yg).sum(-1))):
        # the kernel sums its fp32 accumulators, the reference the fp32 outputs of cuDNN: both within ~1e-6 relative
        # per element, so the sums agree to 1e-4 of the sum of magnitudes
        scale = (yg.abs() if j == 0 else yg * yg).sum(-1)
        err = ((stats[..., j] - ref).abs() / (1e-4 * scale + 1e-6)).max().item()
        assert err <= 1.0, f"GroupNorm {'sum' if j == 0 else 'sum of squares'}: {err:.3f}x the bar"

    # ---- weight gradient through the engine's unpack (and store_grad for grouped layers): bf16 x twin, bf16 dy
    dy = torch.randn_like(y_ref)
    dyb = bf(dy).float()
    dy_nhwc = bf(nhwc(dy))
    xb = bf(x).float()
    dw_ref = torch.nn.grad.conv2d_weight(xb, w_g.shape, dyb, stride=stride, padding=pad, groups=cg)
    x_b = torch.zeros(B, hw, hw, ci, device=DEV, dtype=torch.bfloat16)
    x_b[..., :ci_real] = bf(nhwc(x))
    acc = torch.zeros(k * k * ci, co, device=DEV)
    if family in ("halo", "gather+halo_wgrad"):
        ops.conv_halo_wgrad(x_b, dy_nhwc, acc, B, hw, hw, ci, co, 3)
    else:
        ops.conv_wgrad(x_b, dy_nhwc, acc, s)
    ops.unpack_conv_wgrad(acc, c.grad_target(), ci)
    c.store_grad()
    torch.cuda.synchronize()
    check("wgrad", c.w.grad, dw_ref, 2e-3, 2e-3, [zero_last_tile(dw_ref, dim=0)])
    if family == "stem":
        return

    # ---- data gradient (bf16 weight image x bf16 dy), without and with the fused residual-gradient addend.
    # The operands are the kernel's, exactly; the bf16 output rounds by at most 2^-8 relative (8 significand bits), and
    # the fp32 accumulation adds ~1e-6: rtol 8e-3 is twice the rounding bound, atol 2e-3 of the max covers values near 0.
    wb = bf(w_g).float()
    dgrad_ref = lambda d: torch.nn.grad.conv2d_input(x.shape, wb, d, stride=stride, padding=pad, groups=cg)  # noqa: E731
    dx_ref = dgrad_ref(dyb)
    dx_pert = [zero_last_tile(dx_ref)]
    if co > 64:   # the last 64-channel chunk of the reduction (K = Co x k x k) dropped
        dyk = dyb.clone()
        dyk[:, co - 64:] = 0
        dx_pert.append(dgrad_ref(dyk))
    dx = torch.empty(B, hw, hw, ci, device=DEV, dtype=torch.bfloat16)
    addend = bf(torch.randn(B, hw, hw, ci, device=DEV))
    for add in (None, addend):
        if halo:
            ops.conv_halo(dy_nhwc, wht, dx, B, hw, hw, co, ci, 3, 1, addend=add)
        else:
            ops.conv_dgrad(dy_nhwc, wt, dx, s, addend=add)
        torch.cuda.synchronize()
        ref = dx_ref if add is None else dx_ref + nchw(add.float())
        check("dgrad" + ("" if add is None else "+addend"), nchw(dx.float()), ref, 8e-3, 2e-3,
              dx_pert if add is None else ())


# ---------------------------------------------------------------------------------------------
# GroupNorm at the deep shapes: 32 / 64 channels per group (C = 512 / 1024, 16 groups) and 1 group over 128 channels
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,G", [(512, 16), (1024, 16), (128, 1)])
@pytest.mark.parametrize("hw", [64, 16])
def test_groupnorm_deep(hb, C, G, hw):
    from habitat_lab_b200 import ops

    B, H = 24, int(math.isqrt(hw))
    torch.manual_seed(C + hw)
    y = hf(torch.randn(B, C, H, H, device=DEV) * 1.5 + 0.3).float()
    res = hf(torch.randn(B, C, H, H, device=DEV)).float()
    gamma, beta = torch.rand(C, device=DEV) + 0.5, torch.randn(C, device=DEV) * 0.2
    yd = y.double()
    yg = yd.reshape(B, G, -1)
    stats = torch.stack([yg.sum(-1), (yg * yg).sum(-1)], -1).contiguous()
    yb, resb = hf(nhwc(y)), hf(nhwc(res))
    g = bf(torch.randn(B, C, H, H, device=DEV)).float()
    gb = bf(nhwc(g))
    gn64 = lambda t, ga, be: F.group_norm(t, G, ga.double(), be.double(), eps=1e-5)  # noqa: E731

    # forward: GN + ReLU (fp16 output + bf16 twin), residual block output with and without downsample GN
    out = torch.empty_like(yb)
    out_b = torch.empty_like(yb, dtype=torch.bfloat16)
    ops.gn_apply(yb, stats, gamma, beta, out, B, hw, C, G, relu=True, out_bf16=out_b)
    a_ref = F.relu(gn64(yd, gamma, beta))
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(out.float()).double(), a_ref, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(nchw(out_b.float()).double(), a_ref, rtol=8e-3, atol=8e-3)
    blk = torch.empty_like(yb)
    ops.gn_residual_relu(yb, stats, gamma, beta, resb, blk, B, hw, C, G)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(blk.float()).double(), F.relu(gn64(yd, gamma, beta) + res.double()), rtol=2e-3,
                               atol=4e-3)
    gd, bd = torch.rand(C, device=DEV) + 0.5, torch.randn(C, device=DEV) * 0.1
    rg = res.double().reshape(B, G, -1)
    rstats = torch.stack([rg.sum(-1), (rg * rg).sum(-1)], -1).contiguous()
    ops.gn_residual_relu(yb, stats, gamma, beta, resb, blk, B, hw, C, G, rstats, gd, bd)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(blk.float()).double(), F.relu(gn64(yd, gamma, beta) + gn64(res.double(), gd, bd)),
                               rtol=2e-3, atol=6e-3)

    # backward, modes 0 (GN), 1 (GN + ReLU), 2 (residual block: mask from the block output, gz written)
    o2 = F.relu(gn64(yd, gamma, beta) + res.double())
    act = hf(nhwc(o2.float()))
    for mode in (0, 1, 2):
        yr = yd.clone().requires_grad_(True)
        gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        rr = res.double().requires_grad_(True)
        z = F.group_norm(yr, G, gr, br, eps=1e-5)
        if mode == 1:
            z = F.relu(z)
        elif mode == 2:
            # the mask is the stored fp16 block output > 0 (what the kernel reads)
            z = (z + rr) * (nchw(act.float()).double() > 0)
        z.backward(g.double())
        dga, dbe = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        dy = torch.empty_like(gb)
        gz = torch.empty_like(gb) if mode == 2 else None
        ops.gn_bwd(gb, act if mode == 2 else None, yb, stats, gamma, beta, dga, dbe, dy, gz, B, hw, C, G, mode)
        torch.cuda.synchronize()
        sc = yr.grad.abs().max().item()
        torch.testing.assert_close(nchw(dy.float()).double(), yr.grad, rtol=2e-2, atol=1e-2 * sc)
        torch.testing.assert_close(dga.double(), gr.grad, rtol=1e-3, atol=1e-3 * gr.grad.abs().max().item())
        torch.testing.assert_close(dbe.double(), br.grad, rtol=1e-3, atol=1e-3 * br.grad.abs().max().item())
        if mode == 2:
            torch.testing.assert_close(nchw(gz.float()).double(), rr.grad, rtol=1e-2, atol=1e-2)
        # dgamma / dbeta are summed across frames: the same bits every run, on either stream
        got = _twice(lambda: ops.gn_bwd(gb, act if mode == 2 else None, yb, stats, gamma, beta, dga, dbe, dy, gz, B, hw,
                                        C, G, mode), [dga, dbe])
        assert torch.equal(got[0], dga) and torch.equal(got[1], dbe)


# ---------------------------------------------------------------------------------------------
# generic 1-D sensors and embeddings (configs #3 / #4: compass, gps, objectgoal, prev-action)
# ---------------------------------------------------------------------------------------------
def _features64(x, transform):
    x = x.double()
    if transform == 1:
        return torch.stack([x[:, 0], torch.cos(-x[:, 1]), torch.sin(-x[:, 1])], -1)
    if transform == 2:
        s = torch.sin(x[:, 2])
        return torch.stack([x[:, 0], torch.cos(-x[:, 1]) * s, torch.sin(-x[:, 1]) * s, torch.cos(x[:, 2])], -1)
    if transform == 3:
        return torch.stack([torch.cos(x[:, 0]), torch.sin(x[:, 0])], -1)
    return x


SENSOR_CASES = [  # transform, in_dim, out_dim
    (0, 1, 1), (0, 2, 32), (0, 3, 64), (0, 8, 17), (0, 5, 5), (1, 2, 32), (2, 3, 64), (3, 1, 32), (3, 1, 7)]


@pytest.mark.parametrize("rows_kind", ["shuffled", "repeated"])
@pytest.mark.parametrize("transform,in_dim,out_dim", SENSOR_CASES)
@pytest.mark.parametrize("raw", [False, True], ids=["linear", "raw_copy"])
def test_sensor_linear(hb, transform, in_dim, out_dim, rows_kind, raw):
    from habitat_lab_b200 import ops

    if raw and not (transform == 0 and out_dim == in_dim):
        pytest.skip("the raw copy exists for identity features only")
    torch.manual_seed(transform * 100 + in_dim * 10 + out_dim)
    n_rows, B, col0, ld = 3000, 2500, 5, 80
    x = torch.randn(n_rows, in_dim, device=DEV) * 3.0
    rows = (torch.randperm(n_rows, device=DEV)[:B] if rows_kind == "shuffled"
            else torch.randint(0, 4, (B,), device=DEV)).to(torch.int32)
    ft = _features64(x[rows.long()], transform)
    nf = ft.shape[1]
    w = None if raw else torch.randn(out_dim, nf, device=DEV) / math.sqrt(nf)
    b = None if raw else torch.randn(out_dim, device=DEV)
    out = torch.full((B, ld), 7.0, device=DEV)
    ops.sensor_linear_fwd(x, rows, transform, w, b, out, col0, out_dim)
    ref = ft if raw else ft @ w.double().t() + b.double()
    torch.cuda.synchronize()
    torch.testing.assert_close(out[:, col0:col0 + out_dim].double(), ref, rtol=1e-5, atol=1e-5)
    assert (out[:, :col0] == 7).all() and (out[:, col0 + out_dim:] == 7).all()
    if raw:
        return
    d_out = torch.randn(B, ld, device=DEV)
    d_w0, d_b0 = torch.randn(out_dim, nf, device=DEV), torch.randn(out_dim, device=DEV)
    d_w, d_b = d_w0.clone(), d_b0.clone()
    ops.sensor_linear_bwd(x, rows, transform, d_out, col0, out_dim, d_w, d_b)
    g = d_out[:, col0:col0 + out_dim].double()
    torch.cuda.synchronize()
    # the kernel adds to what the gradient buffers hold
    torch.testing.assert_close(d_w.double(), d_w0.double() + g.t() @ ft, rtol=1e-5, atol=2e-4 * math.sqrt(B))
    torch.testing.assert_close(d_b.double(), d_b0.double() + g.sum(0), rtol=1e-5, atol=2e-4 * math.sqrt(B))
    d_w2, d_b2 = d_w0.clone(), d_b0.clone()
    ops.sensor_linear_bwd(x, rows, transform, d_out, col0, out_dim, d_w2, d_b2)
    torch.cuda.synchronize()
    assert torch.equal(d_w2, d_w) and torch.equal(d_b2, d_b)


@pytest.mark.parametrize("kind", ["objectgoal", "prev_action"])
@pytest.mark.parametrize("spread", ["uniform", "one_row"])
def test_index_embed(hb, kind, spread):
    from habitat_lab_b200 import ops

    torch.manual_seed(3 if kind == "objectgoal" else 4)
    B, width, col0, ld = 3000, 32, 64, 128
    n_table = 21 if kind == "objectgoal" else 7   # objectgoal categories; prev-action: 6 actions + the start token
    table = torch.randn(n_table, width, device=DEV)
    if kind == "objectgoal":
        n_src = 4000
        idx = (torch.randint(0, n_table, (n_src, 1), device=DEV) if spread == "uniform"
               else torch.full((n_src, 1), 5, device=DEV, dtype=torch.int64))
        rows = torch.randperm(n_src, device=DEV)[:B].to(torch.int32)
        masks = None
        k = idx.view(-1)[rows.long()]
    else:
        idx = (torch.randint(0, n_table - 1, (B,), device=DEV) if spread == "uniform"
               else torch.full((B,), 2, device=DEV, dtype=torch.int64))
        rows = None
        masks = torch.rand(B, device=DEV) > 0.2
        k = torch.where(masks, idx + 1, torch.zeros_like(idx))
    out = torch.zeros(B, ld, device=DEV)
    ops.index_embed_fwd(idx, rows, masks, table, out, col0, B)
    torch.cuda.synchronize()
    assert torch.equal(out[:, col0:col0 + width], table[k])
    d_out = torch.randn(B, ld, device=DEV)
    d0 = torch.randn(n_table, width, device=DEV)
    ref = d0.double().index_add(0, k, d_out[:, col0:col0 + width].double())
    d_table = d0.clone()
    ops.index_embed_bwd(idx, rows, masks, d_out, col0, d_table, B)
    torch.cuda.synchronize()
    torch.testing.assert_close(d_table.double(), ref, rtol=1e-5, atol=1e-5 * B)
    d_table2 = d0.clone()
    ops.index_embed_bwd(idx, rows, masks, d_out, col0, d_table2, B)
    torch.cuda.synchronize()
    assert torch.equal(d_table2, d_table)
    # an index outside the table poisons the forward row with NaN and adds nothing in the backward pass
    bad = idx.clone()
    f_bad = 17
    src_bad = rows[f_bad].long() if rows is not None else f_bad
    bad.view(-1)[src_bad] = n_table + 3
    if masks is not None:
        masks[f_bad] = True
    ops.index_embed_fwd(bad, rows, masks, table, out, col0, B)
    d_table3 = d0.clone()
    ops.index_embed_bwd(bad, rows, masks, d_out, col0, d_table3, B)
    torch.cuda.synchronize()
    assert torch.isnan(out[f_bad, col0:col0 + width]).all()
    keep = torch.ones(B, dtype=torch.bool, device=DEV)
    keep[f_bad] = False
    if rows is not None:
        keep &= rows.long() != src_bad
    kk = torch.where(masks, bad + 1, torch.zeros_like(bad)) if masks is not None else bad.view(-1)[rows.long()]
    ref3 = d0.double().index_add(0, kk[keep], d_out[keep, col0:col0 + width].double())
    torch.testing.assert_close(d_table3.double(), ref3, rtol=1e-5, atol=1e-5 * B)


# ---------------------------------------------------------------------------------------------
# generic visual input prep (configs #3 / #4): u8 / f32 / i32 sources -> 2x2 average pool -> RunningMeanAndVar
# ---------------------------------------------------------------------------------------------
PREP_SOURCES = {   # name -> [(dtype, channels, pre-pool scale)], in concatenation order
    "u8": [(torch.uint8, 3, 1.0 / 255.0)],
    "f32": [(torch.float32, 1, 1.0)],
    "i32": [(torch.int32, 1, 1.0)],
    "u8+f32+i32": [(torch.uint8, 3, 1.0 / 255.0), (torch.float32, 1, 1.0), (torch.int32, 1, 1.0)],   # config #3's set
    "u8+u8": [(torch.uint8, 3, 1.0 / 255.0), (torch.uint8, 3, 1.0 / 255.0)],
}


@pytest.mark.parametrize("H,W", [(32, 48), (33, 47), (6, 2)], ids=["even", "odd", "tiny"])
@pytest.mark.parametrize("kind", list(PREP_SOURCES))
def test_prep_generic(hb, kind, H, W):
    from habitat_lab_b200 import ops
    from oracle import torch_oracle as O

    torch.manual_seed(len(kind) * 100 + H + W)
    n_rows, B = 40, 300
    srcs, xs = [], []
    for dt, C, scale in PREP_SOURCES[kind]:
        if dt == torch.uint8:
            t = torch.randint(0, 256, (n_rows, H, W, C), device=DEV, dtype=dt)
        elif dt == torch.int32:
            t = torch.randint(0, 40, (n_rows, H, W, C), device=DEV, dtype=dt)   # semantic class ids
        else:
            t = torch.rand(n_rows, H, W, C, device=DEV)
        srcs.append((t, scale))
    rows = torch.randint(0, n_rows, (B,), device=DEV, dtype=torch.int32)   # shuffled, with repeats
    for t, scale in srcs:
        # the kernel scales each value in fp32 before pooling (ATen's order for u8 keys: x.float() / high)
        xs.append((t[rows.long()].permute(0, 3, 1, 2).float() * scale).double())
    x = F.avg_pool2d(torch.cat(xs, 1), 2)   # drops the odd last row / column
    C = x.shape[1]
    hw = (H // 2) * (W // 2)

    # statistics pass: fp64 per-channel sum / sum of squares of the pooled values, frame count
    stats = torch.zeros(17, dtype=torch.float64, device=DEV)
    ops.prep_generic(srcs, rows, H, W, stats_acc=stats)
    torch.cuda.synchronize()
    xc = x.transpose(0, 1).reshape(C, -1)
    # fp32 pooled values summed per thread in fp32 (a few dozen each), then in fp64
    torch.testing.assert_close(stats[:C], xc.sum(-1), rtol=1e-5, atol=1e-6 * xc.abs().sum(-1).max().item())
    torch.testing.assert_close(stats[8:8 + C], (xc * xc).sum(-1), rtol=1e-5, atol=0)
    assert (stats[C:8] == 0).all() and (stats[8 + C:16] == 0).all() and stats[16].item() == B

    # running mean / var update (prep_finalize, as the policy calls it) vs the oracle's RunningMeanAndVar
    mean, var, count = torch.rand(1, C, 1, 1, dtype=torch.float64), torch.rand(1, C, 1, 1, dtype=torch.float64) + 0.01, \
        torch.tensor(7.0, dtype=torch.float64)
    m2, v2, c2 = O.running_mean_var_update(x.cpu(), mean, var, count)
    rm, rv, rc = mean.view(-1).float().to(DEV), var.view(-1).float().to(DEV), count.view(1).float().to(DEV)
    ss = torch.zeros(16, device=DEV)
    ops.prep_finalize(stats, rm, rv, rc, ss, C, hw, True)
    torch.cuda.synchronize()
    torch.testing.assert_close(rm.double().cpu(), m2.view(-1), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(rv.double().cpu(), v2.view(-1), rtol=1e-4, atol=1e-6)
    assert rc.item() == c2.item()

    # apply pass: normalised fp16 NHWC padded to 8 channels, and its bf16 twin
    ref = O.running_mean_var_apply(x.cpu(), rm.double().cpu().view(1, -1, 1, 1), rv.double().cpu().view(1, -1, 1, 1))
    out = torch.full((B, H // 2, W // 2, 8), 5.0, device=DEV, dtype=torch.float16)
    out_b = torch.full_like(out, 5.0, dtype=torch.bfloat16)
    ops.prep_generic(srcs, rows, H, W, scale_shift=ss, out=out, out_bf16=out_b)
    torch.cuda.synchronize()
    got, got_b = nchw(out.float()).double().cpu(), nchw(out_b.float()).double().cpu()
    sc = ref.abs().max().item()
    torch.testing.assert_close(got[:, :C], ref, rtol=2e-3, atol=2e-3 * sc)    # fp16: 2^-11 relative rounding
    torch.testing.assert_close(got_b[:, :C], ref, rtol=8e-3, atol=8e-3 * sc)  # bf16: 2^-8
    assert (got[:, C:] == 0).all() and (got_b[:, C:] == 0).all()
    # without scale_shift the pass writes the pooled values themselves
    ops.prep_generic(srcs, rows, H, W, out=out)
    torch.cuda.synchronize()
    torch.testing.assert_close(nchw(out.float()).double().cpu()[:, :C], x.cpu(), rtol=1e-3, atol=1e-3)


# ---------------------------------------------------------------------------------------------
# run-to-run identity of the kernels that sum across blocks (second launch also on a side stream)
# ---------------------------------------------------------------------------------------------
_side_stream = []


def side_stream():
    """one side stream for the module, as the learner keeps one (SideStream)"""
    if not _side_stream:
        _side_stream.append(torch.cuda.Stream())
    return _side_stream[0]


def _twice(fn, outs):
    """fn() twice on the main stream and once on a side stream into zeroed outputs: all three bit-identical"""
    got = []
    for side in (False, False, True):
        for o in outs:
            o.zero_()
        if side:
            s = side_stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn()
            torch.cuda.current_stream().wait_stream(s)
        else:
            fn()
        torch.cuda.synchronize()
        got.append([o.clone() for o in outs])
    for run in got[1:]:
        for a, b in zip(got[0], run):
            assert torch.equal(a, b)
    return got[0]


def test_relu_bias_bwd_is_deterministic_and_exact(hb):
    from habitat_lab_b200 import ops

    torch.manual_seed(11)
    B, hw, C = 512, 31 * 31, 32   # SimpleCNN conv 2 of config #1
    g = bf(torch.randn(B * hw, C, device=DEV))
    out = hf(torch.randn(B * hw, C, device=DEV))
    dy = torch.empty_like(g)
    db = torch.zeros(C, device=DEV)
    (d,) = _twice(lambda: ops.relu_bias_bwd(g, out, dy, db, B * hw, C), [db])
    gm = g.double() * (out.float() > 0)
    # fp32 partials of ~450 pixels added over ~1000 blocks: ~1e-3 absolute; a lost block moves a sum by ~20
    torch.testing.assert_close(d.double(), gm.sum(0), rtol=1e-5, atol=2e-2)
    assert torch.equal(dy, bf(gm.float()))
    (d0,) = _twice(lambda: ops.relu_bias_bwd(g, None, None, db, B * hw, C), [db])
    torch.testing.assert_close(d0.double(), g.double().sum(0), rtol=1e-5, atol=2e-2)


@pytest.mark.parametrize("M,N,K", [(4097, 512, 256), (2050, 96, 66)])
def test_sgemm_split_k_is_deterministic_and_accumulates(hb, M, N, K):
    """fp32 linear weight gradient over M frames (M % 4 != 0: the TF32 path is refused): split-K over frames"""
    from habitat_lab_b200 import ops

    torch.manual_seed(M + N)
    dy, x = torch.randn(M, N, device=DEV), torch.randn(M, K, device=DEV)
    dw0 = torch.randn(N, K, device=DEV)
    dw = torch.empty(N, K, device=DEV)

    def run():
        dw.copy_(dw0)
        ops.linear_bwd_weight(dy, x, dw, accumulate=True, tf32=True)

    (got,) = _twice(run, [dw])
    ref = dw0.double() + dy.double().t() @ x.double()
    torch.testing.assert_close(got.double(), ref, rtol=1e-4, atol=1e-4 * ref.abs().max().item())


@pytest.mark.parametrize("route", ["gather", "halo", "halo_small"])
def test_conv_wgrad_is_deterministic(hb, route):
    from habitat_lab_b200 import ops

    B, hw, C, N = {"gather": (1024, 8, 256, 512), "halo": (512, 32, 32, 32), "halo_small": (1024, 4, 512, 512)}[route]
    k = 1 if route == "gather" else 3
    torch.manual_seed(B + hw)
    x = bf(torch.randn(B, hw, hw, C, device=DEV))
    dy = bf(torch.randn(B, hw, hw, N, device=DEV))
    acc = torch.zeros(k * k * C, N, device=DEV)
    if route == "gather":
        s = ops.conv_shape(B, hw, hw, C, N, 1, 1, 1, 0)
        _twice(lambda: ops.conv_wgrad(x, dy, acc, s), [acc])
    else:
        _twice(lambda: ops.conv_halo_wgrad(x, dy, acc, B, hw, hw, C, N, 3), [acc])


def test_sensor_and_embedding_grads_are_deterministic(hb):
    from habitat_lab_b200 import ops

    torch.manual_seed(5)
    B = 65536
    x = torch.randn(B, 2, device=DEV) * 3
    rows = torch.randperm(B, device=DEV).to(torch.int32)
    d_out = torch.randn(B, 96, device=DEV)
    d_w, d_b = torch.zeros(32, 3, device=DEV), torch.zeros(32, device=DEV)
    _twice(lambda: ops.sensor_linear_bwd(x, rows, 1, d_out, 0, 32, d_w, d_b), [d_w, d_b])
    idx = torch.randint(0, 6, (B,), device=DEV)
    masks = torch.rand(B, device=DEV) > 0.1
    d_table = torch.zeros(7, 32, device=DEV)
    _twice(lambda: ops.index_embed_bwd(idx, None, masks, d_out, 32, d_table, B), [d_table])


# ---------------------------------------------------------------------------------------------
# end to end: the same minibatch twice from the same state gives the same bits (configs #1, #3, #4)
# ---------------------------------------------------------------------------------------------
def _config_policy(hb, config):
    from habitat_lab_b200 import synthetic as syn

    if config == 1:
        import numpy as np
        from habitat_lab_b200.common import spaces
        from habitat_lab_b200.rl.policy import PointNavBaselinePolicy

        obs_space = spaces.Dict({"depth": spaces.Box(0.0, 1.0, (128, 128, 1), np.float32),
                                 "pointgoal_with_gps_compass": spaces.Box(-1e9, 1e9, (2,), np.float32)})
        act_space = spaces.Discrete(4)
        return PointNavBaselinePolicy(obs_space, act_space, hidden_size=512), obs_space, act_space, 4
    if config == 3:
        obs_space, act_space = syn.objectnav_spaces(256, 256, 6, 21)
        pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=1, rnn_type="GRU",
                                      resnet_baseplanes=32, backbone="resnet50", normalize_visual_inputs=True)
        return pol, obs_space, act_space, 6
    obs_space, act_space = syn.imagenav_spaces(256, 256, 4)
    pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=2, rnn_type="LSTM",
                                  resnet_baseplanes=32, backbone="resneXt50", normalize_visual_inputs=True)
    return pol, obs_space, act_space, 4


@pytest.mark.parametrize("config", [1, 3, 4])
def test_loss_and_backward_is_run_to_run_identical(hb, config):
    from habitat_lab_b200.synthetic import fill_rollout_

    torch.manual_seed(config)
    pol, obs_space, act_space, A = _config_policy(hb, config)
    pol.to(DEV).train()
    T, N = 16, 16   # 256 frames
    st = hb.RolloutStorage(T, N, obs_space, act_space, pol)
    st.to(DEV)
    nv = fill_rollout_(st, seed=config, observation_space=obs_space if config != 1 else None, n_actions=A)
    st.compute_returns(nv, True, 0.99, 0.95)
    ppo = hb.PPO(pol, clip_param=0.2, ppo_epoch=1, num_mini_batch=1, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4,
                 eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True, use_normalized_advantage=False)
    adv = ppo.get_advantages(st)
    sd = {k: v.clone() for k, v in pol.state_dict().items()}   # running mean / var buffers included
    runs = []
    for _ in range(2):
        pol.load_state_dict(sd)
        torch.manual_seed(77)
        batch = next(iter(st.data_generator(adv, 1)))
        m = pol.loss_and_backward(batch, 0.2, 0.5, 0.01, True).clone()
        torch.cuda.synchronize()
        runs.append((m, {n: p.grad.clone() for n, p in pol.named_parameters() if p.grad is not None}))
    (m1, g1), (m2, g2) = runs
    assert torch.equal(m1, m2)
    assert g1.keys() == g2.keys() and len(g1) > 0
    differ = [n for n in g1 if not torch.equal(g1[n], g2[n])]
    assert not differ, f"gradients differ run to run: {differ}"
