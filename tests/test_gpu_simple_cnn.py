"""GPU: BASELINE config #1 (PointNavBaselinePolicy = SimpleCNN + GRU, rl/policy.py) kernel by kernel against float64 /
exact torch restatements, then the whole minibatch against the fp32 oracle.

Three observation spaces run throughout:
  depth 128x128        conv outputs 31 -> 14 -> 12,            flatten  4608  (config #1 as benchmarked)
  RGB + depth 256x256  conv outputs 63 -> 30 -> 28,            flatten 25088  (the reference's own PointNav sensors)
  RGB 84x116           conv outputs 20x28 -> 9x13 -> 7x11,     flatten  2464  (non-square, RGB-only prep, even conv-2
                                                                               input: parity-class data gradient)
and four batches: 2 and 6 frames (the actor's env counts: few row tiles, sliced N tiles, deep cp.async ring) and 128 /
256 frames (minibatches of T = 128 with 6 envs split into 4 minibatches of 2, 2, 1, 1 envs).

Layout and dtype kernels (prep, flatten, converts, ReLU mask, transpose) must be bit-exact; the convolution epilogue is
held to the tolerance of test_gpu_kernels.py::test_conv_fwd_dgrad_wgrad; column sums to fp32 accumulation error."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"

# name -> (H, W, rgb, depth)
SPACES = {
    "depth128": (128, 128, False, True),
    "rgbd256": (256, 256, True, True),
    "rgb84x116": (84, 116, True, False),
}
BATCHES = [2, 6, 128, 256]
# SimpleCNN's three convolutions (simple_cnn.py:68-93): (Co, k, stride), padding 0, Ci = 8 (padded input) / 32 / 64
LAYERS = [(32, 8, 4), (64, 4, 2), (32, 3, 1)]


def _dims(H, W):
    dims = [(H, W)]
    for _, k, s in LAYERS:
        h, w = dims[-1]
        dims.append(((h - k) // s + 1, (w - k) // s + 1))
    return dims


def test_space_geometry():
    """the table above: conv outputs and flatten width per space (the shapes the tests below rely on)"""
    assert _dims(128, 128)[1:] == [(31, 31), (14, 14), (12, 12)] and 32 * 12 * 12 == 4608
    assert _dims(256, 256)[1:] == [(63, 63), (30, 30), (28, 28)] and 32 * 28 * 28 == 25088
    assert _dims(84, 116)[1:] == [(20, 28), (9, 13), (7, 11)] and 32 * 7 * 11 == 2464


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _assert_bits_equal(got, ref, what):
    """bit-exact, except that NaN only has to be NaN (its payload may differ)"""
    assert got.shape == ref.shape and got.dtype == ref.dtype, what
    gn, rn = torch.isnan(got), torch.isnan(ref)
    assert torch.equal(gn, rn), f"{what}: NaN positions differ ({int((gn != rn).sum())} elements)"
    diff = (_bits(got) != _bits(ref)) & ~rn
    if diff.any():
        i = int(diff.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ, first at flat index {i}: "
                             f"{got.flatten()[i].item()!r} vs {ref.flatten()[i].item()!r}")


# ---------------------------------------------------------------------------------------------
# 1. conv + bias (+ ReLU) forward: the SimpleCNN epilogue of conv_igemm_kernel
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", [0, 1, 2])
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("space", list(SPACES))
def test_conv_bias_act_fwd(hb, space, B, layer):
    """fp16 x fp16 -> fp32 implicit GEMM + per-channel bias + optional ReLU, fp16 out, vs float64 F.conv2d of the same
    fp16-rounded operands.  The bias is drawn at the scale of the convolution itself, so about half of the outputs
    are negative before the ReLU and a bias read from the wrong channel (e.g. of another N slice) moves outputs by O(1)."""
    from habitat_lab_b200 import ops

    H, W, rgb, depth = SPACES[space]
    dims = _dims(H, W)
    co, k, stride = LAYERS[layer]
    ci_real = (3 * rgb + depth) if layer == 0 else LAYERS[layer - 1][0]
    ci = 8 if layer == 0 else ci_real
    hi, wi = dims[layer]
    g = torch.Generator(device=DEV).manual_seed(1000 * layer + 10 * B + hi)
    if layer == 0:   # pixels: rgb / 255 and depth in [0, 1)
        x = torch.rand(B, ci_real, hi, wi, device=DEV, generator=g)
    else:            # post-ReLU activations
        x = torch.randn(B, ci_real, hi, wi, device=DEV, generator=g).clamp_min(0)
    w = torch.randn(co, ci_real, k, k, device=DEV, generator=g) / math.sqrt(ci_real * k * k)
    xh, wh = x.half(), w.half()
    conv64 = F.conv2d(xh.double(), wh.double(), stride=stride)
    bias = (torch.randn(co, device=DEV, generator=g) * conv64.std()).float()
    pre = conv64 + bias.double().view(1, -1, 1, 1)
    assert 0.15 < (pre < 0).double().mean().item() < 0.85

    s = ops.conv_shape(B, hi, wi, ci, co, k, k, stride, 0)
    assert (s.ho, s.wo) == dims[layer + 1]
    x_nhwc = torch.zeros(B, hi, wi, ci, device=DEV, dtype=torch.float16)
    x_nhwc[..., :ci_real] = xh.permute(0, 2, 3, 1)
    wp, _ = ops.pack_conv_weight(w, ci, want_t=False)
    for relu in (False, True):
        ref = pre.clamp_min(0) if relu else pre
        outs = []
        for _ in range(2):
            y = torch.full((B, s.ho, s.wo, co), float("nan"), device=DEV, dtype=torch.float16)
            ops.conv_bias_act_fwd(x_nhwc, wp, bias, y, s, relu)
            outs.append(y)
        torch.cuda.synchronize()
        y = outs[0]
        assert not torch.isnan(y).any(), "rows or channels left unwritten"
        _assert_bits_equal(outs[1], y, "second launch")
        got = y.permute(0, 3, 1, 2).double()
        torch.testing.assert_close(got, ref, rtol=2e-3, atol=2e-3, msg=lambda m: f"relu={relu}: {m}")
        neg = pre < -1e-2
        if relu:
            assert bool((_bits(y.permute(0, 3, 1, 2).contiguous())[neg] == 0).all()), "ReLU must give +0 where the reference is negative"
            assert bool((got[pre > 1e-2] > 0).all())
        else:
            assert bool((got[neg] < 0).all())


# ---------------------------------------------------------------------------------------------
# 3. input prep (rgb / 255 and raw depth -> fp16 NHWC, 8 channels)
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("has_rgb,has_depth", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("H,W", [(37, 53), (84, 116)])
def test_prep_plain(hb, has_rgb, has_depth, H, W):
    """bit-exact against (rgb.float() / 255).half() and depth.half() in NHWC, gathered through shuffled and repeated
    frame_rows; channels past the real ones are exactly +0.  The fp16 pack saturates on purpose (DESIGN.md section 3:
    an overflow must not become inf): depth beyond 65504 and +-inf become +-65504, NaN stays NaN."""
    from habitat_lab_b200 import ops

    rows = 9
    g = torch.Generator().manual_seed(H * W + 2 * has_rgb + has_depth)
    rgb = torch.randint(0, 256, (rows, H, W, 3), generator=g, dtype=torch.uint8)
    rgb[0, 0, :8, 0] = torch.tensor([0, 1, 127, 128, 254, 255, 3, 85], dtype=torch.uint8)
    depth = torch.rand(rows, H, W, 1, generator=g) * 10
    special = torch.tensor([65504.0, 65519.0, 65520.0, 70000.0, 1e30, float("inf"), -65520.0, -1e30, float("-inf"),
                            float("nan"), 0.0, -0.0, 6e-8, 3e-5, -1e-6, 2.0 ** -24, 1 / 3])
    depth.view(-1)[: special.numel()] = special          # frame 0
    depth[4].view(-1)[-special.numel():] = special       # the last pixels of frame 4
    frame_rows = torch.tensor([4, 0, 8, 4, 3, 3, 0, 7, 1, 4, 2], dtype=torch.int32)
    B = frame_rows.numel()
    fr = frame_rows.long()
    C = 3 * has_rgb + has_depth
    ref = torch.zeros(B, H, W, 8, dtype=torch.float16)
    if has_rgb:
        ref[..., :3] = (rgb[fr].float() / 255).half()
    if has_depth:
        ref[..., C - 1] = depth[fr][..., 0].clamp(-65504, 65504).half()   # clamp keeps NaN
        assert torch.isinf(depth[fr].half()).any()    # without the saturation these would be inf
    out = torch.full((B, H, W, 8), float("nan"), device=DEV, dtype=torch.float16)
    ops.prep_plain(rgb.to(DEV) if has_rgb else None, depth.to(DEV) if has_depth else None, frame_rows.to(DEV), H, W,
                   3 if has_rgb else 0, 1 if has_depth else 0, out)
    torch.cuda.synchronize()
    out = out.cpu()
    _assert_bits_equal(out, ref, "prep_plain")
    assert bool((_bits(out[..., C:]) == 0).all()), "padding channels must be +0"
    if has_depth:
        d = out[..., C - 1]
        assert d[1, 0, 3].item() == 65504.0 and d[1, 0, 5].item() == 65504.0 and d[1, 0, 8].item() == -65504.0
        assert math.isnan(d[1, 0, 9].item())


# ---------------------------------------------------------------------------------------------
# 4. flatten (fp16 NHWC -> f32 CHW) and its gradient (f32 CHW -> bf16 NHWC)
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [8, 32, 64, 256])
@pytest.mark.parametrize("hw", [1, 49, 144, 784, 961])
def test_layout_conversions(hb, hw, C):
    from habitat_lab_b200 import ops

    for B in (1, 7, 256):
        g = torch.Generator(device=DEV).manual_seed(hw * C + B)
        x = (torch.randn(B, hw, C, device=DEV, generator=g) * 3).half()
        out = torch.full((B, C * hw), float("nan"), device=DEV)
        ops.bf16_hwc_to_f32_chw(x, out, B, hw, C)
        d = torch.randn(B, C * hw, device=DEV, generator=g) * 3
        dout = torch.full((B, hw, C), float("nan"), device=DEV, dtype=torch.bfloat16)
        ops.f32_chw_to_bf16_hwc(d, dout, B, hw, C)
        torch.cuda.synchronize()
        _assert_bits_equal(out, x.float().permute(0, 2, 1).flatten(1), f"bf16_hwc_to_f32_chw B={B}")
        _assert_bits_equal(dout, d.view(B, C, hw).permute(0, 2, 1).bfloat16(), f"f32_chw_to_bf16_hwc B={B}")


def test_flatten_matches_nn_flatten_of_the_feature_map(hb):
    """the (c, h, w) order of nn.Flatten on SimpleCNN's last map (7 x 11 x 32, non-square) against an explicit NCHW
    tensor, and the gradient conversion as its exact inverse on bf16-representable values"""
    from habitat_lab_b200 import ops

    B, h, w, C = 3, 7, 11, 32
    y = torch.arange(B * C * h * w, device=DEV, dtype=torch.float32).view(B, C, h, w) % 2039   # fp16-exact ids
    flat = torch.empty(B, C * h * w, device=DEV)
    ops.bf16_hwc_to_f32_chw(y.permute(0, 2, 3, 1).contiguous().half(), flat, B, h * w, C)
    back = torch.empty(B, h * w, C, device=DEV, dtype=torch.bfloat16)
    ops.f32_chw_to_bf16_hwc(flat % 256, back, B, h * w, C)
    torch.cuda.synchronize()
    assert torch.equal(flat, torch.nn.Flatten()(y))
    assert torch.equal(back.float(), (y % 256).permute(0, 2, 3, 1).reshape(B, h * w, C))


# ---------------------------------------------------------------------------------------------
# 5. dtype conversions
# ---------------------------------------------------------------------------------------------
N_LARGE = 8 * (132 * 16 * 256 * 2 + 7)   # > one pass of the capped grid: the grid-stride loop runs


def _f16_inputs(n, seed):
    """every fp16 bit pattern (ties for the bf16 rounding, subnormals, max finite, +-0, +-inf, NaN), then random"""
    allp = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(max(n, 1), generator=g) * 100).half()
    m = min(n, allp.numel())
    x[:m] = allp[:m]
    return x[:n]


def _f32_inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g) * torch.exp(torch.randn(n, generator=g) * 10)
    bits = torch.randint(-2 ** 31, 2 ** 31, (4096,), generator=g, dtype=torch.int64)
    ties = ((bits & ~0xFFFF) | 0x8000).to(torch.int32).view(torch.float32)          # exactly half a bf16 step
    near = ((bits & ~0xFFFF) | 0x7FFF).to(torch.int32).view(torch.float32)          # just below a tie
    special = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 3.4028234663852886e38,
                            -3.4028234663852886e38, 3.3895313892515355e38, 3.3961775292304770e38, 65504.0, -65504.0,
                            2.0 ** -24, 2.0 ** -14, 5.9604645e-08 * 3, 1e-40, -1e-40, 1.17549435e-38, 2.0 ** -149])
    f16 = _f16_inputs(65536, seed).float()   # fp16 subnormals / max finite as fp32 values
    pool = torch.cat([special, ties, near, f16])
    m = min(n, pool.numel())
    x[:m] = pool[:m]
    return x


@pytest.mark.parametrize("n", [8, 8 * 12345, 8 * 65537, N_LARGE])
def test_dtype_conversions(hb, n):
    from habitat_lab_b200 import ops

    assert n % 8 == 0
    x16 = _f16_inputs(n, n)
    o = torch.full((n,), float("nan"), device=DEV, dtype=torch.bfloat16)
    ops.f16_to_bf16(x16.to(DEV), o)
    x32 = _f32_inputs(n, n + 1)
    o2 = torch.full((n,), float("nan"), device=DEV, dtype=torch.bfloat16)
    ops.f32_to_bf16(x32.to(DEV), o2)
    xb = _f16_inputs(n, n + 2).view(torch.int16).view(torch.bfloat16)   # every bf16 bit pattern first
    o3 = torch.full((n,), float("nan"), device=DEV)
    ops.bf16_to_f32(xb.to(DEV), o3)
    torch.cuda.synchronize()
    _assert_bits_equal(o.cpu(), x16.to(torch.bfloat16), "f16_to_bf16")
    _assert_bits_equal(o2.cpu(), x32.to(torch.bfloat16), "f32_to_bf16")
    _assert_bits_equal(o3.cpu(), xb.float(), "bf16_to_f32")


# ---------------------------------------------------------------------------------------------
# 6. ReLU backward on a column block; 7. transpose; 8. column sums
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 7, 4099])
def test_relu_bwd_column_block(hb, rows):
    """d[r, c] = 0 where !(y[r, c] > 0) for c < cols, on views into wider matrices (ld_d != ld_y, both > cols): y = 0,
    -0, NaN and negatives zero d; tiny positives (subnormal too) keep it; columns >= cols keep their bits"""
    from habitat_lab_b200 import ops

    cols, ld_d, ld_y, c0_d, c0_y = 512, 524, 518, 4, 2
    g = torch.Generator().manual_seed(rows)
    y_full = torch.randn(rows, ld_y, generator=g)
    pool = torch.tensor([0.0, -0.0, 1e-45, 1e-38, 1e-30, -1e-45, -1e-30, float("nan"), float("-inf"), float("inf"),
                         1.0, -1.0])
    pick = torch.randint(0, pool.numel(), (rows, ld_y), generator=g)
    y_full = torch.where(torch.rand(rows, ld_y, generator=g) < 0.5, pool[pick], y_full)
    d_full = torch.randn(rows, ld_d, generator=g)
    d_full[:, ::7] = float("nan")        # masked NaN gradients must become 0 as well
    y_dev, d_dev = y_full.to(DEV), d_full.to(DEV)
    ops.relu_bwd(d_dev[:, c0_d:], y_dev[:, c0_y:], cols)
    torch.cuda.synchronize()
    ref = d_full.clone()
    blk = slice(c0_d, c0_d + cols)
    ref[:, blk] = torch.where(y_full[:, c0_y:c0_y + cols] > 0, d_full[:, blk], torch.zeros(()))
    _assert_bits_equal(d_dev.cpu(), ref, "relu_bwd")
    assert torch.equal(y_dev.cpu().view(torch.int32), y_full.view(torch.int32))


TRANSPOSE_SHAPES = [(r, c) for r in (1, 31, 33, 514, 25088) for c in (1, 31, 33, 514, 25088) if r * c < 25088 * 600]


@pytest.mark.parametrize("rows,cols", TRANSPOSE_SHAPES)
def test_transpose_f32(hb, rows, cols):
    """dst[c, r] = src[r, c] for views with leading dimensions larger than the extents; everything outside the
    written [cols x rows] block keeps its NaN sentinel"""
    from habitat_lab_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(rows * 7 + cols)
    src_full = torch.randn(rows + 1, cols + 5, device=DEV, generator=g)
    dst_full = torch.full((cols + 2, rows + 3), float("nan"), device=DEV)
    src = src_full[1:, 3:3 + cols]
    dst = dst_full[1:1 + cols, 2:2 + rows]
    assert src.stride(0) > cols and dst.stride(0) > rows
    ops.transpose_f32(src, dst)
    torch.cuda.synchronize()
    assert torch.equal(dst, src.t())
    written = torch.zeros_like(dst_full, dtype=torch.bool)
    written[1:1 + cols, 2:2 + rows] = True
    assert bool(torch.isnan(dst_full[~written]).all())


@pytest.mark.parametrize("M", [1, 128, 4099])
@pytest.mark.parametrize("n_cols,width", [(512, 514), (33, 40), (1, 9)])
def test_colsum(hb, M, n_cols, width):
    """out[c] (+)= sum_r x[r, c] for c < n_cols of a wider matrix, vs float64; out[n_cols:] untouched"""
    from habitat_lab_b200 import ops

    g = torch.Generator().manual_seed(M + n_cols)
    x = torch.randn(M, width, generator=g) * torch.rand(1, width, generator=g) * 3 + 0.25
    x_dev = x.to(DEV)
    ref = x[:, :n_cols].double().sum(0)
    tol = 4e-6 * x[:, :n_cols].double().abs().sum(0) + 1e-6
    for accumulate in (False, True):
        out0 = torch.randn(n_cols + 5, generator=g)
        out0[n_cols:] = float("nan")
        out = out0.to(DEV)
        ops.colsum(x_dev, out, accumulate=accumulate, n_cols=n_cols)
        torch.cuda.synchronize()
        got = out.cpu()
        exp = ref + (out0[:n_cols].double() if accumulate else 0)
        err = (got[:n_cols].double() - exp).abs()
        assert bool((err <= tol + 1e-6 * exp.abs()).all()), (accumulate, err.max().item())
        assert bool(torch.isnan(got[n_cols:]).all())


# ---------------------------------------------------------------------------------------------
# 10. the whole policy: minibatch loss + backward, act / get_value, vs the fp32 oracle
# ---------------------------------------------------------------------------------------------
T_ROLL, N_ENVS = 128, 6
# Gradient bars of the minibatch test: (cosine of the visual encoder's tensors, cosine of the other tensors, max
# |norm ratio - 1| of any tensor).  SimpleCNN has no GroupNorm to re-centre its fp16 activations, so these were measured
# rather than taken from config #2.  Measured on one H100 80GB HBM3 (700 W power limit), worst tensor per space:
#   depth128   encoder cos 0.999978 (cnn.0.weight), others >= 0.9999995, |ratio - 1| 0.0009 (cnn.0.bias)
#   rgbd256    encoder cos 0.999955 (cnn.0.weight), others >= 0.9999995, |ratio - 1| 0.0020 (critic.fc.bias)
#   rgb84x116  encoder cos 0.999940 (cnn.0.weight), others >= 0.9999995, |ratio - 1| 0.0035 (cnn.0.bias)
# The bars leave 10x headroom on 1 - cos for the encoder, 20x for the rest and ~6x on the norm ratio.  For scale: rgb
# prepared as x / 256 instead of x / 255 (a 0.4 % input error) drops rgbd256 to 0.99987 on critic.fc.weight and moves a
# norm by 7 %.
POLICY_BARS = (0.9994, 0.99999, 0.02)


@pytest.fixture(scope="module", params=list(SPACES))
def baseline_case(hb, request):
    """PointNavBaselinePolicy on one observation space with recipe weights, a synthetic T = 128 x 6-env rollout and its
    GAE returns (oracle), all on the CPU; the policy on the GPU"""
    from habitat_lab_b200.common import spaces
    from habitat_lab_b200.rl.policy import PointNavBaselinePolicy
    from helpers import recipe_state_dict, synthetic_rollout
    from oracle import torch_oracle as O
    import numpy as np

    name = request.param
    H, W, rgb, depth = SPACES[name]
    sp = {"pointgoal_with_gps_compass": spaces.Box(-1e9, 1e9, (2,), np.float32)}
    if rgb:
        sp["rgb"] = spaces.Box(0, 255, (H, W, 3), np.uint8)
    if depth:
        sp["depth"] = spaces.Box(0.0, 1.0, (H, W, 1), np.float32)
    obs_space = spaces.Dict(sp)
    pol = PointNavBaselinePolicy(obs_space, spaces.Discrete(4), hidden_size=512)
    seed = 31 + list(SPACES).index(name)
    shapes = {k: tuple(v.shape) for k, v in pol.state_dict().items()}
    assert shapes["net.visual_encoder.cnn.6.weight"][1] == 32 * math.prod(_dims(H, W)[3])
    sd = recipe_state_dict(shapes, seed)
    pol.load_state_dict(sd)
    pol.to(DEV)
    bufs, next_value = synthetic_rollout(T_ROLL, N_ENVS, H, W, 4, 1, 512, seed, rgb=rgb, depth=depth)
    bufs["returns"] = O.compute_returns(bufs["rewards"], bufs["value_preds"], bufs["masks"], next_value, T_ROLL, True,
                                        0.99, 0.95)
    adv = O.get_advantages(bufs["returns"], bufs["value_preds"], normalize=False)
    yield dict(name=name, pol=pol, sd=sd, bufs=bufs, adv=adv)
    del pol
    torch.cuda.empty_cache()


def _to_dev(batch):
    out = {k: v.to(DEV) for k, v in batch.items() if k != "observations"}
    out["observations"] = {k: v.to(DEV).contiguous() for k, v in batch["observations"].items()}
    return out


def test_baseline_policy_minibatch_vs_oracle(hb, baseline_case):
    """loss_and_backward on the first minibatch of the 4-way split (2 envs x 128 steps = 256 frames): per-frame values
    and log-probs, the three losses, and every parameter's gradient (cosine and norm ratio) vs the fp32 oracle's
    evaluate_actions_baseline + ppo_loss on the same weights.  The oracle runs without storage emulation (DESIGN.md
    section 3: emulating the roundings is not the tighter yardstick)."""
    from helpers import gather_minibatch, minibatch_env_inds
    from oracle import torch_oracle as O

    c = baseline_case
    pol, name = c["pol"], c["name"]
    inds = minibatch_env_inds(77, N_ENVS, 4)[0]
    assert inds.numel() == 2
    ob = gather_minibatch(c["bufs"], c["adv"], inds, T_ROLL)
    pol.train()
    metrics = pol.loss_and_backward(_to_dev(ob), 0.2, 0.5, 0.01, True).cpu()
    torch.cuda.synchronize()
    last = {k: v.detach().cpu() for k, v in pol._last.items()}
    grads = {k: p.grad.detach().double().cpu().flatten() for k, p in pol.named_parameters()}

    sdr = {k: (v.clone().requires_grad_(True) if v.dtype.is_floating_point else v) for k, v in c["sd"].items()}
    obs = {k: v for k, v in ob["observations"].items()}
    value, lp, ent, hid, _ = O.evaluate_actions_baseline(obs, ob["recurrent_hidden_states"], ob["prev_actions"],
                                                         ob["masks"], ob["actions"], sdr)
    ref = O.ppo_loss(value, lp, ent, ob, 0.2, 0.5, 0.01, True)
    ref["total_loss"].backward()

    dv = (last["values"] - value.detach().view(-1)).abs().max().item()
    dlp = (last["log_probs"] - lp.detach().view(-1)).abs().max().item()
    dh = (last["hidden_out"] - hid.detach()).abs().max().item()
    losses = {k: (metrics[i].item(), ref[k].item()) for i, k in enumerate(("value_loss", "action_loss", "dist_entropy"))}
    rows = []
    for k, g in grads.items():
        r = sdr[k].grad.double().flatten()
        rows.append(((g @ r / (g.norm() * r.norm() + 1e-30)).item(), (g.norm() / (r.norm() + 1e-30)).item(), k))
    rows.sort()
    enc = [x for x in rows if "visual_encoder" in x[2]]
    rest = [x for x in rows if "visual_encoder" not in x[2]]
    print(f"\n{name}: values max diff {dv:.2e}, log-probs {dlp:.2e}, hidden {dh:.2e}, losses {losses}")
    print(f"{name}: worst encoder cos {enc[0][0]:.6f} ({enc[0][2]}), worst other cos {rest[0][0]:.6f} ({rest[0][2]}), "
          f"max |norm ratio - 1| {max(abs(x[1] - 1) for x in rows):.5f}")
    for cos, ratio, k in rows:
        print(f"  {k:45s} cos {cos:.6f} ratio {ratio:.5f}")

    assert dv < 5e-3 * max(1.0, value.abs().max().item()), dv
    assert dlp < 5e-3, dlp
    assert dh < 5e-3, dh
    for k, (a, b) in losses.items():
        assert a == pytest.approx(b, rel=1e-3, abs=2e-4), (k, a, b)
    cos_enc, cos_rest, ratio_tol = POLICY_BARS
    for cos, ratio, k in rows:
        assert cos > (cos_enc if "visual_encoder" in k else cos_rest), (k, cos)
        assert abs(ratio - 1) < ratio_tol, (k, ratio)


def test_baseline_policy_act_and_get_value_vs_oracle(hb, baseline_case):
    """the actor path at 6 envs (one rollout step, eval mode): act(deterministic=True) and get_value vs the oracle's
    values, greedy actions (where the oracle's two best logits are apart), their log-probs and the GRU state"""
    from oracle import torch_oracle as O

    c = baseline_case
    pol, b, sd = c["pol"], c["bufs"], c["sd"]
    step = 1
    obs = {k: v[step] for k, v in b["observations"].items()}
    hid, pa, mk = b["recurrent_hidden_states"][step], b["prev_actions"][step], b["masks"][step]
    pol.eval()
    dev = lambda t: t.to(DEV).contiguous()  # noqa: E731
    out = pol.act({k: dev(v) for k, v in obs.items()}, dev(hid), dev(pa), dev(mk), deterministic=True)
    val = pol.get_value({k: dev(v) for k, v in obs.items()}, dev(hid), dev(pa), dev(mk))
    torch.cuda.synchronize()
    with torch.no_grad():
        zeros = torch.zeros(N_ENVS, 1, dtype=torch.int64)
        value, _, _, hid_ref, feats = O.evaluate_actions_baseline(obs, hid, pa, mk, zeros, sd)
        logp = torch.log_softmax(F.linear(feats, sd["action_distribution.linear.weight"],
                                          sd["action_distribution.linear.bias"]), -1)
    print(f"\n{c['name']} act: values max diff {(out.values.cpu() - value).abs().max().item():.2e}, "
          f"get_value {(val.cpu() - value).abs().max().item():.2e}, "
          f"hidden {(out.rnn_hidden_states.cpu() - hid_ref).abs().max().item():.2e}")
    assert (out.values.cpu() - value).abs().max().item() < 5e-3
    assert (val.cpu() - value).abs().max().item() < 5e-3
    assert (out.rnn_hidden_states.cpu() - hid_ref).abs().max().item() < 5e-3
    top2 = logp.topk(2, dim=-1).values
    decided = (top2[:, 0] - top2[:, 1]) > 5e-3
    ref_act = logp.argmax(-1, keepdim=True)
    assert torch.equal(out.actions.cpu()[decided], ref_act[decided])
    same = (out.actions.cpu() == ref_act).view(-1)
    assert (out.action_log_probs.cpu() - logp.gather(1, out.actions.cpu()))[same].abs().max().item() < 5e-3
