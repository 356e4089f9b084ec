"""Launch shapes of the persistent im2col-TMA convolution (conv_igemm_kernel<MODE, SPLIT_N>) and run-to-run identity.

The kernel takes the learner-sized stride-1 forward and data-gradient launches that gather whole 64-channel chunks.
Its grid is one CTA per SM (132); a CTA tile is 256 pixels x 128 channels when the output has 128 channels (the two
consumer warpgroups split the pixels) and 128 x 256 from 256 channels up (they split the channels).  The cases put the
tile count at exactly one and two per SM, one either side of a multiple of the grid, below the grid, odd (the last CTA
of the grid has a tile its neighbour lacks), and end in a ragged tile inside a frame (12 x 12 and 12 x 10 frames put
tile boundaries mid-frame).  The stride-2 block entries next to them stay on the gather kernel (parity classes for the
data gradient); data gradients run with and without the residual addend.

Each result is compared with an fp32 convolution of the same rounded operands (tolerances as in test_gpu_kernels.py),
and a second launch on the same inputs must give bit-identical outputs and GroupNorm statistics.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

DEV = "cuda"


def bf(x):
    return x.to(torch.bfloat16)


def hf(x):
    return x.to(torch.float16)


def nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


def nchw(x_nhwc):
    return x_nhwc.permute(0, 3, 1, 2).contiguous()


def _check_stats(stats, y_ref, B, G):
    yg = y_ref.reshape(B, G, -1)
    torch.testing.assert_close(stats[..., 0].float(), yg.sum(-1), rtol=1e-3, atol=2e-2)
    torch.testing.assert_close(stats[..., 1].float(), (yg * yg).sum(-1), rtol=1e-3, atol=2e-2)


WS_CASES = [
    # B, H, W, Ci, Co, k, stride, pad        CTA tiles of the forward (256 x 128 at Co = 128, else 128 x 256)
    (528, 8, 8, 128, 128, 3, 1, 1),          # layer3: 132 = one per SM
    (1056, 8, 8, 128, 128, 3, 1, 1),         # 264 = two per SM
    (532, 8, 8, 128, 128, 3, 1, 1),          # 133: one past the grid, odd
    (524, 8, 8, 128, 128, 3, 1, 1),          # 131: one short of the grid, odd
    (200, 8, 8, 128, 128, 3, 1, 1),          # 50: fewer than the grid
    (265, 8, 8, 128, 128, 3, 1, 1),          # 67: the last tile's second 128 rows are past the end
    (150, 12, 12, 128, 128, 3, 1, 1),        # 85 (84.4): ragged last tile inside a frame, tiles cross frames
    (131, 12, 10, 128, 128, 3, 1, 1),        # 62 (61.4): non-square frames
    (1056, 4, 4, 256, 256, 3, 1, 1),         # layer4, channels split between the consumers: 132
    (1064, 4, 4, 256, 256, 3, 1, 1),         # 133
    (1048, 4, 4, 256, 256, 3, 1, 1),         # 131
    (600, 4, 4, 256, 128, 3, 1, 1),          # compression conv: 38 (37.5), ragged
    (300, 4, 4, 256, 512, 3, 1, 1),          # two 256-wide column tiles per row tile: 76
    (300, 8, 8, 128, 256, 1, 1, 0),          # 1x1 stride 1: 150
    (300, 16, 16, 64, 128, 3, 2, 1),         # stride-2 entry of layer3: the gather kernel, beside the new one's launches
    (300, 16, 16, 64, 128, 1, 2, 0),         # its 1x1 stride-2 downsample
    (300, 8, 8, 128, 256, 3, 2, 1),          # stride-2 entry of layer4
]


@pytest.mark.parametrize("with_addend", [True, False], ids=["addend", "no_addend"])
@pytest.mark.parametrize("case", WS_CASES)
def test_conv_igemm_ws(hb, case, with_addend):
    from habitat_lab_b200 import ops

    B, H, W, ci, co, k, stride, pad = case
    G = 16
    torch.manual_seed(sum(case))
    x = torch.randn(B, ci, H, W, device=DEV)
    w = torch.randn(co, ci, k, k, device=DEV) * (1.0 / math.sqrt(ci * k * k))
    xb, wb, wh_ = hf(x).float(), bf(w).float(), hf(w).float()
    y_ref = F.conv2d(xb, wh_, stride=stride, padding=pad)
    s = ops.conv_shape(B, H, W, ci, co, k, k, stride, pad)
    x_nhwc = hf(nhwc(x))
    wp, wt = ops.pack_conv_weight(w, ci, want_t=True)
    dy = torch.randn_like(y_ref)
    dyb, dy_nhwc = bf(dy).float(), bf(nhwc(dy))
    dx_ref = torch.nn.grad.conv2d_input(xb.shape, wb, dyb, stride=stride, padding=pad)
    addend = bf(torch.randn(B, H, W, ci, device=DEV)) if with_addend else None
    runs = []
    for _ in range(2):
        y = torch.full((B, s.ho, s.wo, co), float("nan"), device=DEV, dtype=torch.float16)
        stats = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
        ops.conv_fwd(x_nhwc, wp, y, s, stats, G)
        dx = torch.full((B, H, W, ci), float("nan"), device=DEV, dtype=torch.bfloat16)
        ops.conv_dgrad(dy_nhwc, wt, dx, s, addend=addend)
        torch.cuda.synchronize()
        runs.append((y, stats, dx))
    y, stats, dx = runs[0]
    torch.testing.assert_close(nchw(y.float()), y_ref, rtol=2e-3, atol=2e-3)
    _check_stats(stats, y_ref, B, G)
    dx_want = dx_ref + nchw(addend.float()) if with_addend else dx_ref
    torch.testing.assert_close(nchw(dx.float()), dx_want, rtol=1e-2, atol=2e-2 * max(1.0, dx_ref.abs().max().item()))
    assert torch.equal(runs[0][0].view(torch.uint8), runs[1][0].view(torch.uint8))
    assert torch.equal(runs[0][1], runs[1][1])
    assert torch.equal(runs[0][2].view(torch.uint8), runs[1][2].view(torch.uint8))
