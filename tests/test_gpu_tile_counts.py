"""Tile-count edge cases of the tensor-core convolutions at the launch shapes of the learner, and run-to-run identity.

conv_halo_ws_kernel hands the tiles of a CTA alternately to two consumer warpgroups, so a CTA with an odd number of
tiles, or with a single one, leaves the second warpgroup with one tile fewer or none.  Its grid is one CTA per SM (132)
for the 32- and 64-channel layers and two per SM for the stem, so the cases put the tile count below the grid, at one
and two tiles per CTA, and one tile past a multiple of the grid.  The 16 x 8 images are one 128-pixel tile per frame.

conv_igemm_kernel runs two CTAs per SM at the full 128-wide N tile; the cases put its CTA count below the SM count
(without the narrow N slices the actor's launches get), at exactly one and two CTAs per SM, one past that, and stride-2
data gradients whose four parity classes end in partial row tiles.

Each result is compared with an fp32 convolution of the same rounded operands (tolerances as in test_gpu_kernels.py),
and a second launch on the same inputs must give bit-identical outputs and GroupNorm statistics.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

DEV = "cuda"
SMS = 132


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


HALO_TILE_CASES = [
    # B, H, W, C   (one tile per 16 x 8 frame; grid 132 CTAs)
    (7, 16, 8, 32),               # fewer tiles than SMs, one tile per CTA: warpgroup 1 idle
    (131, 16, 8, 32),             # odd, below the grid
    (SMS, 16, 8, 32),             # exactly one tile per CTA
    (2 * SMS, 16, 8, 32),         # exactly two: one per warpgroup
    (2 * SMS + 1, 16, 8, 32),     # one CTA with three tiles
    (5 * SMS + 3, 16, 8, 32),     # odd tile count per CTA (5 or 6), ring of 6 stages wraps
    (2 * SMS + 1, 16, 8, 64),     # 64 channels, 2-stage ring
    (37, 32, 32, 32),             # 296 tiles on 132 CTAs
]


@pytest.mark.parametrize("B,H,W,C", HALO_TILE_CASES)
def test_conv_halo_ws_tile_counts(hb, B, H, W, C):
    from habitat_lab_b200 import ops

    N, G = C, 16
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
    dy = torch.randn_like(y_ref)
    dyb, dy_nhwc = bf(dy).float(), bf(nhwc(dy))
    dx_ref = torch.nn.grad.conv2d_input(xb.shape, wb, dyb, padding=1)
    addend = bf(torch.randn(B, H, W, C, device=DEV))
    runs = []
    for _ in range(2):
        y = torch.full((B, H, W, N), float("nan"), device=DEV, dtype=torch.float16)
        stats = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
        ops.conv_halo(x_nhwc, wh, y, B, H, W, C, N, 3, 0, gn_stats=stats, gn_groups=G)
        dx = torch.full((B, H, W, C), float("nan"), device=DEV, dtype=torch.bfloat16)
        ops.conv_halo(dy_nhwc, wht, dx, B, H, W, N, C, 3, 1, addend=addend)
        torch.cuda.synchronize()
        runs.append((y, stats, dx))
    y, stats, dx = runs[0]
    torch.testing.assert_close(nchw(y.float()), y_ref, rtol=2e-3, atol=2e-3)
    _check_stats(stats, y_ref, B, G)
    torch.testing.assert_close(nchw(dx.float()), dx_ref + nchw(addend.float()), rtol=1e-2,
                               atol=2e-2 * max(1.0, dx_ref.abs().max().item()))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a.view(torch.uint8) if a.dtype != torch.float64 else a,
                           b.view(torch.uint8) if b.dtype != torch.float64 else b)


def test_conv_halo_stem_tile_counts(hb):
    """the stem (4x4 over the space-to-depth input, 16 -> 32 channels) on the same kernel, 2 CTAs per SM: 265 tiles"""
    from habitat_lab_b200 import ops

    B, H, W, C, N, G = 2 * 2 * SMS + 1, 16, 8, 16, 32, 16
    torch.manual_seed(3)
    x = torch.randn(B, 4, 2 * H, 2 * W, device=DEV)
    w = torch.randn(N, 4, 7, 7, device=DEV) / math.sqrt(4 * 49)
    wh = torch.empty(16 * C * N, device=DEV, dtype=torch.float16)
    ops.pack_halo_weight(w, wh, C, N, 4, 2)
    # s2d: [B, H, W, (dy, dx, c)]
    xs = hf(x).view(B, 4, H, 2, W, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, H, W, 16).contiguous()
    y_ref = F.conv2d(hf(x).float(), hf(w).float(), stride=2, padding=3)
    runs = []
    for _ in range(2):
        y = torch.full((B, H, W, N), float("nan"), device=DEV, dtype=torch.float16)
        stats = torch.zeros(B, G, 2, device=DEV, dtype=torch.float64)
        ops.conv_halo(xs, wh, y, B, H, W, C, N, 4, 0, gn_stats=stats, gn_groups=G)
        torch.cuda.synchronize()
        runs.append((y, stats))
    torch.testing.assert_close(nchw(runs[0][0].float()), y_ref, rtol=2e-3, atol=2e-3)
    _check_stats(runs[0][1], y_ref, B, G)
    assert torch.equal(runs[0][0].view(torch.uint8), runs[1][0].view(torch.uint8))
    assert torch.equal(runs[0][1], runs[1][1])


CONV_TILE_CASES = [
    # B, H, W, Ci, Co, k, stride, pad    (row tiles x N tiles of 128 = CTAs of the forward launch)
    (320, 4, 4, 256, 256, 3, 1, 1),      # 40 x 2 = 80 CTAs: fewer than SMs, full-width tiles
    (1056, 4, 4, 256, 256, 3, 1, 1),     # 132 x 2 = 264: exactly two CTAs per SM
    (528, 4, 4, 256, 256, 3, 1, 1),      # 66 x 2 = 132: exactly one
    (1064, 4, 4, 256, 256, 3, 1, 1),     # 133 x 2: one row tile past the resident grid
    (265, 8, 8, 128, 128, 3, 1, 1),      # 133 x 1: odd, 64 pixels of frames per tile
    (37, 16, 16, 64, 128, 3, 2, 1),      # stride 2: dgrad parity classes of 2368 rows, 18.5 tiles each
    (67, 8, 8, 128, 256, 3, 2, 1),       # stride 2 into layer4 shapes: classes of 1072 rows
    (67, 8, 8, 128, 256, 1, 2, 0),       # the 1x1 stride-2 downsample at the same sizes
]


@pytest.mark.parametrize("case", CONV_TILE_CASES)
def test_conv_igemm_tile_counts(hb, case):
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
    addend = bf(torch.randn(B, H, W, ci, device=DEV))
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
    torch.testing.assert_close(nchw(dx.float()), dx_ref + nchw(addend.float()), rtol=1e-2,
                               atol=2e-2 * max(1.0, dx_ref.abs().max().item()))
    assert torch.equal(runs[0][0].view(torch.uint8), runs[1][0].view(torch.uint8))
    assert torch.equal(runs[0][1], runs[1][1])
    assert torch.equal(runs[0][2].view(torch.uint8), runs[1][2].view(torch.uint8))
