"""CPU pins of the index algebra behind the warp-specialised conv_igemm_kernel<MODE, SPLIT_N> (csrc/conv.cu; no GPU).

The kernel's A operand is one TMA im2col box per K chunk (one filter tap x 64 channels).  As the PTX ISA defines the
im2col mode, the box walks `pixelsPerColumn` pixels through the map's bounding box of window origins -- W innermost,
then H, then N, each spatial step the map's element stride, wrapping from the last origin of a dimension to its lower
corner -- starting from the origin given in the instruction, and reads each pixel's channels at origin + the im2col
offsets.  Coordinates outside the tensor (padding, or frames past the batch for a ragged last tile) read zeros.

`launch_params` restates what `launch_igemm_ws` / the producer compute (corners, element strides, the first row's
origin, the tap offsets), `im2col_box` emulates the traversal, and both are checked against F.unfold -- and, as a GEMM
with the packed weight's chunk order, against the convolution / data gradient -- for the launch shapes of configs
#2-#4: forward at stride 1 (the launches the kernel takes) and stride 2 (which the map supports through its element
strides), and stride-1 dgrad as a forward conv over dy with the flipped filter.  Tiles cross frame boundaries and the
last one is ragged."""
import pytest
import torch
import torch.nn.functional as F

CHUNK = 64   # channels per pixel of one box (128 bytes of bf16: one 128-byte-swizzle row)


def launch_params(mode, src_h, src_w, out_h, out_w, k, stride, pad):
    """(lower corner, upper corner, element step) per spatial dim {W, H}, as launch_igemm_ws computes them"""
    step = stride if mode == 0 else 1
    lo = -pad if mode == 0 else -(k - 1 - pad)
    lower = (lo, lo)
    upper = (lo + (out_w - 1) * step - (src_w - 1), lo + (out_h - 1) * step - (src_h - 1))
    return lower, upper, step


def tap_offsets(mode, k, r, s):
    """im2col offsets {W, H} of filter tap (r, s): the forward reads origin + (s, r), dgrad origin + (k-1-s, k-1-r)"""
    return (s, r) if mode == 0 else (k - 1 - s, k - 1 - r)


def im2col_box(src, lower, upper, step, start, offs, c0, pixels):
    """src: [B, H, W, C] (NHWC).  The `pixels` x CHUNK box that one im2col load deposits (before the swizzle)."""
    B, H, W, _ = src.shape
    assert -128 <= min(lower + upper) and max(lower + upper) <= 127   # rank-4 corner range of cuTensorMapEncodeIm2col
    hi_w, hi_h = W - 1 + upper[0], H - 1 + upper[1]
    n, h, w = start
    out = torch.zeros(pixels, CHUNK, dtype=src.dtype)
    for p in range(pixels):
        ih, iw = h + offs[1], w + offs[0]
        if 0 <= n < B and 0 <= ih < H and 0 <= iw < W:
            out[p] = src[n, ih, iw, c0:c0 + CHUNK]
        w += step
        if w > hi_w:
            w = lower[0]
            h += step
            if h > hi_h:
                h = lower[1]
                n += 1
    return out


def kernel_a_operand(mode, src, out_h, out_w, k, stride, pad, rows_per_tile):
    """[tiles * rows_per_tile, taps * C] as the kernel's A tiles hold it, K in the packed weight's (tap, channel) order"""
    B, SH, SW, C = src.shape
    assert C % CHUNK == 0
    lower, upper, step = launch_params(mode, SH, SW, out_h, out_w, k, stride, pad)
    M = B * out_h * out_w
    tiles = (M + rows_per_tile - 1) // rows_per_tile
    hw = out_h * out_w
    rows = []
    for t in range(tiles):
        m0 = t * rows_per_tile
        ob, rem = divmod(m0, hw)
        oh, ow = divmod(rem, out_w)
        start = (ob, oh * step + lower[1], ow * step + lower[0])   # the producer's first-row origin
        chunks = []
        for c in range(k * k * C // CHUNK):
            tap, c0 = divmod(c * CHUNK, C)
            r, s = divmod(tap, k)
            chunks.append(im2col_box(src, lower, upper, step, start, tap_offsets(mode, k, r, s), c0, rows_per_tile))
        rows.append(torch.cat(chunks, 1))
    return torch.cat(rows, 0), M


def unfold_tap_major(x_nchw, k, stride, pad):
    """F.unfold -> [pixels, (r, s, c)]"""
    B, C = x_nchw.shape[:2]
    u = F.unfold(x_nchw, k, padding=pad, stride=stride)              # [B, (c, r, s), L]
    u = u.view(B, C, k * k, -1).permute(0, 3, 2, 1)                 # [B, L, (r, s), c]
    return u.reshape(-1, k * k * C)


# (B, H, W, C, N, k, stride, pad): spatial shapes of the launches the kernel takes in configs #2-#4 (ResNet18 /
# ResNet50 / ResNeXt50 encoders on 128 x 128 after the input pooling: 32 / 16 / 8 / 4-pixel stages, the 3x3 compression
# conv), at small batches with channel counts cut to two 64-channel chunks; odd frames put tile edges mid-frame
SHAPES = [
    (5, 8, 8, 128, 128, 3, 1, 1),     # layer3 3x3 (ResNet18), 3x3 of the ResNet50 layer3 blocks
    (9, 4, 4, 128, 256, 3, 1, 1),     # layer4 3x3, compression conv
    (3, 16, 16, 64, 128, 3, 2, 1),    # stride-2 entry of layer3
    (3, 16, 16, 64, 128, 1, 2, 0),    # its 1x1 downsample
    (5, 8, 8, 128, 256, 3, 2, 1),     # stride-2 entry of layer4
    (5, 8, 8, 128, 256, 1, 2, 0),     # its 1x1 downsample
    (2, 32, 32, 128, 256, 1, 2, 0),   # ResNet50 layer2 downsample
    (2, 16, 16, 128, 128, 3, 2, 1),   # ResNet50 layer3 3x3 stride 2 (conv2 of the first bottleneck)
    (2, 16, 16, 64, 256, 1, 1, 0),    # ResNet50 bottleneck 1x1 expansions / reductions
    (3, 8, 8, 128, 128, 1, 1, 0),
    (7, 4, 4, 128, 256, 1, 1, 0),
    (3, 12, 12, 128, 128, 3, 1, 1),   # frames that are not a whole number of 128-row tiles
    (3, 12, 10, 64, 128, 3, 1, 1),
]


@pytest.mark.parametrize("rows_per_tile", [256, 128], ids=["split_m", "split_n"])
@pytest.mark.parametrize("shape", SHAPES)
def test_forward_box_is_unfold(shape, rows_per_tile):
    B, H, W, C, N, k, stride, pad = shape
    torch.manual_seed(sum(shape))
    x = torch.randn(B, C, H, W, dtype=torch.float64)
    w = torch.randn(N, C, k, k, dtype=torch.float64)
    ho, wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    a, M = kernel_a_operand(0, x.permute(0, 2, 3, 1).contiguous(), ho, wo, k, stride, pad, rows_per_tile)
    assert torch.equal(a[:M], unfold_tap_major(x, k, stride, pad))
    assert not a[M:].any()   # rows past the batch read the zero fill (and are not stored)
    wk = w.permute(0, 2, 3, 1).reshape(N, -1)                         # forward image: [co][(r, s, ci)]
    y = (a[:M] @ wk.t()).view(B, ho, wo, N).permute(0, 3, 1, 2)
    torch.testing.assert_close(y, F.conv2d(x, w, stride=stride, padding=pad), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("rows_per_tile", [256, 128], ids=["split_m", "split_n"])
@pytest.mark.parametrize("shape", [s for s in SHAPES if s[6] == 1])
def test_stride1_dgrad_box_is_unfold_of_flipped_taps(shape, rows_per_tile):
    B, H, W, C, N, k, stride, pad = shape
    torch.manual_seed(sum(shape) + 1)
    w = torch.randn(N, C, k, k, dtype=torch.float64)
    ho, wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    dy = torch.randn(B, N, ho, wo, dtype=torch.float64)
    # dgrad gathers dy (N channels) and writes dx rows (H x W pixels)
    a, M = kernel_a_operand(1, dy.permute(0, 2, 3, 1).contiguous(), H, W, k, 1, pad, rows_per_tile)
    u = unfold_tap_major(dy, k, 1, k - 1 - pad).view(M, k, k, N)
    assert torch.equal(a[:M].view(M, k, k, N), u.flip(1, 2))   # tap (r, s) reads unfold tap (k-1-r, k-1-s)
    assert not a[M:].any()
    wt = w.permute(2, 3, 0, 1).reshape(-1, C)                          # transposed image: [(r, s, co)][ci]
    dx = (a[:M] @ wt).view(B, H, W, C).permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_input((B, C, H, W), w, dy, stride=1, padding=pad)
    torch.testing.assert_close(dx, ref, rtol=1e-12, atol=1e-12)


def test_corners_of_the_learner_shapes():
    # layer3 3x3 pad 1: origins -1..6 on 8 pixels; stride 2 from 16: -1, 1, .., 13 (upper -2 from the last element 15)
    assert launch_params(0, 8, 8, 8, 8, 3, 1, 1) == ((-1, -1), (-1, -1), 1)
    assert launch_params(0, 16, 16, 8, 8, 3, 2, 1) == ((-1, -1), (-2, -2), 2)
    assert launch_params(0, 16, 16, 8, 8, 1, 2, 0) == ((0, 0), (-1, -1), 2)
    # stride-1 dgrad: lower corner -(k-1-pad)
    assert launch_params(1, 4, 4, 4, 4, 3, 1, 1) == ((-1, -1), (-1, -1), 1)
    assert launch_params(1, 8, 8, 8, 8, 1, 1, 0) == ((0, 0), (0, 0), 1)
