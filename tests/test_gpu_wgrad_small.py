"""The small-image weight gradient (`conv_wgrad_small_ws_kernel`, the 8x8 / 4x4 path of hb200_conv_halo_wgrad)
against float64, at config #2's 4096-frame shapes and at every 8x8 / 4x4 layer configs #3 / #4 send to it.

Reference: dw[(r*3+s)*Ci + ci][co] = sum over frames and output pixels of x[ci] (tap-shifted, zero padded) * dy[co],
evaluated in float64 (unfold + matmul) on the same bf16 operands the kernel reads, so every product is exact in both.

Bar, per element: |kernel - reference| <= 2 * L * 2^-24 * sum |x * dy|, the first-order bound of L roundings in fp32
along the longest chain of additions an element's terms go through (factor 2: the tensor core's fp32 accumulation is
not round-to-nearest).  L restates the launcher: a worker adds 8 K16 MMA results per 16 x 8-pixel tile (16 / H frames;
plus up to 8 roundings inside one MMA) over ceil(tiles / workers) tiles, then reduce_partials adds the workers' partials (at most
`workers` additions along any chain, +1 into the caller's accumulator).  The bar is shown tight by perturbed references
that must miss it: the horizontal taps s = 0 and 2 exchanged (every case), and the ragged last tile's frame dropped
(the small ragged cases).
"""
import pytest
import torch
import torch.nn.functional as F

DEV = "cuda"
U32 = 2.0 ** -24
NUM_SMS = 132
COLS = 128   # output channels per CTA slice

# (B, H = W, Ci, Co): config #2 at 4096 frames (layer3, layer4, compression), ragged B (a tile holds 4 / 2 frames),
# the smallest Ci = 32, and a 64-frame minibatch
CONFIG2 = [(4096, 8, 128, 128), (4096, 4, 256, 256), (4096, 4, 256, 128)]
EDGE = [(4093, 4, 256, 256), (7, 4, 32, 128), (5, 8, 32, 256), (64, 8, 96, 128), (1, 4, 64, 384)]
# the 8x8 / 4x4 weight gradients configs #3 / #4 route here (test_engine_shapes_are_covered keeps this list complete)
DEEP = [(4096, 8, 128, 128), (4096, 4, 256, 256), (4096, 4, 1024, 128), (4096, 8, 256, 256), (4096, 4, 512, 512)]


def _workers(B, H, Ci, Co):
    nimg = 16 // H
    ntiles = -(-B // nimg)
    slices = -(-Ci // 64) * 3 * (Co // COLS)
    return ntiles, max(1, min(ntiles, NUM_SMS // slices))


def chain_length(B, H, Ci, Co):
    ntiles, workers = _workers(B, H, Ci, Co)
    return 8 * (-(-ntiles // workers)) + 8 + workers + 1


def reference(x, dy, chunk=256):
    """x [B, Ci, H, W], dy [B, Co, H, W] (float64 values of bf16 operands) -> (dw, sum |x * dy|), both [9 * Ci, Co]"""
    B, Ci = x.shape[:2]
    Co = dy.shape[1]
    dw = torch.zeros(Co, Ci * 9, dtype=torch.float64, device=x.device)
    sa = torch.zeros_like(dw)
    for b0 in range(0, B, chunk):
        xu = F.unfold(x[b0:b0 + chunk], 3, padding=1)   # [b, Ci*9 (ci, r, s), HW]
        d = dy[b0:b0 + chunk].flatten(2)                  # [b, Co, HW]
        dw += torch.matmul(d, xu.transpose(1, 2)).sum(0)
        sa += torch.matmul(d.abs(), xu.abs().transpose(1, 2)).sum(0)

    def rows(m):   # [Co, (ci, r, s)] -> [(r, s, ci), Co]
        return m.view(Co, Ci, 3, 3).permute(2, 3, 1, 0).reshape(9 * Ci, Co)

    return rows(dw), rows(sa)


def swap_s(m, Ci):
    """the reference with the horizontal taps s = 0 and s = 2 exchanged"""
    v = m.view(3, 3, Ci, -1)
    return v[:, [2, 1, 0]].reshape(m.shape)


def run(ops, xb, dyb, B, H, Ci, Co):
    acc = torch.zeros(9 * Ci, Co, device=DEV)
    ops.conv_halo_wgrad(xb, dyb, acc, B, H, H, Ci, Co, 3)
    return acc


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("B,H,Ci,Co", CONFIG2 + EDGE + [s for s in DEEP if s not in CONFIG2])
def test_wgrad_small_vs_float64(hb, B, H, Ci, Co):
    from habitat_lab_b200 import ops

    assert ops.conv_halo_wgrad_supported(Ci, Co, 3, H, H) and not ops.conv_halo_supported(Ci, Co, 3, H, H)
    torch.manual_seed(B * 7 + H * 3 + Ci + Co)
    xb = torch.randn(B, H, H, Ci, device=DEV).bfloat16()   # NHWC, as the engine stores the bf16 twins
    dyb = torch.randn(B, H, H, Co, device=DEV).bfloat16()
    acc = run(ops, xb, dyb, B, H, Ci, Co)
    acc2 = run(ops, xb, dyb, B, H, Ci, Co)
    torch.cuda.synchronize()
    assert torch.equal(acc, acc2), "two calls must give bit-identical accumulators"

    x64 = xb.double().permute(0, 3, 1, 2)
    dy64 = dyb.double().permute(0, 3, 1, 2)
    ref, sabs = reference(x64, dy64)
    bar = 2 * chain_length(B, H, Ci, Co) * U32 * sabs
    ratio = ((acc.double() - ref).abs() / bar).max().item()
    assert ratio <= 1.0, f"worst error / bar = {ratio:.3g}"
    # guards: each perturbed reference must miss the bar
    miss = ((acc.double() - swap_s(ref, Ci)).abs() / bar).max().item()
    assert miss > 10.0, f"exchanged horizontal taps only reach {miss:.3g} x the bar"
    nimg = 16 // H
    if B % nimg and B < 64:
        ref_d, _ = reference(x64[:-1], dy64[:-1])
        miss = ((acc.double() - ref_d).abs() / bar).max().item()
        assert miss > 10.0, f"dropping the ragged tile's last frame only reaches {miss:.3g} x the bar"


@pytest.mark.gpu
def test_wgrad_small_accumulates_into_caller(hb):
    """the partial sums are added to the caller's accumulator, not written over it"""
    from habitat_lab_b200 import ops

    B, H, Ci, Co = 9, 4, 64, 128
    torch.manual_seed(3)
    xb = torch.randn(B, H, H, Ci, device=DEV).bfloat16()
    dyb = torch.randn(B, H, H, Co, device=DEV).bfloat16()
    acc = run(ops, xb, dyb, B, H, Ci, Co)
    acc_twice = acc.clone()
    ops.conv_halo_wgrad(xb, dyb, acc_twice, B, H, H, Ci, Co, 3)
    torch.cuda.synchronize()
    torch.testing.assert_close(acc_twice, 2 * acc, rtol=1e-6, atol=0)


def _small_image_wgrads(config):
    import habitat_lab_b200 as hb
    from habitat_lab_b200 import synthetic as syn
    from habitat_lab_b200.rl.resnet_policy import EncoderEngine, ResNetEncoder

    spaces, backbone = {2: (syn.pointnav_spaces(256, 256), "resnet18"),
                        3: (syn.objectnav_spaces(256, 256, 6, 21), "resnet50"),
                        4: (syn.imagenav_spaces(256, 256, 4), "resneXt50")}[config]
    pol = hb.PointNavResNetPolicy(*spaces, hidden_size=512, num_recurrent_layers=1, rnn_type="GRU",
                                  resnet_baseplanes=32, backbone=backbone, normalize_visual_inputs=True)
    shapes = set()
    for enc in [m for m in pol.modules() if isinstance(m, ResNetEncoder)]:
        for c in EncoderEngine(enc, allow_s2d=False).convs:
            if c.halo_w and not c.halo and c.in_hw[0] in (4, 8):
                shapes.add((c.in_hw[0], c.ci, c.co))
    return shapes


@pytest.mark.parametrize("config", [2, 3, 4])
def test_engine_shapes_are_covered(config):
    """every 8x8 / 4x4 weight gradient the engine builds is one of the shapes tested above"""
    tested = {(H, Ci, Co) for _, H, Ci, Co in CONFIG2 + DEEP}
    shapes = _small_image_wgrads(config)
    assert shapes, f"config #{config} has no small-image weight gradient"
    assert shapes <= tested, f"untested small-image weight gradients of config #{config}: {sorted(shapes - tested)}"
