"""layer2.0 of the resnet18 encoder at 4096 frames (32x32x32 -> 16x16x64 + downsample): the fused stride-2 kernels
(conv_s2.cu) against the gather kernels they replace."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
hb.load()
B, H, W, C, NA, NB, G = int(sys.argv[1]) if len(sys.argv) > 1 else 4096, 32, 32, 32, 64, 64, 16
torch.manual_seed(0)
x = torch.randn(B, H, W, C, device=dev).half()
wa = torch.randn(NA, C, 3, 3, device=dev) * 0.05
wd = torch.randn(NB, C, 1, 1, device=dev) * 0.1
wcat = torch.zeros(NA + NB, C, 3, 3, device=dev)
wcat[:NA] = wa
wcat[NA:, :, 1, 1] = wd[:, :, 0, 0]
img = torch.empty(9 * C * (NA + NB), device=dev, dtype=torch.float16)
img_t = torch.empty(9 * C * (NA + NB), device=dev, dtype=torch.bfloat16)
ops.pack_halo_weight(wcat, img, C, NA + NB, 3, 0)
ops.pack_halo_weight(wcat, img_t, NA + NB, C, 3, 1)
ya = torch.empty(B, H // 2, W // 2, NA, device=dev, dtype=torch.float16)
yb = torch.empty_like(ya)
sa = torch.zeros(B, G, 2, device=dev, dtype=torch.float64)
sb = torch.zeros_like(sa)
dya = torch.randn(B, H // 2, W // 2, NA, device=dev).bfloat16()
dyb = torch.randn(B, H // 2, W // 2, NB, device=dev).bfloat16()
dx = torch.empty(B, H, W, C, device=dev, dtype=torch.bfloat16)
s_a = ops.conv_shape(B, H, W, C, NA, 3, 3, 2, 1)
s_d = ops.conv_shape(B, H, W, C, NB, 1, 1, 2, 0)
wpa, wta = ops.pack_conv_weight(wa, C, want_t=True)
wpd, wtd = ops.pack_conv_weight(wd, C, want_t=True)


def timed(fn, n=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


def gather_fwd():
    ops.conv_fwd(x, wpa, ya, s_a, sa, G)
    ops.conv_fwd(x, wpd, yb, s_d, sb, G)


def gather_dgrad():
    ops.conv_dgrad(dya, wta, dx, s_a, addend=None)
    ops.conv_dgrad(dyb, wtd, dx, s_d, addend=dx)


print(f"B={B}: forward  fused {timed(lambda: ops.conv_s2_fwd(x, img, ya, yb, B, H, W, C, NA, NB, stats_a=sa, groups_a=G, stats_b=sb, groups_b=G)):7.1f} us"
      f"   gather (2 launches) {timed(gather_fwd):7.1f} us")
print(f"B={B}: dgrad    fused {timed(lambda: ops.conv_s2_dgrad(dya, dyb, img_t, dx, B, H, W, C, NA, NB)):7.1f} us"
      f"   gather (2 launches) {timed(gather_dgrad):7.1f} us")

xb = x.bfloat16()
acc = torch.zeros(16 * C, NA, device=dev)
acc_g = torch.zeros(9 * C, NA, device=dev)
print(f"B={B}: wgrad 3x3 s2d  {timed(lambda: ops.conv_s2_wgrad(xb, dya, acc, B, H, W, C, NA)):7.1f} us"
      f"   gather {timed(lambda: ops.conv_wgrad(xb, dya, acc_g, s_a)):7.1f} us")
