"""Halo convolutions of the resnet18 encoder at 4096 frames: the 3x3 stride-1 layers (forward, dgrad, weight gradient)
and the space-to-depth stem (forward, weight gradient)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
hb.load()
B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096


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


for H, C in ((32, 32), (16, 64)):
    torch.manual_seed(0)
    x = torch.randn(B, H, H, C, device=dev).half()
    dy = torch.randn(B, H, H, C, device=dev).bfloat16()
    w = torch.randn(C, C, 3, 3, device=dev) * 0.05
    wh = torch.empty(9 * C * C, device=dev, dtype=torch.float16)
    wt = torch.empty(9 * C * C, device=dev, dtype=torch.bfloat16)
    ops.pack_halo_weight(w, wh, C, C, 3, 0)
    ops.pack_halo_weight(w, wt, C, C, 3, 1)
    y = torch.empty_like(x)
    dx = torch.empty_like(dy)
    st = torch.zeros(B, 16, 2, device=dev, dtype=torch.float64)
    flop = 2.0 * B * H * H * C * C * 9
    tf = timed(lambda: ops.conv_halo(x, wh, y, B, H, H, C, C, 3, 0, gn_stats=st, gn_groups=16))
    td = timed(lambda: ops.conv_halo(dy, wt, dx, B, H, H, C, C, 3, 1))
    print(f"{C}ch {H}x{H} B={B}: fwd {tf:7.1f} us ({flop / tf / 1e6:6.1f} TF/s)  dgrad {td:7.1f} us "
          f"({flop / td / 1e6:6.1f} TF/s)")

# stem forward (7x7 s2 as 4x4 s1 over the space-to-depth input, 16 -> 32 channels @ 64x64)
x = torch.randn(B, 64, 64, 16, device=dev).half()
w = torch.randn(32, 4, 7, 7, device=dev) * 0.05
wh = torch.empty(16 * 16 * 32, device=dev, dtype=torch.float16)
ops.pack_halo_weight(w, wh, 16, 32, 4, 2)
y = torch.empty(B, 64, 64, 32, device=dev, dtype=torch.float16)
st = torch.zeros(B, 16, 2, device=dev, dtype=torch.float64)
t = timed(lambda: ops.conv_halo(x, wh, y, B, 64, 64, 16, 32, 4, 0, gn_stats=st, gn_groups=16))
t0 = timed(lambda: ops.conv_halo(x, wh, y, B, 64, 64, 16, 32, 4, 0))
print(f"stem 64x64 B={B}: fwd {t:7.1f} us   (without the GroupNorm sums: {t0:7.1f} us)")

# weight gradients (x halo and dy tile by TMA)
for H, C in ((32, 32), (16, 64)):
    x = torch.randn(B, H, H, C, device=dev).bfloat16()
    dy = torch.randn(B, H, H, C, device=dev).bfloat16()
    acc = torch.zeros(9 * C, C, device=dev)
    t = timed(lambda: ops.conv_halo_wgrad(x, dy, acc, B, H, H, C, C, 3))
    print(f"{C}ch {H}x{H} B={B} wgrad: {t:7.1f} us")
x = torch.randn(B, 64, 64, 16, device=dev).bfloat16()
dy = torch.randn(B, 64, 64, 32, device=dev).bfloat16()
acc = torch.zeros(16 * 16, 32, device=dev)
t = timed(lambda: ops.conv_halo_wgrad(x, dy, acc, B, 64, 64, 16, 32, 4))
print(f"stem 16ch(s2d) 64x64 B={B} wgrad: {t:7.1f} us")
