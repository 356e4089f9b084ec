"""One forward + one dgrad launch of a halo conv for ncu: `python tools/halo_probe.py C H`."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402

C, H = int(sys.argv[1]), int(sys.argv[2])
B = 4096
dev = torch.device("cuda:0")
hb.load()
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
for _ in range(2):
    ops.conv_halo(x, wh, y, B, H, H, C, C, 3, 0, gn_stats=st, gn_groups=16)
    ops.conv_halo(dy, wt, dx, B, H, H, C, C, 3, 1)
torch.cuda.synchronize()
torch.cuda.profiler.start()
ops.conv_halo(x, wh, y, B, H, H, C, C, 3, 0, gn_stats=st, gn_groups=16)
ops.conv_halo(dy, wt, dx, B, H, H, C, C, 3, 1)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
