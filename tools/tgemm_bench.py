"""TF32 dense layers of config #2 (visual_fc, LSTM input projections: forward, data gradient, weight gradient) through
hb200_tgemm: CUDA-event time per launch and TFLOP/s."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
hb.load()
torch.manual_seed(0)
M = int(sys.argv[1]) if len(sys.argv) > 1 else 4096


def timed(fn, n=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


for name, N, K in (("visual_fc", 512, 2048), ("lstm_l0_ih", 2048, 576), ("lstm_l1_ih", 2048, 512)):
    x = torch.randn(M, K, device=dev)
    w = torch.randn(N, K, device=dev) * 0.02
    b = torch.randn(N, device=dev)
    out = torch.empty(M, N, device=dev)
    dy = torch.randn(M, N, device=dev)
    dx = torch.empty(M, K, device=dev)
    dw = torch.zeros(N, K, device=dev)
    t_f = timed(lambda: ops.linear_fwd(x, w, b, out, relu=True, tf32=True))
    t_d = timed(lambda: ops.linear_bwd_input(dy, w, dx, tf32=True))
    t_w = timed(lambda: ops.linear_bwd_weight(dy, x, dw, accumulate=True, tf32=True))
    fl = 2.0 * M * N * K
    print(f"{name:11s} M={M} N={N} K={K}: fwd {t_f * 1e3:7.1f} us ({fl / t_f / 1e9:6.1f} TF/s)  "
          f"dgrad(+transpose) {t_d * 1e3:7.1f} us  wgrad(+transposes) {t_w * 1e3:7.1f} us")
