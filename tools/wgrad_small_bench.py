"""Weight gradients of the 3x3 stride-1 layers on 8x8 / 4x4 images (hb200_conv_halo_wgrad's small-image path) at
4096 frames: config #2's layer3 (128 -> 128 @ 8x8), layer4 (256 -> 256 @ 4x4) and compression (256 -> 128 @ 4x4),
and the other shapes of configs #3 / #4: the ResNet50 compression (1024 -> 128 @ 4x4) and the ResNeXt50 3x3s
(256 -> 256 @ 8x8, 512 -> 512 @ 4x4).

Per shape: the whole call (weight-gradient kernel + reduce_partials) timed with CUDA events over --iters launches
after --warmup, then one profiled window (torch.profiler, CUDA activities) that splits it into the weight-gradient
kernel and the partial sums.  TF/s are algorithmic: 2 * B * H * W * Ci * Co * 9 over the time.

    python tools/wgrad_small_bench.py [--frames 4096] [--iters 50] [--warmup 10] [--json out.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402

SHAPES = [(8, 128, 128), (4, 256, 256), (4, 256, 128), (4, 1024, 128), (8, 256, 256), (4, 512, 512)]   # (H = W, Ci, Co)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wgrad_small_bench: no CUDA device")
    hb.load()
    dev = torch.device("cuda:0")
    B = args.frames
    rows = []
    for H, Ci, Co in SHAPES:
        torch.manual_seed(0)
        x = torch.randn(B, H, H, Ci, device=dev).bfloat16()
        dy = torch.randn(B, H, H, Co, device=dev).bfloat16()
        acc = torch.zeros(9 * Ci, Co, device=dev)

        def call():
            ops.conv_halo_wgrad(x, dy, acc, B, H, H, Ci, Co, 3)

        for _ in range(args.warmup):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        total_us = e0.elapsed_time(e1) / args.iters * 1e3
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                call()
            torch.cuda.synchronize()
        kern_us = red_us = 0.0
        kern_name = None
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if "reduce_partials" in ev.key:
                red_us += t / args.iters
            elif "wgrad" in ev.key:
                kern_us += t / args.iters
                kern_name = ev.key
        flop = 2.0 * B * H * H * Ci * Co * 9
        row = dict(shape=f"{Ci}->{Co} @{H}x{H}", frames=B, kernel=kern_name, total_us=round(total_us, 1),
                   wgrad_us=round(kern_us, 1), reduce_us=round(red_us, 1), wgrad_tflops=round(flop / kern_us / 1e6, 1),
                   total_tflops=round(flop / total_us / 1e6, 1))
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(device=torch.cuda.get_device_name(0), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
