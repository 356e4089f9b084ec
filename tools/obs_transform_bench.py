"""Time the fused observation transform (ResizeShortestEdge(256) + CenterCropper(256, 256) written straight into a
rollout-storage slot, one launch) against the same work done the way the reference's trainer does it on CUDA:
per key F.interpolate(img.permute(0, 3, 1, 2).float(), mode).to(dtype).permute(0, 2, 3, 1), the centre slice,
then the storage copy_.

Workloads: 480x640 raw frames, the ObjectNav sensor set of config #3 (rgb u8 x3, depth f32, semantic i32) and the
PointNav rgb-d set, at N = 4 / 32 / 64 / 256 envs.  Each point: CUDA events over enough calls for >= 1 s, three
repeats (median and spread).  GB/s uses a bytes model computed here: every input byte the window depends on,
rounded up to 32-byte sectors per row, plus the output bytes.

    python tools/obs_transform_bench.py [--n 4 32 64 256] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402
from habitat_lab_b200.common import spaces  # noqa: E402
from habitat_lab_b200.common.obs_transformers import (CenterCropper, ObsTransformPlan,  # noqa: E402
                                                      ResizeShortestEdge, apply_obs_transforms_obs_space)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
SETS = {
    "objectnav": {"rgb": (torch.uint8, 3), "depth": (torch.float32, 1), "semantic": (torch.int32, 1)},
    "pointnav": {"rgb": (torch.uint8, 3), "depth": (torch.float32, 1)},
}
H, W, SIZE = 480, 640, 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else \
        torch.cuda.get_device_name()


def model_bytes(plan, keys, n):
    """Input sectors the window reaches (per row, 32-byte granularity, rows 32-byte aligned when the pitch is) plus
    output bytes."""
    total = 0
    for k, (mode, (hr, wr), (y0, x0), (h, w)) in plan.keys.items():
        dt, c = keys[k]
        es = torch.empty((), dtype=dt).element_size()
        if mode == ops.OBS_AREA:
            r0, r1 = (y0 * H) // hr, ((y0 + h) * H + hr - 1) // hr
            c0, c1 = (x0 * W) // wr, ((x0 + w) * W + wr - 1) // wr
        elif mode == ops.OBS_NEAREST:
            sh, sw = torch.tensor(H / hr, dtype=torch.float32), torch.tensor(W / wr, dtype=torch.float32)
            rows = {min(int(torch.floor(torch.tensor(float(i), dtype=torch.float32) * sh)), H - 1)
                    for i in range(y0, y0 + h)}
            r0, r1 = 0, len(rows)
            c0 = min(int(torch.floor(torch.tensor(float(x0), dtype=torch.float32) * sw)), W - 1)
            c1 = min(int(torch.floor(torch.tensor(float(x0 + w - 1), dtype=torch.float32) * sw)), W - 1) + 1
        else:
            r0, r1, c0, c1 = y0, y0 + h, x0, x0 + w
        pitch = W * c * es
        sectors = 0
        for r in range(r0, r1):
            base = r * pitch if pitch % 32 == 0 else 0
            sectors += -(-(base + c1 * c * es) // 32) - (base + c0 * c * es) // 32
        total += n * (sectors * 32 + h * w * c * es)
    return total


def timed(fn, min_s=1.0, repeats=3):
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = 20
    while True:   # calibrate so one repeat lasts >= min_s
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= 1000 * min_s:
            break
        iters = max(iters * 2, int(iters * 1.2 * 1000 * min_s / max(ms, 1e-3)))
    out = []
    for _ in range(repeats):
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / iters)   # us per call
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[4, 32, 64, 256])
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("obs_transform_bench: no CUDA device")
    hb.load()
    dev = torch.device("cuda")
    print(f"card: {card()}")
    active = [ResizeShortestEdge(SIZE), CenterCropper(SIZE)]
    rows = []
    print(f"{'set':10s} {'N':>4s} {'MB':>8s} {'fused us':>18s} {'torch us':>18s} {'speedup':>8s} "
          f"{'fused GB/s':>10s} {'of 3.35TB/s':>11s}")
    for name, keys in SETS.items():
        raw = spaces.Dict({k: spaces.Box(0, 1, (H, W, c), torch.empty((), dtype=dt).numpy().dtype)
                           for k, (dt, c) in keys.items()})
        space = apply_obs_transforms_obs_space(raw, active)
        plan = ObsTransformPlan(active, raw)
        for n in a.n:
            g = torch.Generator(device=dev).manual_seed(n)
            obs = {}
            for k, (dt, c) in keys.items():
                if dt == torch.float32:
                    obs[k] = torch.rand((n, H, W, c), generator=g, device=dev)
                else:
                    obs[k] = torch.randint(0, 256 if dt == torch.uint8 else 40, (n, H, W, c), generator=g,
                                           device=dev, dtype=dt)
            store = {k: torch.zeros((2, n, *space[k].shape), dtype=keys[k][0], device=dev) for k in keys}
            slot = {k: v[1] for k, v in store.items()}

            def fused():
                plan.apply_(obs, slot)

            def torch_seq():
                for k, (mode, (hr, wr), (y0, x0), (h, w)) in plan.keys.items():
                    x = obs[k]
                    y = F.interpolate(x.permute(0, 3, 1, 2).float(), size=(hr, wr),
                                      mode="nearest" if mode == ops.OBS_NEAREST else "area")
                    y = y.to(x.dtype).permute(0, 2, 3, 1)
                    slot[k].copy_(y[:, y0:y0 + h, x0:x0 + w, :])

            tf = timed(fused, a.min_seconds)
            tt = timed(torch_seq, a.min_seconds)
            nbytes = model_bytes(plan, keys, n)
            mf, mt = statistics.median(tf), statistics.median(tt)
            gbs = nbytes / (mf * 1e-6) / 1e9
            row = dict(set=name, n=n, bytes=nbytes, fused_us=tf, torch_us=tt, speedup=mt / mf, fused_gbs=gbs,
                       share_of_peak=gbs * 1e9 / HBM_BYTES_PER_S)
            rows.append(row)
            print(f"{name:10s} {n:4d} {nbytes / 1e6:8.1f} {mf:9.1f} ({min(tf):.1f}-{max(tf):.1f}) "
                  f"{mt:9.1f} ({min(tt):.1f}-{max(tt):.1f}) {mt / mf:7.2f}x {gbs:10.0f} {row['share_of_peak']:10.1%}")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
