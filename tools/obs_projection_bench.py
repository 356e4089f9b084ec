"""Time the cube-map projection kernel (ops.obs_project: every target in one launch, written into a rollout-storage
slot) per env step, against the reference's own op sequence run with torch on the same GPU: stack the six faces,
permute to NCHW, .float(), multiply by the input z-factor (depth), repeat the grid per env, grid_sample every face
at every output pixel, sum over the faces, .to(dtype), permute back.

Workloads: six 256 x 256 cube faces into
  - a 256 x 512 equirect, u8 RGB (CubeMap2Equirect's default size),
  - a 256 x 256 equirect, f32 depth (the trainer's depth rig),
  - a 256 x 256 fisheye, u8 RGB (CubeMap2Fisheye's defaults),
at N = 4 / 16 / 64 / 256 envs.  Each point: CUDA events over enough calls for each repeat to last >= --min-seconds
(default 1 s), three repeats (median and spread).  The bytes model is the minimum traffic: every face byte read once plus every output byte written once.
The torch path runs CUDA's grid_sample, which does not round like the CPU grid_sample the kernel reproduces, so only
its time is compared.

    python tools/obs_projection_bench.py [--n 4 16 64 256] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402
from habitat_lab_b200.common.obs_transformers import CubeMap2Equirect, CubeMap2Fisheye  # noqa: E402
from obs_transform_bench import HBM_BYTES_PER_S, card, timed  # noqa: E402

FACE = 256
WORKLOADS = {
    "eq512_rgb": (lambda u: CubeMap2Equirect(u, (256, 512)), "rgb", torch.uint8, 3),
    "eq256_depth": (lambda u: CubeMap2Equirect(u, (256, 256)), "depth", torch.float32, 1),
    "fish256_rgb": (lambda u: CubeMap2Fisheye(u, (256, 256), 180, (0.2, 0.2, 0.2)), "rgb", torch.uint8, 3),
}


def torch_path(t, faces, is_depth):
    """The reference's ProjectionTransformer.forward for one group, on CUDA tensors (the grids repeated per env
    once, as its _grids_cache does)."""
    s = t.stitch
    B = faces[0].shape[0]
    n_in = len(faces)
    h, w = s.out_hw
    grids = s.grids.to(faces[0].device)                                            # [n_in, 1, h, w, 2]
    cache = grids.repeat(B, 1, 1, 1, 1).view(B * n_in, h, w, 2)
    in_zf = None if s.in_zfactor is None or not is_depth else s.in_zfactor.to(faces[0].device).repeat(B, 1, 1, 1)

    def run():
        imgs = torch.flatten(torch.stack(faces, dim=1), end_dim=1).permute(0, 3, 1, 2).float()
        if in_zf is not None:
            imgs = imgs * in_zf
        out = F.grid_sample(imgs, cache, align_corners=True, padding_mode="zeros")
        out = out.view(B, n_in, imgs.shape[1], h, w).sum(dim=1)
        return out.to(faces[0].dtype).permute(0, 2, 3, 1)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[4, 16, 64, 256])
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("obs_projection_bench: no CUDA device")
    hb.load()
    dev = torch.device("cuda")
    print(f"card: {card()}")
    print(f"{'workload':12s} {'N':>4s} {'MB':>8s} {'kernel us':>18s} {'torch us':>20s} {'speedup':>8s} "
          f"{'GB/s':>7s} {'of 3.35TB/s':>11s}")
    rows = []
    for name, (make, key, dt, c) in WORKLOADS.items():
        uuids = [f"{key}_{i}" for i in range(6)]
        t = make(uuids)
        _, _, is_depth = t.groups[0]
        h, w = t.img_shape
        for n in a.n:
            g = torch.Generator(device=dev).manual_seed(n)
            if dt == torch.uint8:
                faces = [torch.randint(0, 256, (n, FACE, FACE, c), generator=g, device=dev, dtype=dt) for _ in uuids]
            else:
                faces = [torch.rand((n, FACE, FACE, c), generator=g, device=dev) for _ in uuids]
            obs = dict(zip(uuids, faces))
            slot = torch.empty((3, n, h, w, c), dtype=dt, device=dev)[1]   # one slot of a storage buffer
            jobs = t.jobs(obs, {uuids[0]: slot})
            ref = torch_path(t, faces, is_depth)
            k_us = timed(lambda: ops.obs_project(jobs), a.min_seconds)
            t_us = timed(lambda: slot.copy_(ref()), a.min_seconds)
            es = torch.empty((), dtype=dt).element_size()
            nbytes = n * (6 * FACE * FACE + h * w) * c * es
            km, tm = statistics.median(k_us), statistics.median(t_us)
            gbs = nbytes / (km * 1e-6) / 1e9
            row = dict(workload=name, n=n, bytes=nbytes, kernel_us=k_us, torch_us=t_us, speedup=tm / km,
                       gbps=gbs, frac_hbm=gbs * 1e9 / HBM_BYTES_PER_S)
            rows.append(row)
            print(f"{name:12s} {n:4d} {nbytes / 1e6:8.1f} {km:9.1f} [{min(k_us):.0f}-{max(k_us):.0f}] "
                  f"{tm:10.1f} [{min(t_us):.0f}-{max(t_us):.0f}] {tm / km:7.1f}x {gbs:7.0f} "
                  f"{100 * row['frac_hbm']:10.1f}%")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
