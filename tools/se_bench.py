"""Cost of the squeeze-excite branch: learner frames/s of config #3 / #4 (bench.py's workloads) with the plain backbone
against its SE variant (resnet50 -> se_resnet50, resneXt50 -> se_resneXt50), measured in one process, and the SE kernels'
share of one SE minibatch under torch.profiler.

    python tools/se_bench.py [--configs 3 4] [--rounds 3] [--updates 5] [--out DIR]

Each round times `--updates` minibatch updates (forward + loss + backward + clip / Adam on T * N / num_mini_batch frames)
of the plain policy, then of the SE policy, so drift of the shared machine hits both alike; the median over rounds is
reported with the range.  With --out, DIR receives se_bench.json."""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import habitat_lab_b200 as hb  # noqa: E402

SE_OF = {"resnet50": "se_resnet50", "resneXt50": "se_resneXt50"}
SE_KERNELS = ("gn_se_residual_relu_kernel", "gn_se_bwd_kernel")


def make_learner(dev, backbone, seed=100):
    cfg = bench.CFG
    cfg["backbone"] = backbone
    torch.manual_seed(seed)
    obs_space, act_space = bench.make_spaces()
    policy = bench.make_policy(hb, obs_space, act_space).to(dev).train()
    ppo = hb.PPO(policy, clip_param=cfg["clip_param"], ppo_epoch=1, num_mini_batch=cfg["num_mini_batch"],
                 value_loss_coef=cfg["value_loss_coef"], entropy_coef=cfg["entropy_coef"], lr=cfg["lr"], eps=cfg["eps"],
                 max_grad_norm=cfg["max_grad_norm"], use_clipped_value_loss=True, use_normalized_advantage=False)
    st = hb.RolloutStorage(cfg["T"], cfg["N"], obs_space, act_space, policy)
    st.to(dev)
    nv = bench.fill(st, seed, obs_space)
    st.compute_returns(nv, True, cfg["gamma"], cfg["tau"])
    batch = next(iter(st.data_generator(ppo.get_advantages(st), cfg["num_mini_batch"])))
    metrics = collections.defaultdict(list)

    def update():
        ppo._update_from_batch(batch, 0, st, metrics)

    for _ in range(2):   # allocations, weight images, autotuned launches
        update()
    torch.cuda.synchronize()
    return update, cfg["T"] * cfg["N"] // cfg["num_mini_batch"]


def timed(update, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        update()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def se_share(update, frames):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        update()
        torch.cuda.synchronize()
    rows = collections.defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name.split("(")[0].removeprefix("void ").strip() or e.name
        rows[name][0] += 1
        rows[name][1] += e.time_range.elapsed_us()
    total = sum(us for _, us in rows.values())
    se = {n: (c, us) for n, (c, us) in rows.items() if any(k in n for k in SE_KERNELS)}
    return total, se


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[3, 4])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("se_bench: no CUDA device")
    hb.load()
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print("GPU:", gpu[0] if gpu else torch.cuda.get_device_name(dev))
    report = {"gpu": gpu[0] if gpu else torch.cuda.get_device_name(dev), "configs": {}}
    for cid in args.configs:
        bench.select_workload(cid)
        plain = bench.CFG["backbone"]
        learners = {bb: make_learner(dev, bb) for bb in (plain, SE_OF[plain])}
        bench.CFG["backbone"] = plain
        rates = {bb: [] for bb in learners}
        for _ in range(args.rounds):
            for bb, (update, frames) in learners.items():
                rates[bb].append(args.updates * frames / timed(update, args.updates))
        update, frames = learners[SE_OF[plain]]
        total_us, se = se_share(update, frames)
        se_us = sum(us for _, us in se.values())
        med = {bb: statistics.median(r) for bb, r in rates.items()}
        rep = {"frames_per_minibatch": frames, "frames_per_s": rates, "median": med,
               "se_over_plain": med[SE_OF[plain]] / med[plain], "profiled_device_us": total_us,
               "se_kernels": {n: {"count": c, "us": us, "share": us / total_us} for n, (c, us) in se.items()},
               "se_share": se_us / total_us}
        report["configs"][cid] = rep
        print(f"config #{cid} ({frames} frames per minibatch update):")
        for bb, r in rates.items():
            print(f"  {bb:14s} {med[bb]:9.0f} frames/s  (range {min(r):.0f}-{max(r):.0f}, {args.rounds} rounds)")
        print(f"  SE / plain = {rep['se_over_plain']:.4f}")
        print(f"  SE kernels in one {SE_OF[plain]} minibatch: {se_us / 1e3:.3f} ms of {total_us / 1e3:.2f} ms summed "
              f"device time ({100 * rep['se_share']:.2f} %)")
        for n, (c, us) in sorted(se.items(), key=lambda kv: -kv[1][1]):
            print(f"    {us / 1e3:8.3f} ms {100 * us / total_us:6.2f} % {c:5d}x  {n}")
        del learners, update
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "se_bench.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
