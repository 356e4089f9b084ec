"""One config-#2 minibatch pass (forward + backward + clip/Adam) for timing / profiling:
warm-up pass, then the measured pass between cudaProfilerStart/Stop (for an external profiler started with
profiling from start off).

    python tools/profile_step.py [n_envs T]                  # CUDA-event time of one minibatch
    python tools/profile_step.py --kernels DIR [n_envs T]    # + torch.profiler per-kernel table in DIR

Defaults: 64 envs x T=128 -> two minibatches of 4096 frames.  With --kernels, the measured pass runs under
torch.profiler with CUDA activities and DIR receives kernels.md / kernels.json: every device activity of that pass by
name (template arguments kept, call arguments dropped) with launch count, summed device time and share of the summed
device time.  Kernels on the side stream overlap the main stream, so the summed device time exceeds the elapsed time;
both are reported."""
import argparse
import collections
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200.synthetic import fill_rollout_, pointnav_spaces  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("n_envs", type=int, nargs="?", default=64)
ap.add_argument("T", type=int, nargs="?", default=128)
ap.add_argument("--kernels", metavar="DIR", default=None, help="write the per-kernel table of the measured pass here")
args = ap.parse_args()
n_envs, T = args.n_envs, args.T
dev = torch.device("cuda:0")
hb.load()
torch.manual_seed(100)
obs_space, act_space = pointnav_spaces(256, 256)
policy = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=2, rnn_type="LSTM",
                                 normalize_visual_inputs=True).to(dev)
ppo = hb.PPO(policy, clip_param=0.2, ppo_epoch=1, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4,
             eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True, use_normalized_advantage=False)
policy.train()
st = hb.RolloutStorage(T, n_envs, obs_space, act_space, policy)
st.to(dev)
nv = fill_rollout_(st, seed=100)
st.compute_returns(nv, True, 0.99, 0.95)
adv = ppo.get_advantages(st)
gen = st.data_generator(adv, 2)
b0 = next(gen)
b1 = next(gen)

lm = collections.defaultdict(list)
ppo._update_from_batch(b0, 0, st, lm)  # warm-up (allocations, attribute setup)
ppo._update_from_batch(b0, 0, st, lm)
torch.cuda.synchronize()


def measured_pass():
    torch.cuda.profiler.start()
    t0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ppo._update_from_batch(b1, 0, st, lm)
    e1.record()
    t_enq = (time.perf_counter() - t0) * 1e3
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    return e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3, t_enq


frames = T * n_envs // 2
dev_ms, wall_ms, enq_ms = measured_pass()
print(f"minibatch of {frames} frames: {dev_ms:.2f} ms device, {wall_ms:.2f} ms wall, {enq_ms:.2f} ms host enqueue")

if args.kernels:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        p_dev_ms, _, _ = measured_pass()
    rows = collections.defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name.split("(")[0].removeprefix("void ").strip() or e.name
        rows[name][0] += 1
        rows[name][1] += e.time_range.elapsed_us()
    total_us = sum(us for _, us in rows.values())
    table = sorted(((n, c, us) for n, (c, us) in rows.items()), key=lambda r: -r[2])
    os.makedirs(args.kernels, exist_ok=True)
    gpu = torch.cuda.get_device_name(dev)
    head = (f"One {frames}-frame config-#2 minibatch (forward + backward + clip / Adam) on {gpu} under torch.profiler: "
            f"{p_dev_ms:.2f} ms elapsed (CUDA events; {dev_ms:.2f} ms without the profiler), {total_us / 1e3:.2f} ms "
            f"summed device time over {sum(c for _, c, _ in table)} activities.")
    with open(os.path.join(args.kernels, "kernels.md"), "w") as f:
        f.write(head + "\n\n| kernel | count | total us | share |\n|---|---|---|---|\n")
        for n, c, us in table:
            f.write(f"| `{n}` | {c} | {us:.1f} | {100 * us / total_us:.2f} % |\n")
    with open(os.path.join(args.kernels, "kernels.json"), "w") as f:
        json.dump({"gpu": gpu, "frames": frames, "elapsed_ms": p_dev_ms, "elapsed_ms_unprofiled": dev_ms,
                   "summed_device_us": total_us,
                   "kernels": [{"name": n, "count": c, "total_us": us, "share": us / total_us} for n, c, us in table]},
                  f, indent=1)
    print(head)
    for n, c, us in table[:25]:
        print(f"{us / 1e3:9.3f} ms {100 * us / total_us:6.2f} % {c:5d}x  {n[:140]}")
