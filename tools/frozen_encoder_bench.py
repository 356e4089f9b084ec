#!/usr/bin/env python
"""Learner frames/s with the visual encoder trained (train_encoder=True) against frozen (train_encoder=False, the
encoder's output cached in the rollout storage), at BASELINE config #2 and #3 shapes on one GPU, plus the rollout-step
cost the frozen mode adds (one encoder forward at batch N per environment step) next to act().

One learner step = RolloutStorage.compute_returns + PPO.update on a full synthetic rollout (bench.py's definition);
frames/s = T * N / step time.  The two arms of a config are built once and timed alternately, `--rounds` times, each
after `--warmup` untimed steps; times are host clocks around work that ends in a device synchronise.

    python tools/frozen_encoder_bench.py [--configs 2 3] [--steps 3] [--warmup 1] [--rounds 2] [--out result.json]

Prints one JSON line with the card name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SHAPES = {   # bench.py WORKLOADS[2] / [3]
    2: dict(T=128, N=64, H=256, W=256, layers=2, rnn="LSTM", backbone="resnet18", ppo_epoch=2, num_mini_batch=2,
            sensors="pointnav", n_actions=4),
    3: dict(T=64, N=32, H=256, W=256, layers=1, rnn="GRU", backbone="resnet50", ppo_epoch=4, num_mini_batch=2,
            sensors="objectnav", n_actions=6),
}
PPO_KW = dict(clip_param=0.2, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4, eps=1e-5, max_grad_norm=0.2,
              use_clipped_value_loss=True, use_normalized_advantage=False)


def card():
    out = dict(name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.split(",")][:2]
    except Exception as e:   # the numbers are still reported, with the reason the query failed
        out["power_limit"] = f"unknown ({type(e).__name__})"
    return out


class Arm:
    def __init__(self, hb, c, frozen, seed=0):
        from habitat_lab_b200 import synthetic as syn
        from habitat_lab_b200.rl.single_agent_access_mgr import get_rollout_obs_space

        if c["sensors"] == "pointnav":
            space, act = syn.pointnav_spaces(c["H"], c["W"], c["n_actions"])
        else:
            space, act = syn.objectnav_spaces(c["H"], c["W"], c["n_actions"])
        torch.manual_seed(seed)
        pol = hb.PointNavResNetPolicy(space, act, hidden_size=512, num_recurrent_layers=c["layers"], rnn_type=c["rnn"],
                                      resnet_baseplanes=32, backbone=c["backbone"], normalize_visual_inputs=True)
        if frozen:
            for p in pol.net.visual_encoder.parameters():
                p.requires_grad_(False)
        self.pol = pol.cuda()
        cfg = SimpleNamespace(habitat_baselines=SimpleNamespace(rl=SimpleNamespace(
            ddppo=SimpleNamespace(train_encoder=not frozen))))
        rspace = get_rollout_obs_space(space, pol, cfg)
        self.st = hb.RolloutStorage(c["T"], c["N"], rspace, act, pol)
        self.st.to("cuda")
        self.nv = syn.fill_rollout_(self.st, seed=1, observation_space=rspace if c["sensors"] != "pointnav" else None,
                                    n_actions=c["n_actions"])
        self.ppo = hb.PPO(pol, ppo_epoch=c["ppo_epoch"], num_mini_batch=c["num_mini_batch"], **PPO_KW)
        self.frozen, self.c = frozen, c
        if frozen:
            self.encode_all()   # the cached features the learner reads (and the encode path's warm-up)

    def encode_all(self):
        """the trainer's per-step encode (batch N, eval mode) on every slot; returns ms per step"""
        obs = self.st.buffers["observations"]
        self.pol.eval()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(self.c["T"] + 1):
            self.pol.encode_visual_features(obs[t], obs["visual_features"][t])
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0) / (self.c["T"] + 1)

    def act_ms(self, reps=20):
        b = self.st.buffers
        self.pol.eval()
        args = (b["observations"][1], b["recurrent_hidden_states"][1], b["prev_actions"][1], b["masks"][1])
        self.pol.act(*args)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            self.pol.act(*args)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0) / reps

    def step(self):
        self.st.current_rollout_step_idxs = [self.c["T"]]
        self.st.compute_returns(self.nv, True, 0.99, 0.95)
        self.pol.train()
        self.ppo.update(self.st)

    def timed(self, steps, warmup):
        for _ in range(warmup):
            self.step()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            self.step()
        torch.cuda.synchronize()
        return self.c["T"] * self.c["N"] * steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 3])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frozen_encoder_bench: no CUDA device (the hot path has no CPU fallback)")
    import habitat_lab_b200 as hb

    hb.load()
    res = dict(card=card(), steps=a.steps, warmup=a.warmup, rounds=a.rounds, configs={})
    for k in a.configs:
        c = SHAPES[k]
        arms = {"train_encoder=True": Arm(hb, c, False), "train_encoder=False": Arm(hb, c, True)}
        fps = {name: [] for name in arms}
        for r in range(a.rounds):
            for name, arm in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
                fps[name].append(arm.timed(a.steps, a.warmup if r == 0 else 0))
        best = {n: max(v) for n, v in fps.items()}
        fr = arms["train_encoder=False"]
        res["configs"][k] = dict(
            shape=c, learner_fps=fps, learner_fps_best=best,
            speedup=best["train_encoder=False"] / best["train_encoder=True"],
            rollout_encode_ms_per_step=fr.encode_all(), act_ms_cached_features=fr.act_ms(),
            act_ms_encoder=arms["train_encoder=True"].act_ms())
        del arms, fr
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
