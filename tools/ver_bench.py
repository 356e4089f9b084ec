"""VER on the GPU: compute_returns (the packed GAE kernel against the reference's host path), learner frames/s of a
packed VER minibatch against a [T, n] minibatch of the same frames, and the padding share of the packed recurrence.

    python tools/ver_bench.py [--envs 18] [--steps 128] [--reps 20] [--rounds 30]

The reference arm runs the unmodified reference VERRolloutStorage.compute_returns from oracle/_ref (build() installs
it) on the same device buffers.  The learner arms time loss_and_backward on the same frames as a [T, n] rectangle and
as a shuffled VER minibatch of its episodes (short episodes: much padding; long episodes: little), with CUDA events,
the arms alternated round by round; each arm reports the median and the spread over rounds.  Prints the card's name,
power limit and SM clocks with the numbers, as one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


class _HiddenShape:
    """what a rollout storage reads from its actor_critic"""
    num_recurrent_layers, recurrent_hidden_size = 4, 8


def filled_storage(cls, N, T, dev, spaces):
    """a flat VER buffer with unequal steps per environment and episodes ending mid-rollout"""
    obs, act = spaces
    r = cls(T, N, obs, act, _HiddenShape(), variable_experience=True)
    seed = 0
    rng = np.random.default_rng(seed)
    M = (T + 1) * N
    env = np.concatenate([np.arange(N), rng.choice(N, M - N, p=np.linspace(1, 3, N) / np.linspace(1, 3, N).sum())])
    ep, step = np.zeros(M, np.int64), np.zeros(M, np.int64)
    for e in range(N):
        rows = np.nonzero(env == e)[0]
        ep[rows] = np.cumsum(rng.random(rows.size) < 0.02)
        step[rows] = np.arange(rows.size)
    b = r.buffers
    for k, v in (("environment_ids", env), ("episode_ids", ep), ("step_ids", step)):
        b[k].copy_(torch.from_numpy(v).view(-1, 1))
    b["rewards"].copy_(torch.from_numpy(rng.normal(size=(M, 1)).astype(np.float32)))
    b["value_preds"].copy_(torch.from_numpy(rng.normal(size=(M, 1)).astype(np.float32)))
    b["policy_version"].fill_(1)
    r.to(dev)
    return r


def time_returns(r, reps):
    rets = r.buffers["returns"].clone()
    times = []
    for _ in range(reps + 2):
        r.buffers["returns"].copy_(rets)
        r.after_rollout()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r.compute_returns(True, 0.99, 0.95)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return float(np.median(times[2:]))


def _policy(hw):
    import habitat_lab_b200 as hb
    from habitat_lab_b200.synthetic import pointnav_spaces
    torch.manual_seed(0)
    obs_space, act_space = pointnav_spaces(hw, hw)
    p = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, num_recurrent_layers=2, rnn_type="LSTM",
                                normalize_visual_inputs=True).cuda()
    p.train()
    return p, obs_space


def _batches(p, obs_space, T, n, p_done, seed=1):
    """one [T, n] minibatch with episodes ending at rate p_done, and the same frames as a shuffled VER minibatch"""
    from habitat_lab_b200.common.ver_rollout_storage import PackedSequenceInfo, build_pack_info_from_episode_ids
    from habitat_lab_b200.rl.resnet_policy import RolloutObservations
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev, B, sp = torch.device("cuda"), T * n, obs_space.spaces
    obs = {"rgb": torch.randint(0, 256, (B, *sp["rgb"].shape), generator=g, device=dev, dtype=torch.uint8),
           "depth": torch.rand((B, *sp["depth"].shape), generator=g, device=dev),
           "pointgoal_with_gps_compass": torch.rand((B, 2), generator=g, device=dev)}
    f = lambda: torch.randn(B, 1, generator=g, device=dev)  # noqa: E731
    actions = torch.randint(0, 4, (B, 1), generator=g, device=dev)
    rect = dict(actions=actions, prev_actions=actions.roll(1, 0), masks=torch.rand(B, 1, generator=g, device=dev) >= p_done,
                action_log_probs=f() - 1.4, advantages=f(), value_preds=f(), returns=f(),
                recurrent_hidden_states=torch.randn(n, 4, 512, generator=g, device=dev) * 0.5)
    m = rect["masks"].view(T, n).cpu().numpy()
    ep, env = np.cumsum(~m, 0), np.tile(np.arange(n), (T, 1))
    st = np.tile(np.arange(T)[:, None], (1, n))
    perm = np.random.default_rng(seed).permutation(B)
    info = build_pack_info_from_episode_ids(ep.reshape(-1)[perm], env.reshape(-1)[perm], st.reshape(-1)[perm])
    pt = torch.from_numpy(perm).to(dev)
    packed = {k: v[pt] for k, v in rect.items() if k != "recurrent_hidden_states"}
    packed.update(recurrent_hidden_states=rect["recurrent_hidden_states"],
                  rnn_build_seq_info=PackedSequenceInfo.build(info, dev),
                  observations=RolloutObservations(obs, pt.int()))
    rect["observations"] = RolloutObservations(obs, torch.arange(B, device=dev, dtype=torch.int32))
    return rect, packed


def learner(args):
    T, n = args.learner_T, args.learner_n
    p, obs_space = _policy(args.hw)
    out = {}
    for label, p_done in (("short_episodes", 0.15), ("long_episodes", 0.01)):
        rect, packed = _batches(p, obs_space, T, n, p_done)
        arms = {"rect": rect, "packed": packed}
        for b in arms.values():
            for _ in range(3):
                p.loss_and_backward(b, 0.2, 0.5, 0.01, True)
        ms = {k: [] for k in arms}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(args.rounds):                     # alternate the arms, several updates per timing
            for k, b in arms.items():
                torch.cuda.synchronize()
                ev[0].record()
                for _ in range(args.reps):
                    p.loss_and_backward(b, 0.2, 0.5, 0.01, True)
                ev[1].record()
                torch.cuda.synchronize()
                ms[k].append(ev[0].elapsed_time(ev[1]) / args.reps)
        seq = packed["rnn_build_seq_info"]
        res = dict(frames=T * n, sequences=seq.num_seqs, t_max=seq.max_len, padding_fraction=seq.padding_fraction)
        for k, v in ms.items():
            v = np.array(v)
            res[f"{k}_ms_median"] = float(np.median(v))
            res[f"{k}_ms_p10_p90"] = [float(np.percentile(v, 10)), float(np.percentile(v, 90))]
            res[f"{k}_frames_per_s"] = T * n / (float(np.median(v)) * 1e-3)
        out[label] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=18)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--learner-T", type=int, default=64)
    ap.add_argument("--learner-n", type=int, default=16)
    ap.add_argument("--hw", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ver_bench: no CUDA device")
    dev = torch.device("cuda")
    from habitat_lab_b200.common.ver_rollout_storage import VERRolloutStorage
    from oracle import ref_shim
    from habitat_lab_b200.common import spaces
    res = dict(card=card(), envs=args.envs, num_steps=args.steps)
    our_spaces = (spaces.Dict({"pointgoal_with_gps_compass": spaces.Box(-1e9, 1e9, (2,), np.float32)}),
                  spaces.Discrete(4))
    ours = filled_storage(VERRolloutStorage, args.envs, args.steps, dev, our_spaces)
    res["returns_kernel_s"] = time_returns(ours, args.reps)
    if ref_shim.reference_available():
        ref_shim.install()
        from habitat_baselines.rl.ver.ver_rollout_storage import VERRolloutStorage as RefStorage
        gs = sys.modules["gym.spaces"]
        ref_spaces = (gs.Dict({"pointgoal_with_gps_compass": gs.Box(-1e9, 1e9, (2,), np.float32)}), gs.Discrete(4))
        ref = filled_storage(RefStorage, args.envs, args.steps, dev, ref_spaces)
        res["returns_reference_host_s"] = time_returns(ref, args.reps)
        same = torch.equal(torch.nan_to_num(ours.buffers["returns"], nan=1e30),
                           torch.nan_to_num(ref.buffers["returns"], nan=1e30))
        res["returns_identical_to_reference"] = bool(same)
    else:
        res["returns_reference_host_s"] = "not measured: oracle/_ref missing"
    res.update(learner(args))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
