"""Time the Gaussian action head kernels against the reference's torch op sequence on CUDA.

  act  : hb200_gaussian_act at N frames (one rollout step) vs GaussianNet + CriticHead + CustomNormal.rsample +
         log_probs (HB/utils/common.py:99-175, HB/rl/ppo/policy.py:330-342) as torch ops.
  loss : hb200_gaussian_ppo_loss forward + backward at B frames vs the same head, PPO's loss section
         (HB/rl/ppo/ppo.py:195-250) and autograd's backward to the features and head parameters.

Prints one JSON line: per leg the median over `--runs` runs of the mean time per call (CUDA events around `--iters`
calls after warm-up), with the card's name, power limit and max SM clock read in the same process.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import habitat_lab_b200 as hb  # noqa: E402
from habitat_lab_b200 import ops  # noqa: E402


def _time(fn, iters, warmup=20):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters   # us


def _params(H, A, std_param, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    L = A if std_param else 2 * A
    return dict(w_mu=torch.randn(L, H, generator=g, device=dev) / math.sqrt(H),
                b_mu=torch.zeros(L, device=dev),
                std=(torch.randn(A, generator=g, device=dev) * 0.01 - 1.0) if std_param else None,
                w_val=torch.randn(1, H, generator=g, device=dev) / math.sqrt(H), b_val=torch.zeros(1, device=dev))


def _torch_head(P, x, A, lo, hi):
    z = torch.nn.functional.linear(x, P["w_mu"], P["b_mu"]).float()
    mu, s = (z, P["std"]) if P["std"] is not None else torch.chunk(z, 2, -1)
    mu = torch.tanh(mu)
    s = torch.exp(torch.clamp(s, lo, hi))
    return torch.distributions.Normal(mu, s, validate_args=False), torch.nn.functional.linear(x, P["w_val"], P["b_val"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hidden", type=int, default=512)
    ap.add_argument("--actions", type=int, default=7)
    ap.add_argument("--act-n", type=int, default=64)
    ap.add_argument("--loss-b", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--std-param", action="store_true", help="social_nav.yaml's use_std_param (default: monolithic)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gaussian_bench: needs a CUDA device")
    hb.load()
    dev = torch.device("cuda")
    H, A = a.hidden, a.actions
    lo, hi = -5.0, 2.0
    flags = ops.GAUSS_LOG_STD | ops.GAUSS_CLAMP_STD | ops.GAUSS_TANH | (ops.GAUSS_STD_PARAM if a.std_param else 0)
    P = _params(H, A, a.std_param, dev)
    # ---- act at N
    N = a.act_n
    xa = torch.randn(N, H, device=dev)
    act, alp, val = torch.empty(N, A, device=dev), torch.empty(N, device=dev), torch.empty(N, device=dev)

    def ours_act():
        eps = torch.randn(N, A, device=dev)
        ops.gaussian_act(xa, P["w_mu"], P["b_mu"], P["std"], P["w_val"], P["b_val"], eps, flags, lo, hi, act, alp, val)

    def ref_act():
        with torch.no_grad():
            d, v = _torch_head(P, xa, A, lo, hi)
            s = d.rsample()
            return s, d.log_prob(s).sum(-1, keepdim=True), v

    # ---- loss forward + backward at B
    B = a.loss_b
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, H, generator=g, device=dev)
    acts = torch.randn(B, A, generator=g, device=dev)
    old_lp, adv = torch.randn(B, generator=g, device=dev) - 5.0, torch.randn(B, generator=g, device=dev)
    old_v, ret = torch.randn(B, generator=g, device=dev), torch.randn(B, generator=g, device=dev)
    L = P["w_mu"].shape[0]
    out = dict(values=torch.empty(B, device=dev), log_probs=torch.empty(B, device=dev),
               entropy=torch.empty(B, device=dev), metrics=torch.empty(12, device=dev),
               d_features=torch.empty(B, H, device=dev), d_w_mu=torch.empty(L, H, device=dev),
               d_b_mu=torch.empty(L, device=dev), d_std=torch.empty(A, device=dev) if a.std_param else None,
               d_w_val=torch.empty(1, H, device=dev), d_b_val=torch.empty(1, device=dev))
    ws = ops.gaussian_ppo_loss_workspace(B, H, A, dev)

    def ours_loss():
        ops.gaussian_ppo_loss(x, P["w_mu"], P["b_mu"], P["std"], P["w_val"], P["b_val"], acts, old_lp, adv, old_v, ret,
                              flags, lo, hi, 0.2, 0.5, 0.01, True, True, out, ws)

    Pr = {k: None if v is None else v.clone().requires_grad_(True) for k, v in P.items()}
    xr = x.clone().requires_grad_(True)

    def ref_loss():
        for t in list(Pr.values()) + [xr]:
            if t is not None:
                t.grad = None
        d, v = _torch_head(Pr, xr, A, lo, hi)
        lp, ent = d.log_prob(acts).sum(-1, keepdim=True), d.entropy().sum(-1, keepdim=True)
        ratio = torch.exp(lp - old_lp[:, None])
        s1, s2 = ratio * adv[:, None], torch.clamp(ratio, 0.8, 1.2) * adv[:, None]
        a_loss = -torch.min(s1, s2)
        delta = v.detach() - old_v[:, None]
        vc = old_v[:, None] + delta.clamp(-0.2, 0.2)
        vv = torch.where(delta.abs() < 0.2, v, vc)
        v_loss = 0.5 * torch.nn.functional.mse_loss(vv, ret[:, None], reduction="none")
        (0.5 * v_loss.mean() + a_loss.mean() - 0.01 * ent.mean()).backward()

    legs = dict(act=(ours_act, ref_act), loss=(ours_loss, ref_loss))
    res = {}
    for name, (ours, ref) in legs.items():
        t_o, t_r = [], []
        for _ in range(a.runs):   # alternate the two arms
            t_o.append(_time(ours, a.iters))
            t_r.append(_time(ref, a.iters))
        res[name] = dict(hb200_us=round(statistics.median(t_o), 2), reference_torch_cuda_us=round(statistics.median(t_r), 2),
                         runs_hb200_us=[round(t, 2) for t in t_o], runs_reference_us=[round(t, 2) for t in t_r])
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card, hidden=H, actions=A, act_n=N, loss_b=B, std_param=a.std_param, **res)))


if __name__ == "__main__":
    main()
