"""Float64 restatement of VER's return computation over packed sequences, and a scripted VER collection that drives a
rollout storage through the inference worker's bookkeeping (habitat_baselines/rl/ver/inference_worker.py:219-450).

Both the reference's VERRolloutStorage (tests/golden/make_golden_ver.py) and ours (the tests) are driven by
`drive_rollout` with the same seeded script, so their buffers can be compared stage by stage.

Error bar of the GAE kernel: it accumulates in fp64 in the reference's operation order and rounds each return once to
fp32, so a return may differ from the restatement's by at most half an fp32 ulp of the return (the fp64 chain's own
error, ~T * 2^-53 relative, is far below it).  `bar(ref)` is that half ulp; perturbed restatements must miss it by 10x.
"""
from __future__ import annotations

import numpy as np
import torch

N_ENVS, NUM_STEPS, LAYERS, HID = 6, 8, 2, 4
GAMMA, TAU = 0.99, 0.95


def ver_gae_reference(rewards, values, returns, is_stale, pack, gamma, tau, use_gae=True, keep_stale=True,
                      zero_bootstrap=True):
    """Returns (f32 [M]) of the packed GAE: each sequence walked backwards in float64.  keep_stale / zero_bootstrap
    False give the perturbed restatements."""
    rewards, values = (np.asarray(x, dtype=np.float32).reshape(-1) for x in (rewards, values))
    out = np.asarray(returns, dtype=np.float32).reshape(-1).copy()
    stale = np.asarray(is_stale).reshape(-1).astype(bool)
    gt = (tau if use_gae else 1.0) * gamma
    lengths, last = pack["sequence_lengths"], pack["last_sequence_in_batch_mask"]
    offs = np.cumsum(pack["num_seqs_at_step"]) - pack["num_seqs_at_step"]
    for s in range(len(lengths)):
        gae, last_v = 0.0, 0.0
        for t in range(lengths[s] - 1, -1, -1):
            i = pack["select_inds"][offs[t] + s]
            v = float(values[i])
            gae = (float(rewards[i]) + gamma * last_v - v) + gt * gae
            boot = last[s] and t == lengths[s] - 1
            if boot and zero_bootstrap:
                gae = 0.0
            if boot:
                out[i] = np.nan
            elif not (keep_stale and stale[i] and np.isfinite(out[i])):
                out[i] = np.float32(gae + v)
            last_v = v
    return out


def bar(ref):
    """Half an fp32 ulp of each finite reference return."""
    ref = np.asarray(ref, dtype=np.float32)
    return 0.5 * np.spacing(np.abs(ref)).astype(np.float64)


# ---- scripted collection ---------------------------------------------------------------------------------------
class Script:
    """Seeded stand-in for environments and policy: per-environment step durations (environment 0 is slow enough to
    contribute a single step to some rollouts), rewards, dones, values, log-probs and hidden states."""

    def __init__(self, seed=0, n_envs=N_ENVS, p_done=0.3):
        self.rng = np.random.default_rng(seed)
        self.p_done = p_done
        self.n = n_envs
        self.speed = 1.0 + 2.0 * self.rng.random(n_envs)
        self.speed[0] = 30.0
        self.ready = np.zeros(n_envs)
        self.now = 0.0
        self.ep = np.zeros(n_envs, np.int64)
        self.step = np.zeros(n_envs, np.int64)
        self.mask = np.zeros(n_envs, bool)
        self.reward = np.zeros(n_envs, np.float32)
        self.new_reqs = list(range(n_envs))
        self.replay = []
        self.n_replay = 0

    def env_step(self, e):
        done = self.rng.random() < self.p_done
        self.reward[e] = np.float32(self.rng.normal())
        self.mask[e] = not done
        if done:
            self.ep[e] += 1
            self.step[e] = 0
        else:
            self.step[e] += 1
        self.ready[e] = self.now + self.speed[e]


def _policy_step(r, sc: Script):
    """inference_worker.py step() for the scripted requests, on a storage with flat buffers."""
    sc.new_reqs.sort(key=lambda e: (int(r.actor_steps_collected[e]), e))
    ptr = int(r.ptr[0])
    num = min(int(r.num_steps_to_collect - r.num_steps_collected[0]), len(sc.new_reqs))
    r.ptr[:] = ptr + num
    r.num_steps_collected += num - sc.n_replay
    final = int(r.num_steps_collected[0]) == r.num_steps_to_collect
    if final:
        r.rollout_done[:] = True
    sc.replay += sc.new_reqs[num:]
    reqs, sc.new_reqs = sc.new_reqs[:num], []
    if num == 0:
        return
    b = r.buffers
    idx = torch.as_tensor(reqs)
    hidden = r.next_hidden_states[idx].clone()
    prev_actions = r.next_prev_actions[idx].clone()
    # stand-ins shaped like the storage's buffers (only the bookkeeping matters to the scripts that use them)
    actions = torch.as_tensor(sc.rng.integers(0, 4, (num, *b["actions"].shape[1:]))).to(b["actions"].dtype)
    new_hidden = torch.as_tensor(sc.rng.normal(size=(num, *b["recurrent_hidden_states"].shape[1:])).astype(np.float32))
    if not final:
        r.next_hidden_states[idx] = new_hidden
        r.next_prev_actions[idx] = actions
    prev = r.prev_inds[reqs].copy()
    r.prev_inds[reqs] = np.arange(ptr, ptr + num)
    for j, e in enumerate(reqs):
        if prev[j] >= 0:
            b["rewards"][int(prev[j])] = float(sc.reward[e])
    rows = slice(ptr, ptr + num)
    b["masks"][rows] = torch.as_tensor(sc.mask[reqs]).view(num, 1)
    pg = b["observations"]["pointgoal_with_gps_compass"]
    pg[rows] = torch.as_tensor(sc.rng.normal(size=(num, 2)).astype(np.float32))
    b["actions"][rows] = actions
    b["action_log_probs"][rows] = torch.as_tensor(sc.rng.normal(size=(num, 1)).astype(np.float32))
    b["recurrent_hidden_states"][rows] = hidden
    b["prev_actions"][rows] = prev_actions
    b["policy_version"][rows] = r.current_policy_version.view(1, 1).expand(num, 1)
    b["episode_ids"][rows] = torch.as_tensor(sc.ep[reqs]).view(num, 1)
    b["environment_ids"][rows] = torch.as_tensor(reqs).view(num, 1)
    b["step_ids"][rows] = torch.as_tensor(sc.step[reqs]).view(num, 1)
    b["value_preds"][rows] = torch.as_tensor(sc.rng.normal(size=(num, 1)).astype(np.float32))
    b["returns"][rows] = float("nan")
    r.actor_steps_collected[reqs] += 1
    r.current_steps[reqs] += 1
    for e in reqs:
        if final:
            sc.replay.append(e)
        else:
            sc.env_step(e)
    sc.n_replay = 0


def drive_rollout(r, sc: Script):
    """Collect one rollout into storage r (flat buffers, CPU), then the finish_rollout bookkeeping."""
    while not r.rollout_done[0]:
        if not sc.new_reqs:
            busy = np.array([e not in sc.replay for e in range(sc.n)])
            sc.now = float(np.min(sc.ready[busy]))
            done = [e for e in range(sc.n) if busy[e] and sc.ready[e] <= sc.now + 0.5]
            for e in done:
                sc.ready[e] = np.inf
            sc.new_reqs += done
        _policy_step(r, sc)
    sc.new_reqs = sc.replay + sc.new_reqs
    sc.replay = []
    sc.n_replay = len(sc.new_reqs)
    r.will_replay_step[sc.new_reqs] = True


def make_spaces():
    from habitat_lab_b200.common import spaces
    obs = spaces.Dict({"pointgoal_with_gps_compass": spaces.Box(-1e9, 1e9, (2,), np.float32)})
    return obs, spaces.Discrete(4)


class FakeActorCritic:
    num_recurrent_layers = LAYERS * 2
    recurrent_hidden_size = HID


BUFFER_KEYS = ("rewards", "value_preds", "returns", "masks", "actions", "action_log_probs", "recurrent_hidden_states",
               "prev_actions", "policy_version", "episode_ids", "environment_ids", "step_ids", "is_stale", "is_coeffs")


def snapshot(r):
    out = {k: r.buffers[k].clone() for k in BUFFER_KEYS}
    out["observations"] = r.buffers["observations"]["pointgoal_with_gps_compass"].clone()
    out["ptr"] = int(r.ptr[0])
    out["prev_inds"] = torch.as_tensor(np.array(r.prev_inds))
    out["current_steps"] = torch.as_tensor(np.array(r.current_steps))
    out["will_replay_step"] = torch.as_tensor(np.array(r.will_replay_step))
    return out


# ---- a whole packed PPO.update (tests/golden/make_golden_ver_update.py, tests/test_gpu_ver.py) ----------------------
UPDATE_CASES = {
    # a small categorical LSTM policy
    "ver_update_small": dict(N=4, T=16, H=64, W=64, layers=2, gaussian=0, seed=61, p_done=0.15, normalized=False),
    # rl_skill.yaml's shape: 18 environments, num_steps 128, 2 minibatches, LSTM-512x2, a Gaussian head (images reduced)
    "ver_update_skill": dict(N=18, T=128, H=64, W=64, layers=2, gaussian=7, seed=62, p_done=0.01, normalized=True),
}
UPDATE_PPO_KW = dict(clip_param=0.2, ppo_epoch=1, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4,
                     eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True)
ID_KEYS = ("masks", "policy_version", "episode_ids", "environment_ids", "step_ids", "is_stale", "is_coeffs")
SMALL_PARAMS = ("action_distribution.", "critic.", "net.prev_action_embedding.")


def fill_float_buffers(buffers, seed):
    """Seeded contents of everything but the bookkeeping of a flat VER buffer (CPU tensors): observations in sorted key
    order, rewards, values, old log-probs, actions, previous actions, stored hidden states; returns NaN."""
    g = torch.Generator().manual_seed(seed)
    obs = buffers["observations"]
    for k in sorted(obs.keys()):
        t = obs[k]
        if t.dtype == torch.uint8:
            t.copy_(torch.randint(0, 256, t.shape, generator=g, dtype=torch.uint8))
        else:
            t.copy_(torch.rand(t.shape, generator=g))
    M = buffers["rewards"].shape[0]
    buffers["rewards"].copy_(torch.randn(M, 1, generator=g) * 0.5)
    buffers["value_preds"].copy_(torch.randn(M, 1, generator=g) * 0.5)
    acts = buffers["actions"]
    if acts.dtype == torch.int64:
        acts.copy_(torch.randint(0, 4, acts.shape, generator=g))
        buffers["prev_actions"].copy_(torch.randint(0, 4, acts.shape, generator=g))
        buffers["action_log_probs"].copy_(np.log(0.25) + 0.2 * torch.randn(M, 1, generator=g))
    else:
        A = acts.shape[1]
        acts.copy_(torch.rand(acts.shape, generator=g) * 3.0 - 1.5)
        buffers["prev_actions"].copy_(torch.rand(acts.shape, generator=g) * 3.0 - 1.5)
        buffers["action_log_probs"].copy_(-A * 0.5 * np.log(2 * np.pi) - 0.5 * (acts ** 2).sum(-1, keepdim=True)
                                          + 0.2 * torch.randn(M, 1, generator=g))
    h = buffers["recurrent_hidden_states"]
    h.copy_(torch.randn(h.shape, generator=g) * 0.5)
    buffers["returns"].fill_(float("nan"))
