"""GPU: fine-tuning with a frozen visual encoder (train_encoder=False).  One PPO.update against the unmodified
reference updater on the CPU (configs #2 and #3, same weights, rollout and cached `visual_features`), with no encoder
kernel launched; the trainer's rollout caching the encoder output in the storage; run-to-run identity; a pretrained
fine-tune end to end; and the DD-PPO exchange restricted to the trainable parameters (two GPUs only).

Bars are those of tests/test_gpu_policy.py::test_ppo_update_vs_reference."""
import collections
import math
import os
import re
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ref_shim

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = "cuda"
T, N, H, W = 8, 4, 128, 128
CONFIGS = {   # BASELINE config #2 (PointNav, ResNet18 + 2-layer LSTM) and #3 (ObjectNav sensors, ResNet50 + GRU)
    2: dict(backbone="resnet18", rnn_type="LSTM", num_recurrent_layers=2),
    3: dict(backbone="resnet50", rnn_type="GRU", num_recurrent_layers=1),
}
PPO_KW = dict(clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01, lr=2.5e-4,
              eps=1e-5, max_grad_norm=0.2, use_clipped_value_loss=True, use_normalized_advantage=False)
# kernels of the input prep, RunningMeanAndVar, the convolutions, GroupNorm and the encoder's weight packing
ENCODER_KERNELS = re.compile(r"conv_|unpack_|gn_(apply|bwd|relu|residual|se|pool)|prep_|maxpool|pack_(halo_)?weight|"
                             r"f16_to_bf16|hwc")


def _spaces(sp, kind):
    od = collections.OrderedDict()
    od["rgb"] = sp.Box(0, 255, (H, W, 3), np.uint8)
    od["depth"] = sp.Box(0, 1, (H, W, 1), np.float32)
    if kind == 2:
        od["pointgoal_with_gps_compass"] = sp.Box(-1e9, 1e9, (2,), np.float32)
    else:
        od["semantic"] = sp.Box(0, 2 ** 30, (H, W, 1), np.int32)
        od["objectgoal"] = sp.Box(0, 20, (1,), np.int64)
        od["compass"] = sp.Box(-np.pi, np.pi, (1,), np.float32)
        od["gps"] = sp.Box(-1e9, 1e9, (2,), np.float32)
    return sp.Dict(od), sp.Discrete(4)


def _frozen_cfg():
    return SimpleNamespace(habitat_baselines=SimpleNamespace(rl=SimpleNamespace(ddppo=SimpleNamespace(train_encoder=False))))


def _frozen_setup(hb, kind, seed=5):
    """native frozen policy + storage holding a random rollout whose visual_features are the encoder's (eval mode)"""
    from habitat_lab_b200.common import spaces
    from habitat_lab_b200.rl.single_agent_access_mgr import get_rollout_obs_space

    obs_space, act_space = _spaces(spaces, kind)
    torch.manual_seed(seed)
    pol = hb.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, resnet_baseplanes=32,
                                  normalize_visual_inputs=True, **CONFIGS[kind])
    rmv = pol.net.visual_encoder.running_mean_and_var
    rmv._mean.uniform_(0.3, 0.6)
    rmv._var.uniform_(0.02, 0.1)
    rmv._count.fill_(64.0)
    for p in pol.net.visual_encoder.parameters():
        p.requires_grad_(False)
    pol.to(DEV)
    space = get_rollout_obs_space(obs_space, pol, _frozen_cfg())
    st = hb.RolloutStorage(T, N, space, act_space, pol)
    st.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    b = st.buffers
    for k, v in b["observations"].items():
        if k == "visual_features":
            continue
        if v.dtype == torch.uint8:
            v.copy_(torch.randint(0, 256, v.shape, generator=g, device=DEV))
        elif v.dtype == torch.int32:
            v.copy_(torch.randint(0, 6, v.shape, generator=g, device=DEV))
        elif v.dtype == torch.int64:
            v.copy_(torch.randint(0, 21, v.shape, generator=g, device=DEV))
        else:
            v.copy_(torch.rand(v.shape, generator=g, device=DEV) * 2 - 0.5)
    b["recurrent_hidden_states"].copy_(torch.randn(b["recurrent_hidden_states"].shape, generator=g, device=DEV) * 0.1)
    b["masks"].copy_(torch.rand(b["masks"].shape, generator=g, device=DEV) > 0.1)
    b["rewards"].copy_(torch.randn(b["rewards"].shape, generator=g, device=DEV))
    b["value_preds"].copy_(torch.randn(b["value_preds"].shape, generator=g, device=DEV))
    b["action_log_probs"].copy_(-torch.rand(b["action_log_probs"].shape, generator=g, device=DEV) * 2)
    b["actions"].copy_(torch.randint(0, 4, b["actions"].shape, generator=g, device=DEV))
    b["prev_actions"].copy_(torch.randint(0, 4, b["prev_actions"].shape, generator=g, device=DEV))
    pol.eval()
    for t in range(T + 1):
        pol.encode_visual_features(b["observations"][t], b["observations"]["visual_features"][t])
    st.current_rollout_step_idxs = [T]
    next_value = torch.randn(N, 1, generator=g, device=DEV)
    return pol, st, next_value, space, act_space


def _reference_update(state_dict, st, next_value, kind, seed):
    """the reference PPO.update on the CPU: same weights, buffers and cached features, encoder frozen like
    SingleAgentAccessMgr._create_policy does it (single_agent_access_mgr.py:230-232)"""
    R = ref_shim.ref()
    obs_space, act_space = _spaces(R.spaces, kind)
    ref = R.PointNavResNetPolicy(obs_space, act_space, hidden_size=512, resnet_baseplanes=32,
                                 normalize_visual_inputs=True, **CONFIGS[kind])
    ref.load_state_dict(state_dict)
    for p in ref.visual_encoder.parameters():
        p.requires_grad_(False)
    ref.train()
    space = R.spaces.Dict({"visual_features": R.spaces.Box(np.finfo(np.float32).min, np.finfo(np.float32).max,
                                                          tuple(ref.visual_encoder.output_shape), np.float32),
                           **obs_space.spaces})
    rst = R.RolloutStorage(T, N, space, act_space, ref)
    for k, v in st.buffers["observations"].items():
        rst.buffers["observations"][k].copy_(v.cpu())
    for k in ("recurrent_hidden_states", "masks", "rewards", "value_preds", "action_log_probs", "actions", "prev_actions"):
        rst.buffers[k].copy_(st.buffers[k].cpu())
    rst.current_rollout_step_idxs = [T]
    rst.compute_returns(next_value.cpu(), True, 0.99, 0.95)
    ppo = R.PPO(ref, **PPO_KW)
    torch.manual_seed(seed)
    return ppo.update(rst), ref, ppo


@pytest.mark.skipif(not ref_shim.reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("kind", [2, 3])
def test_frozen_update_vs_reference(hb, kind, monkeypatch):
    from habitat_lab_b200.rl import resnet_policy as rp

    pol, st, next_value, _, _ = _frozen_setup(hb, kind)
    sd0 = {k: v.detach().cpu().clone() for k, v in pol.state_dict().items()}
    enc_before = {k: v.clone() for k, v in pol.state_dict().items() if k.startswith("net.visual_encoder.")}
    ppo = hb.PPO(pol, **PPO_KW)
    st.compute_returns(next_value, True, 0.99, 0.95)
    pol.train()

    def refuse(*a, **k):
        raise AssertionError("the visual encoder ran during a frozen-encoder update")
    monkeypatch.setattr(rp.EncoderEngine, "forward", refuse)
    monkeypatch.setattr(rp.EncoderEngine, "backward", refuse)
    monkeypatch.setattr(rp.PointNavResNetPolicy, "_visual_prep", refuse)
    torch.manual_seed(2000 + kind)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        metrics = ppo.update(st)
        torch.cuda.synchronize()
    kernels = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert any("gather_rows" in k for k in kernels), sorted(kernels)
    assert not [k for k in kernels if ENCODER_KERNELS.search(k.lower())], sorted(kernels)

    ref_metrics, ref, ref_ppo = _reference_update(sd0, st, next_value, kind, 2000 + kind)
    print(kind, "frozen update got", metrics, "ref", ref_metrics)
    for k in ("value_loss", "action_loss", "dist_entropy"):
        assert metrics[k] == pytest.approx(ref_metrics[k], rel=5e-3, abs=5e-4), k
    assert metrics["grad_norm"] == pytest.approx(ref_metrics["grad_norm"], rel=3e-2), "grad_norm"
    sd, ref_sd = pol.state_dict(), ref.state_dict()
    n_steps = PPO_KW["ppo_epoch"] * PPO_KW["num_mini_batch"]
    for k, p in pol.named_parameters():
        if p.requires_grad:
            worst = 2 * 2.5e-4 * n_steps * math.sqrt(p.numel())
            assert sd[k].float().norm().item() == pytest.approx(ref_sd[k].norm().item(), rel=1e-3,
                                                                abs=0.25 * worst + 1e-5), k
    for k, v in enc_before.items():   # weights and RunningMeanAndVar buffers: bit for bit
        assert torch.equal(sd[k], v), k
    # one Adam state per trainable parameter, in the reference's order: the two state_dicts load into each other
    osd = ppo.optimizer.state_dict()
    assert len(osd["state"]) == len(ref_ppo.optimizer.state_dict()["state"])
    ref_ppo.optimizer.load_state_dict({"state": {i: {kk: vv.cpu() for kk, vv in s.items()} for i, s in osd["state"].items()},
                                       "param_groups": osd["param_groups"]})


class _Recorder:
    """PPOTrainer whose _init_train keeps what the first encode left behind"""

    @staticmethod
    def make(cfg):
        from habitat_lab_b200.rl.ppo_trainer import PPOTrainer

        class Rec(PPOTrainer):
            def _init_train(self):
                super()._init_train()
                obs = self.rollouts.buffers["observations"]
                self.slot0 = {k: v[0].clone() for k, v in obs.items()}
                self.count0 = float(self.actor_critic.net.visual_encoder.running_mean_and_var._count)
                self.ptrs = self._ptrs()

            def _ptrs(self):
                out = {}
                for k, v in self.rollouts.buffers.items():
                    for kk, vv in (v.items() if isinstance(v, dict) else [("", v)]):
                        out[(k, kk)] = vv.data_ptr()
                return out

        return Rec(cfg)


def _trainer_cfg(tmp_path=None, **ddppo):
    from habitat_lab_b200.rl.ppo_trainer import make_config

    cfg = make_config(num_environments=N, num_updates=2, height=H, width=W, num_steps=T, ddppo=ddppo)
    if tmp_path is not None:
        cfg.habitat_baselines.checkpoint_interval = 1
        cfg.habitat_baselines.checkpoint_folder = str(tmp_path)
    return cfg


@pytest.fixture(scope="module")
def frozen_runs(hb):
    runs = []
    for _ in range(2):
        tr = _Recorder.make(_trainer_cfg(train_encoder=False))
        losses = tr.train()
        torch.cuda.synchronize()
        runs.append((tr, losses))
    return runs


def test_trainer_caches_encoder_output(hb, frozen_runs):
    tr, losses = frozen_runs[0]
    pol = tr.actor_critic
    b = tr.rollouts.buffers
    obs = b["observations"]
    assert tr.ptrs == tr._ptrs(), "the storage tensors must keep their addresses"
    for k in ("value_loss", "action_loss", "dist_entropy", "grad_norm"):
        assert math.isfinite(losses[k]), (k, losses)
    # RunningMeanAndVar: updated by the first (training-mode) encode only, over the N first observations
    assert tr.count0 == N
    assert float(pol.net.visual_encoder.running_mean_and_var._count) == N
    pol.eval()
    out = torch.empty_like(obs["visual_features"][0])
    pol.encode_visual_features(tr.slot0, out)
    assert torch.equal(out, tr.slot0["visual_features"]), "slot 0 (training-mode encode)"
    for t in range(T + 1):
        pol.encode_visual_features(obs[t], out)
        assert torch.equal(out, obs["visual_features"][t]), t
        # act reads the cached features: the same numbers as running the encoder
        step = (b["recurrent_hidden_states"][t], b["prev_actions"][t], b["masks"][t])
        raw = {k: v for k, v in obs[t].items() if k != "visual_features"}
        a = pol.act(obs[t], *step, deterministic=True)
        r = pol.act(raw, *step, deterministic=True)
        for x, y in ((a.values, r.values), (a.actions, r.actions), (a.action_log_probs, r.action_log_probs),
                     (a.rnn_hidden_states, r.rnn_hidden_states)):
            assert torch.equal(x, y), t
        v1 = pol.get_value(obs[t], *step)
        assert torch.equal(v1, pol.get_value(raw, *step))
    # the captured actor takes the cached features, and refuses a step that would re-run the frozen encoder
    step = (b["recurrent_hidden_states"][1], b["prev_actions"][1], b["masks"][1])
    with pytest.raises(hb.Hb200Error, match="frozen"):
        hb.GraphedActor(pol, {k: v for k, v in obs[1].items() if k != "visual_features"}, *step, deterministic=True)
    ga = hb.GraphedActor(pol, dict(obs[1]), *step, deterministic=True)
    for t in range(T + 1):
        st_t = (b["recurrent_hidden_states"][t], b["prev_actions"][t], b["masks"][t])
        got = ga(dict(obs[t]), *st_t)
        ref = pol.act(obs[t], *st_t, deterministic=True)
        assert torch.equal(got.values, ref.values) and torch.equal(got.actions, ref.actions), t


def test_frozen_training_is_run_to_run_identical(hb, frozen_runs):
    (a, la), (b, lb) = frozen_runs
    assert la == lb
    for (k, x), (_, y) in zip(a.actor_critic.state_dict().items(), b.actor_critic.state_dict().items()):
        assert torch.equal(x, y), k
    for k, x in a.rollouts.buffers.items():
        y = b.rollouts.buffers[k]
        for kk in (x.keys() if isinstance(x, dict) else [None]):
            assert torch.equal(x[kk] if kk else x, y[kk] if kk else y), (k, kk)


def test_pretrained_fine_tune_end_to_end(hb, tmp_path):
    first = _Recorder.make(_trainer_cfg(tmp_path / "run1"))
    first.config.habitat_baselines.num_updates = 1
    first.train()
    ck = torch.load(str(tmp_path / "run1" / "ckpt.1.pth"), map_location="cpu", weights_only=False)
    sd = ck["state_dict"]
    path = str(tmp_path / "pretrained.pth")
    torch.save({"state_dict": {"actor_critic." + k: v for k, v in sd.items()}}, path)
    second = _Recorder.make(_trainer_cfg(tmp_path / "run2", pretrained=True, pretrained_weights=path,
                                         train_encoder=False, reset_critic=False))
    second._init_train()
    pol = second.actor_critic
    rmv = "net.visual_encoder.running_mean_and_var."
    for k, v in pol.state_dict().items():   # starts from the checkpoint (the statistics took the first batch)
        if not k.startswith(rmv):
            assert torch.equal(v.cpu(), sd[k]), k
    assert float(pol.state_dict()[rmv + "_count"]) == float(sd[rmv + "_count"]) + N
    losses = second.train()   # builds its agent afresh: the same load + first encode
    for k in ("value_loss", "action_loss", "dist_entropy", "grad_norm"):
        assert math.isfinite(losses[k]), (k, losses)
    pol = second.actor_critic
    after = pol.state_dict()
    for k, p in pol.named_parameters():
        if k.startswith("net.visual_encoder."):
            assert not p.requires_grad and torch.equal(after[k].cpu(), sd[k]), k
    moved = [k for k, p in pol.named_parameters() if p.requires_grad and not torch.equal(after[k].cpu(), sd[k])]
    assert "net.visual_fc.1.weight" in moved and "critic.fc.weight" in moved, moved


def test_frozen_parameters_sit_outside_the_reduced_range(hb):
    pol, st, next_value, _, _ = _frozen_setup(hb, 2)
    flat = pol.flatten_parameters_()
    frozen = [p for p in pol.parameters() if not p.requires_grad]
    assert frozen and all(p.grad is None for p in frozen)
    assert flat["grads"].numel() == flat["n"] and flat["plist"] == [p for p in pol.parameters() if p.requires_grad]
    base = flat["params"].data_ptr()
    assert all(p.data_ptr() >= base + 4 * flat["n"] for p in frozen)
    assert 0 < pol.tail_offset() < flat["n"]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        import habitat_lab_b200 as hb

        hb.load()
        pol, st, next_value, _, _ = _frozen_setup(hb, 2, seed=11 + rank)   # different weights and rollouts per rank
        ppo = hb.DDPPO(pol, **{**PPO_KW, "ppo_epoch": 1, "num_mini_batch": 1})
        ppo.init_distributed(find_unused_params=False)
        flat = pol.flatten_parameters_()
        frozen0 = flat["params"][flat["n"]:].clone()
        st.compute_returns(next_value, True, 0.99, 0.95)
        pol.train()
        ppo.update(st)
        torch.cuda.synchronize()
        q.put((rank, flat["grads"].cpu().numpy(), flat["params"].cpu().numpy(), flat["n"],
               bool(torch.equal(frozen0, flat["params"][flat["n"]:]))))
    except BaseException:
        import traceback
        q.put(("error", rank, traceback.format_exc()[-3000:]))
        raise
    finally:
        dist.destroy_process_group()


def test_frozen_ddppo_two_ranks(hb):
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (one rank per GPU, NCCL)")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    try:
        res = [q.get(timeout=600) for _ in range(2)]
    finally:
        for p in procs:
            p.join(30)
            if p.is_alive():
                p.kill()
    assert all(r[0] != "error" for r in res), [r[2] for r in res if r[0] == "error"]
    r0, r1 = sorted(res, key=lambda r: r[0])
    assert np.array_equal(r0[1], r1[1]), "reduced gradients differ across ranks"
    assert np.array_equal(r0[2], r1[2]), "parameters differ across ranks"
    assert r0[1].size == r0[3], "the gradient buffer (the reduced range) holds the trainable parameters only"
    assert r0[4] and r1[4], "frozen parameters changed"
