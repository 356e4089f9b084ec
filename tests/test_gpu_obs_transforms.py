"""GPU: the fused observation resample-and-window kernel (ops.obs_resample, via ResizeShortestEdge / CenterCropper
and ObsTransformPlan) is bit-identical to the CPU restatement of the reference (tests/obs_transform_reference.py),
writes nothing outside its window, repeats bit for bit and refuses bad input before writing; the trainer builds
the policy and the storage for the transformed space and fills every storage slot in place."""
import pytest
import torch

import obs_transform_reference as R

pytestmark = pytest.mark.gpu

SHAPES = [(480, 640), (640, 480), (256, 256), (512, 512), (128, 128), (392, 520), (257, 300), (300, 257)]
# every dtype / channel count the kernel takes, all in one launch (the kernel's limit is 8 keys)
KEYS = {"rgb": (torch.uint8, 3), "depth": (torch.float32, 1), "semantic": (torch.int32, 1),
        "rgba": (torch.uint8, 4), "gray": (torch.uint8, 1), "feat3": (torch.float32, 3), "feat4": (torch.float32, 4)}


def _obs(B, H, W, seed, keys=KEYS, dev="cuda"):
    g = torch.Generator(device=dev).manual_seed(seed)
    out = {}
    for k, (dt, c) in keys.items():
        if dt == torch.uint8:
            out[k] = torch.randint(0, 256, (B, H, W, c), generator=g, device=dev, dtype=dt)
        elif dt == torch.int32:
            out[k] = torch.randint(0, 2 ** 30 + 1, (B, H, W, c), generator=g, device=dev, dtype=dt)
        else:
            out[k] = torch.rand((B, H, W, c), generator=g, device=dev) * 20 - 5
    out["pointgoal_with_gps_compass"] = torch.rand((B, 2), generator=g, device=dev)
    return out


def _space(obs):
    from habitat_lab_b200.common import spaces

    return spaces.Dict({k: spaces.Box(0, 1, tuple(v.shape[1:]), v.cpu().numpy().dtype) for k, v in obs.items()})


def _sentinel(shape, dtype, byte):
    es = torch.empty((), dtype=dtype).element_size()
    return torch.full((*shape[:-1], shape[-1] * es), byte, dtype=torch.uint8, device="cuda").view(dtype)


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t if t.dtype == torch.uint8 else t.view(torch.uint8)


def _assert_same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
    g, w = _bits(got), _bits(want)
    if not torch.equal(g, w):
        bad = (g != w).nonzero()
        pytest.fail(f"{what}: {bad.shape[0]} bytes differ, first at {bad[0].tolist()}")


def _ops(size, crop):
    from habitat_lab_b200.common.obs_transformers import CenterCropper, ResizeShortestEdge

    keys = tuple(KEYS)
    active = []
    if size is not None:
        active.append(ResizeShortestEdge(size, trans_keys=keys))
    if crop is not None:
        active.append(CenterCropper(crop, trans_keys=keys))
    return active


def _run_plan(obs, active):
    """One fused launch into fresh buffers (sentinel-filled) through ObsTransformPlan."""
    from habitat_lab_b200.common.obs_transformers import ObsTransformPlan, apply_obs_transforms_obs_space

    raw = _space(obs)
    space = apply_obs_transforms_obs_space(raw, active)
    plan = ObsTransformPlan(active, raw)
    B = next(iter(obs.values())).shape[0]
    out = {k: _sentinel((B, *space[k].shape), obs[k].dtype, 0x5A) for k in plan.keys}
    rest = plan.apply_(obs, out)
    assert set(rest) == {"pointgoal_with_gps_compass"}
    return out


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("op", ["resize", "crop", "resize_crop"])
def test_all_keys_one_launch_bit_exact(hb, H, W, op):
    size = 256 if op != "crop" else None
    crop = {"resize": None, "crop": (min(H, 200), min(W, 230)), "resize_crop": (200, 230)}[op]
    if op == "resize_crop" and (H, W) == (392, 520):
        crop = (255, 255)   # the resized short edge is 255
    obs = _obs(4, H, W, seed=H * 1000 + W)
    n0 = hb.load().hb200_launch_count()
    out = _run_plan(obs, _ops(size, crop))
    assert hb.load().hb200_launch_count() - n0 == 1
    want = R.transform({k: v.cpu() for k, v in obs.items()}, size, crop, tuple(KEYS))
    for k in out:
        _assert_same(out[k], want[k], f"{op} {H}x{W} {k}")


@pytest.mark.parametrize("B", [1, 4, 37, 256])
def test_batch_sizes_config3_set(hb, B):
    keys = {k: KEYS[k] for k in ("rgb", "depth", "semantic")}
    obs = _obs(B, 480, 640, seed=B, keys=keys)
    out = _run_plan(obs, _ops(256, (256, 256)))
    want = R.transform({k: v.cpu() for k, v in obs.items()}, 256, (256, 256))
    for k in keys:
        _assert_same(out[k], want[k], f"B={B} {k}")


def test_transformer_forward_matches_restatement(hb):
    """The classes' own forward: ResizeShortestEdge runs the kernel over the full window (4-D and 3-D input),
    CenterCropper returns the reference's slice view."""
    from habitat_lab_b200.common.obs_transformers import CenterCropper, ResizeShortestEdge

    obs = _obs(3, 300, 257, seed=5)
    cpu = {k: v.cpu() for k, v in obs.items()}
    got = ResizeShortestEdge(128, trans_keys=tuple(KEYS))(dict(obs))
    for k in KEYS:
        _assert_same(got[k], R.transform(cpu, 128, None, (k,))[k], f"resize {k}")
    one = ResizeShortestEdge(96, trans_keys=("depth", "semantic"))({k: v[1] for k, v in obs.items()})
    for k in ("depth", "semantic"):
        _assert_same(one[k], R.resize(cpu[k][1], 96, R.mode_for(k)), f"resize HWC {k}")
    src = obs["rgb"]
    cropped = CenterCropper((100, 90), trans_keys=("rgb",))({"rgb": src})["rgb"]
    assert cropped.data_ptr() == src[:, 150 - 50, 128 - 45].data_ptr()  # a view, as in the reference
    _assert_same(cropped, R.crop(cpu["rgb"], (100, 90)), "crop view")


def test_direct_load_path_and_upsampling(hb):
    """Rows too wide to stage in shared memory (4096 x 4 f32) take the direct-load path; 37 -> 100 upsamples."""
    from habitat_lab_b200.common.obs_transformers import ResizeShortestEdge

    keys = {"feat4": KEYS["feat4"], "rgb": KEYS["rgb"], "semantic": KEYS["semantic"]}
    obs = _obs(2, 300, 4096, seed=11, keys=keys)
    out = _run_plan(obs, [ResizeShortestEdge(100, trans_keys=tuple(keys))])
    want = R.transform({k: v.cpu() for k, v in obs.items()}, 100, None, tuple(keys))
    for k in keys:
        _assert_same(out[k], want[k], f"direct {k}")
    obs = _obs(3, 37, 53, seed=12, keys=keys)
    out = _run_plan(obs, [ResizeShortestEdge(100, trans_keys=tuple(keys))])
    want = R.transform({k: v.cpu() for k, v in obs.items()}, 100, None, tuple(keys))
    for k in keys:
        _assert_same(out[k], want[k], f"upsample {k}")


def test_slot_write_leaves_other_bytes_and_repeats(hb):
    from habitat_lab_b200 import ops

    T, N, t = 5, 4, 2
    obs = _obs(N, 480, 640, seed=3, keys={k: KEYS[k] for k in ("rgb", "depth", "semantic")})
    bufs = {k: _sentinel((T + 1, N, 256, 256, v.shape[-1]), v.dtype, 0xA7) for k, v in obs.items() if v.dim() == 4}
    jobs = lambda: [(obs[k], bufs[k][t + 1], ops.OBS_NEAREST if k == "semantic" else ops.OBS_AREA,  # noqa: E731
                     (256, 341), (0, 42)) for k in bufs]
    ops.obs_resample(jobs())
    want = R.transform({k: v.cpu() for k, v in obs.items()}, 256, (256, 256))
    first = {k: _bits(v).clone() for k, v in bufs.items()}
    for k, v in bufs.items():
        _assert_same(v[t + 1], want[k], f"slot {k}")
        others = torch.cat([_bits(v[:t + 1]).reshape(-1), _bits(v[t + 2:]).reshape(-1)])
        assert bool((others == 0xA7).all()), k
    ops.obs_resample(jobs())
    assert all(torch.equal(_bits(v), first[k]) for k, v in bufs.items())


def test_bad_input_raises_before_writing(hb):
    from habitat_lab_b200 import Hb200Error, ops
    from habitat_lab_b200.common.obs_transformers import CenterCropper, ResizeShortestEdge

    src = torch.randint(0, 256, (2, 64, 80, 3), device="cuda", dtype=torch.uint8)
    dst = torch.full((2, 32, 32, 3), 7, device="cuda", dtype=torch.uint8)
    n0 = hb.load().hb200_launch_count()
    bad = [
        [(src.transpose(1, 2), dst, ops.OBS_AREA, (32, 40), (0, 0))],            # non-contiguous input
        [(src, dst, ops.OBS_AREA, (32, 40), (1, 0))],                            # window past the bottom
        [(src, dst, ops.OBS_AREA, (32, 40), (0, 9))],                            # window past the right edge
        [(src, dst, ops.OBS_COPY, (32, 40), (0, 0))],                            # copy cannot resize
        [(src[None], dst[None], ops.OBS_AREA, (32, 40), (0, 0))],                # 5-D
        [(src.cpu(), dst, ops.OBS_AREA, (32, 40), (0, 0))],                      # not on the device
        [(src.to(torch.int64), dst.to(torch.int64), ops.OBS_NEAREST, (32, 40), (0, 0))],   # dtype
        [(src, dst[:1], ops.OBS_AREA, (32, 40), (0, 0))],                        # batch mismatch
    ]
    for jobs in bad:
        with pytest.raises(Hb200Error):
            ops.obs_resample(jobs)
    with pytest.raises(Hb200Error, match="larger"):
        CenterCropper((65, 10))({"rgb": src})
    with pytest.raises(Hb200Error):
        ResizeShortestEdge(32, trans_keys=("rgb",))({"rgb": src.transpose(1, 2)})
    with pytest.raises(NotImplementedError):
        ResizeShortestEdge(32, trans_keys=("rgb",))({"rgb": src[None]})
    with pytest.raises(NotImplementedError):
        ResizeShortestEdge(32, channels_last=False)
    torch.cuda.synchronize()
    assert hb.load().hb200_launch_count() == n0 and bool((dst == 7).all())


# ---- the trainer --------------------------------------------------------------------------------------------------
def _trainer(monkeypatch=None, record=None):
    from habitat_lab_b200.common.obs_transformers import CenterCropperConfig, ResizeShortestEdgeConfig
    from habitat_lab_b200.rl import ppo_trainer as PT

    cfg = PT.make_config(num_environments=4, num_updates=1, height=480, width=640, num_steps=6,
                         obs_transforms={"resize_shortest_edge": ResizeShortestEdgeConfig(),
                                         "center_cropper": CenterCropperConfig()})
    if record is None:
        return PT.PPOTrainer(cfg)
    orig = PT.SyntheticVectorEnvFactory.construct_envs

    def construct(self, *a, **k):
        env = orig(self, *a, **k)
        reset, step = env.reset, env.step

        def rec_reset():
            obs = reset()
            record.append({k: v.detach().cpu().clone() for k, v in obs.items()})
            return obs

        def rec_step(actions):
            obs, *rest = step(actions)
            record.append({k: v.detach().cpu().clone() for k, v in obs.items()})
            return (obs, *rest)

        env.reset, env.step = rec_reset, rec_step
        return env

    monkeypatch.setattr(PT.SyntheticVectorEnvFactory, "construct_envs", construct)
    return PT.PPOTrainer(cfg)


def test_trainer_writes_transformed_obs_into_storage(hb, monkeypatch):
    from habitat_lab_b200 import ops

    record, dsts = [], []
    tr = _trainer(monkeypatch, record)
    orig = ops.obs_resample
    monkeypatch.setattr(ops, "obs_resample", lambda keys: (dsts.append({j[1].data_ptr() for j in keys}),
                                                            orig(keys))[1])
    tr._init_train()
    assert tuple(tr._env_spec.observation_space["rgb"].shape) == (256, 256, 3)
    assert tuple(tr._env_spec.observation_space["depth"].shape) == (256, 256, 1)
    assert tuple(tr.actor_critic.observation_space["rgb"].shape) == (256, 256, 3)
    ob = tr.rollouts.buffers["observations"]
    assert tuple(ob["rgb"].shape) == (7, 4, 256, 256, 3) and tuple(ob["depth"].shape) == (7, 4, 256, 256, 1)
    ptrs = {k: v.data_ptr() for k, v in ob.items()}
    inserted = []
    ins = tr.rollouts.insert
    monkeypatch.setattr(tr.rollouts, "insert", lambda **kw: (inserted.append(set(kw["next_observations"].keys())),
                                                             ins(**kw))[1])
    for _ in range(6):
        tr._rollout_step()
    torch.cuda.synchronize()
    assert len(record) == 7 and len(dsts) == 7
    for t in range(7):   # slot t holds the transform of what the env emitted for it, written in place
        assert dsts[t] == {ob["rgb"][t].data_ptr(), ob["depth"][t].data_ptr()}
        want = R.transform(record[t], 256, (256, 256))
        for k in ("rgb", "depth"):
            _assert_same(ob[k][t], want[k], f"slot {t} {k}")
        assert torch.equal(ob["pointgoal_with_gps_compass"][t].cpu(), record[t]["pointgoal_with_gps_compass"])
    assert inserted == [{"pointgoal_with_gps_compass"}] * 6
    assert {k: v.data_ptr() for k, v in ob.items()} == ptrs


def _train_once():
    tr = _trainer()
    losses = tr.train()
    ob = {k: v.detach().cpu().clone() for k, v in tr.rollouts.buffers["observations"].items()}
    params = {k: v.detach().cpu().clone() for k, v in tr.actor_critic.state_dict().items()}
    return losses, ob, params


def test_trainer_trains_and_repeats(hb):
    l1, ob1, p1 = _train_once()
    l2, ob2, p2 = _train_once()
    assert all(v == v for v in l1.values())
    assert ob1.keys() == ob2.keys() and all(torch.equal(_bits(ob1[k]), _bits(ob2[k])) for k in ob1)
    assert p1.keys() == p2.keys() and all(torch.equal(p1[k], p2[k]) for k in p1)
    assert l1 == l2
