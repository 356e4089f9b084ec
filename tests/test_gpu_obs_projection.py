"""GPU: the cube-map projection kernel (ops.obs_project, via CubeMap2Equirect / CubeMap2Fisheye / Equirect2CubeMap
and ObsTransformPlan) is byte-identical to the recorded reference outputs (tests/golden/projection.pt) and to the CPU
restatement on the same grid (tests/projection_reference.py), writes nothing outside its output, repeats bit for bit
and refuses bad input before launching; the trainer stitches a synthetic six-camera depth rig into every storage slot
in place and trains."""
import math
import os

import pytest
import torch

import projection_reference as R

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "projection.pt")
FISH = (180, (0.2, 0.2, 0.2))


def _faces(key, n, B, hw, dtype, seed, C=None):
    g = torch.Generator().manual_seed(seed)
    C = C or (3 if dtype == torch.uint8 else 1)
    out = {}
    for i in range(n):
        shape = (B, *hw, C)
        if dtype == torch.uint8:
            out[f"{key}_{i}"] = torch.randint(0, 256, shape, generator=g, dtype=dtype)
        elif dtype == torch.int32:
            out[f"{key}_{i}"] = torch.randint(-2 ** 30, 2 ** 30, shape, generator=g, dtype=dtype)
        else:
            out[f"{key}_{i}"] = torch.rand(shape, generator=g) * 10
    return out


def _bits(t):
    return t.detach().cpu().reshape(-1).view(torch.uint8)


def _assert_same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
    g, w = _bits(got), _bits(want)
    if not torch.equal(g, w):
        bad = (g != w).nonzero()
        pytest.fail(f"{what}: {bad.shape[0]} bytes differ, first at {bad[0].tolist()}")


def _gpu(obs):
    return {k: v.cuda() for k, v in obs.items()}


def _make(kind, uuids, hw, fish=FISH):
    from habitat_lab_b200.common import obs_transformers as ot

    return {"c2e": lambda: ot.CubeMap2Equirect(uuids, hw), "c2f": lambda: ot.CubeMap2Fisheye(uuids, hw, *fish),
            "e2c": lambda: ot.Equirect2CubeMap(uuids, hw)}[kind]()


def _check_forward(hb, t, obs, what, launches=1):
    n0 = hb.load().hb200_launch_count()
    got = t(_gpu(obs))
    torch.cuda.synchronize()
    assert hb.load().hb200_launch_count() - n0 == launches
    want = R.transform(t, obs)
    for target in want:
        _assert_same(got[target], want[target], f"{what} {target}")
    return got


@pytest.mark.parametrize("name", list(R.GOLDEN_CASES))
def test_kernel_matches_recorded_reference(hb, name):
    """The kernel on the reference's recorded table and depth factors gives the reference's recorded bytes (the
    tables are recorded because their last bits depend on the host that builds them)."""
    from habitat_lab_b200 import ops

    rec = torch.load(GOLDEN)[name]
    key = R.GOLDEN_CASES[name][3]
    obs = _gpu(R.golden_faces(name))
    faces = [obs[f"{key}_{i}"] for i in range(rec["n_in"])]
    dst = torch.full(tuple(rec["out"].shape), 7, dtype=rec["out"].dtype, device="cuda")
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    ops.obs_project([(faces, dst, rec["table"].cuda(), dev(rec["in_zf"]), dev(rec["out_zf"]))])
    _assert_same(dst, rec["out"], name)


def test_rgb_depth_int_cubes_in_one_launch(hb):
    obs = {**_faces("rgb", 6, 4, (256, 256), torch.uint8, 1), **_faces("depth", 6, 4, (256, 256), torch.float32, 2),
           **_faces("semantic", 6, 4, (256, 256), torch.int32, 3)}
    t = _make("c2e", list(obs), (256, 512))
    assert [g[2] for g in t.groups] == [False, True, False]
    _check_forward(hb, t, obs, "three cubes")


@pytest.mark.parametrize("B", [1, 37, 256])
def test_batch_sizes(hb, B):
    obs = _faces("rgb", 6, B, (128, 128), torch.uint8, 10 + B)
    _check_forward(hb, _make("c2e", list(obs), (256, 512)), obs, f"B={B}")


@pytest.mark.parametrize("kind,hw,key,dtype,face", [
    ("c2e", (256, 256), "rgb", torch.uint8, (64, 64)),
    ("c2e", (256, 256), "depth", torch.float32, (256, 256)),
    ("c2f", (256, 256), "rgb", torch.uint8, (96, 96)),
    ("c2f", (256, 256), "depth", torch.float32, (256, 256)),
    ("c2f", (200, 300), "rgb", torch.uint8, (64, 64)),
    ("c2f", (200, 300), "semantic", torch.int32, (50, 50)),
    ("c2f", (200, 300), "depth", torch.float32, (200, 300)),
    ("e2c", (256, 256), "depth", torch.float32, (256, 512)),
    ("e2c", (128, 96), "rgb", torch.uint8, (256, 512)),
    ("e2c", (64, 64), "feat", torch.float32, (64, 128)),
])
def test_shapes_and_dtypes(hb, kind, hw, key, dtype, face):
    n = 1 if kind == "e2c" else 6
    obs = _faces(key, n, 3, face, dtype, 20, C=4 if key == "feat" else None)
    t = _make(kind, list(obs), hw)
    got = _check_forward(hb, t, obs, f"{kind} {hw} {key}")
    if kind == "e2c":   # the reference's [6 * B, h, w, C], with the output z-factors for depth
        assert tuple(got[f"{key}_0"].shape) == (3 * 6, *hw, obs[f"{key}_0"].shape[-1])
        assert (t.stitch.out_zfactor is not None) and t.groups[0][2] == (key == "depth")


def _job(t, obs, dst):
    return t.jobs(obs, {t.target_uuids[0]: dst})


def test_writes_only_its_output_and_repeats(hb):
    from habitat_lab_b200 import ops

    obs = _gpu(_faces("depth", 6, 5, (256, 256), torch.float32, 30))
    t = _make("c2f", list(obs), (256, 256))
    buf = torch.full((3, 5, 256, 256, 1), float("nan"), device="cuda")   # slot 1 of a 3-slot buffer
    before = buf.clone()
    ops.obs_project(_job(t, obs, buf[1]))
    torch.cuda.synchronize()
    want = R.transform(t, {k: v.cpu() for k, v in obs.items()})["depth_0"]
    _assert_same(buf[1], want, "slot 1")
    _assert_same(buf[0], before[0], "slot 0")
    _assert_same(buf[2], before[2], "slot 2")
    first = buf[1].clone()
    buf[1].fill_(-7.0)
    ops.obs_project(_job(t, obs, buf[1]))
    _assert_same(buf[1], first, "second run")


def test_bad_input_raises_before_launch(hb):
    from habitat_lab_b200 import Hb200Error, ops

    obs = _gpu(_faces("rgb", 6, 2, (16, 16), torch.uint8, 40))
    t = _make("c2e", list(obs), (32, 64))
    table, _, _ = t.device_tables(torch.device("cuda", torch.cuda.current_device()))
    faces = [obs[f"rgb_{i}"] for i in range(6)]
    dst = torch.full((2, 32, 64, 3), 7, dtype=torch.uint8, device="cuda")
    n0 = hb.load().hb200_launch_count()
    bad = [
        [(faces, dst.float(), table, None, None)],                                   # output dtype
        [(faces[:5] + [faces[5][:1]], dst, table, None, None)],                      # a face of another batch
        [([f[:, :2, :2] .contiguous() for f in faces], dst, table, None, None)],     # faces below 3x3
        [(faces, dst[:, :16], table, None, None)],                                   # output size
        [(faces, dst, table[..., :2].contiguous(), None, None)],                     # table layout
        [(faces, dst, table, torch.ones(6, 8, 8, device="cuda"), None)],             # z-factor size
        [(faces, dst, table.cpu(), None, None)],                                     # table on the host
        [(faces + faces[:1], dst, table, None, None)],                               # seven faces
        [(faces, dst, table, None, None)] * 9,                                       # nine targets
    ]
    for jobs in bad:
        with pytest.raises(Hb200Error):
            ops.obs_project(jobs)
    torch.cuda.synchronize()
    assert hb.load().hb200_launch_count() == n0 and bool((dst == 7).all())


def _smooth_cube(B, n):
    """Six n x n faces of a smooth function of the viewing direction, in [0, 1]."""
    from habitat_lab_b200.common import projection

    faces = {}
    for i, cam in enumerate(projection.cube_cameras(n, n)):
        d = cam.unproject()[0]                                                     # [n, n, 3] world rays
        v = 0.5 + 0.25 * torch.sin(3 * d[..., 0]) * torch.cos(2 * d[..., 1]) + 0.2 * d[..., 2]
        faces[f"cube_{i}"] = v[None, :, :, None].expand(B, n, n, 1).contiguous()
    return faces


def test_round_trip_cube_equirect_cube(hb):
    from habitat_lab_b200.common import obs_transformers as ot

    faces = _smooth_cube(2, 256)
    uuids = list(faces)
    c2e = ot.CubeMap2Equirect(uuids, (256, 512))
    e2c = ot.Equirect2CubeMap(c2e.target_uuids, (256, 256))
    out = e2c(c2e({k: v.cuda() for k, v in faces.items()}))[uuids[0]]             # [6 * B, 256, 256, 1]
    inp = torch.flatten(torch.stack([faces[k] for k in uuids], dim=1), end_dim=1).cuda()
    blur = torch.nn.AvgPool2d(5, 3, 2)
    diff = (blur(out.permute(0, 3, 1, 2)) - blur(inp.permute(0, 3, 1, 2))).abs()
    assert diff.mean().item() < 0.01


# ---- the trainer --------------------------------------------------------------------------------------------------
def _trainer(transform, monkeypatch=None, record=None):
    from habitat_lab_b200.rl import ppo_trainer as PT

    cfg = PT.make_config(num_environments=4, num_updates=1, height=256, width=256, num_steps=6, cubemap="depth",
                         obs_transforms={"cube": transform})
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


def _transforms():
    from habitat_lab_b200.common.obs_transformers import Cube2EqConfig, Cube2FishConfig

    uuids = [f"depth_{i}" for i in range(6)]
    return [Cube2EqConfig(height=256, width=256, sensor_uuids=uuids), Cube2FishConfig(sensor_uuids=uuids)]


@pytest.mark.parametrize("which", [0, 1], ids=["equirect", "fisheye"])
def test_trainer_stitches_into_storage(hb, monkeypatch, which):
    from habitat_lab_b200 import ops

    record, dsts = [], []
    tr = _trainer(_transforms()[which], monkeypatch, record)
    orig = ops.obs_project
    monkeypatch.setattr(ops, "obs_project", lambda jobs: (dsts.append([j[1].data_ptr() for j in jobs]),
                                                           orig(jobs))[1])
    tr._init_train()
    ob = tr.rollouts.buffers["observations"]
    assert tuple(ob["depth_0"].shape) == (7, 4, 256, 256, 1) and tuple(ob["depth_5"].shape) == (7, 4, 256, 256, 1)
    assert tr.actor_critic.net.visual_encoder._n_input_channels == 6
    inserted = []
    ins = tr.rollouts.insert
    monkeypatch.setattr(tr.rollouts, "insert", lambda **kw: (inserted.append(set(kw["next_observations"].keys())),
                                                             ins(**kw))[1])
    n0 = hb.load().hb200_launch_count()
    for _ in range(6):
        tr._rollout_step()
    torch.cuda.synchronize()
    assert hb.load().hb200_launch_count() > n0
    assert len(record) == 7 and dsts == [[ob["depth_0"][t].data_ptr()] for t in range(7)]
    proj = tr.obs_transforms[0]
    for t in range(7):   # slot t holds the stitch of what the env emitted for it, written in place
        _assert_same(ob["depth_0"][t], R.transform(proj, record[t])["depth_0"], f"slot {t}")
        for k in [f"depth_{i}" for i in range(1, 6)] + ["pointgoal_with_gps_compass"]:
            assert torch.equal(ob[k][t].cpu(), record[t][k]), (t, k)
    assert inserted == [{f"depth_{i}" for i in range(1, 6)} | {"pointgoal_with_gps_compass"}] * 6


def _train_once(which):
    tr = _trainer(_transforms()[which])
    losses = tr.train()
    params = {k: v.detach().cpu().clone() for k, v in tr.actor_critic.state_dict().items()}
    return losses, params


@pytest.mark.parametrize("which", [0, 1], ids=["equirect", "fisheye"])
def test_trainer_trains_and_repeats(hb, which):
    l1, p1 = _train_once(which)
    l2, p2 = _train_once(which)
    assert all(math.isfinite(v) for v in l1.values())
    assert p1.keys() == p2.keys() and all(torch.equal(p1[k], p2[k]) for k in p1)
    assert l1 == l2
