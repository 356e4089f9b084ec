"""CPU: the cube-map projection tables (common/projection.py) against the reference's converters, the restatement
(tests/projection_reference.py) against the reference transformers' forward and against float64, the recorded
reference outputs, and the transformers' config handling, observation spaces and refusals (no GPU)."""
import logging
import os
import sys
import types

import pytest
import torch

import projection_reference as R
from oracle import ref_shim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "projection.pt")
FISH = (180, (0.2, 0.2, 0.2))


@pytest.fixture(scope="module")
def ref_ot():
    if not ref_shim.reference_available():
        pytest.skip("reference tree not available")
    ref_shim.install()
    if "habitat.core.logging" not in sys.modules:
        sys.modules["habitat.core.logging"] = types.ModuleType("habitat.core.logging")
        sys.modules["habitat.core.logging"].logger = logging.getLogger("habitat")
    import habitat_baselines.common.obs_transformers as m

    return m


@pytest.fixture(scope="module")
def ot():
    import habitat_lab_b200  # noqa: F401
    from habitat_lab_b200.common import obs_transformers

    return obs_transformers


@pytest.fixture(scope="module")
def P():
    import habitat_lab_b200  # noqa: F401
    from habitat_lab_b200.common import projection

    return projection


def _same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.reshape(-1).view(torch.uint8),
                                                                     b.reshape(-1).view(torch.uint8))


@pytest.mark.parametrize("case", ["c2e_256x512", "c2e_64x128", "c2f_default", "c2f_200x300", "e2c_256"])
def test_tables_bit_identical_to_reference(ref_ot, P, case):
    ref, mine = {
        "c2e_256x512": lambda: (ref_ot.Cube2Equirect(256, 512), P.cube_to_equirect(256, 512)),
        "c2e_64x128": lambda: (ref_ot.Cube2Equirect(64, 128), P.cube_to_equirect(64, 128)),
        "c2f_default": lambda: (ref_ot.CubeMap2Fisheye(list("abcdef"), (256, 256), *FISH).converter,
                                P.cube_to_fisheye(256, 256, *FISH)),
        "c2f_200x300": lambda: (ref_ot.CubeMap2Fisheye(list("abcdef"), (200, 300), *FISH).converter,
                                P.cube_to_fisheye(200, 300, *FISH)),
        "e2c_256": lambda: (ref_ot.Equirect2Cube(256, 256), P.equirect_to_cube(256, 256)),
    }[case]()
    assert _same_bits(ref.grids, mine.grids)
    assert _same_bits(ref.input_zfactor, mine.in_zfactor)
    assert _same_bits(ref.output_zfactor, mine.out_zfactor)
    # the table holds the one grid point that is not 2, and its input
    tab = mine.table()
    g = mine.grids.permute(1, 0, 2, 3, 4)                                  # [n_out, n_in, h, w, 2]
    claimed = (g != 2).all(-1)
    assert bool((claimed.sum(1) <= 1).all())
    assert torch.equal(torch.where(claimed.any(1), claimed.int().argmax(1), -1), tab[..., 2].long())
    for o in range(g.shape[0]):
        for i in range(g.shape[1]):
            m = claimed[o, i]
            assert torch.equal(tab[o][m][:, :2], g[o, i][m])


def _faces(key, n, B, hw, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for i in range(n):
        shape = (B, *hw, 3 if dtype == torch.uint8 else 1)
        if dtype == torch.uint8:
            out[f"{key}_{i}"] = torch.randint(0, 256, shape, generator=g, dtype=dtype)
        elif dtype == torch.int32:
            out[f"{key}_{i}"] = torch.randint(-2 ** 30, 2 ** 30, shape, generator=g, dtype=dtype)
        else:
            out[f"{key}_{i}"] = torch.rand(shape, generator=g) * 10
    return out


# (ours, reference, face size) per transformer; depth faces of Cube2Equirect must be 256
def _pair(kind, ot, ref_ot, uuids, hw_out):
    if kind == "c2e":
        return ot.CubeMap2Equirect(uuids, hw_out), ref_ot.CubeMap2Equirect(uuids, hw_out)
    if kind == "c2f":
        return ot.CubeMap2Fisheye(uuids, hw_out, *FISH), ref_ot.CubeMap2Fisheye(uuids, hw_out, *FISH)
    return ot.Equirect2CubeMap(uuids, hw_out), ref_ot.Equirect2CubeMap(uuids, hw_out)


@pytest.mark.parametrize("kind,key,dtype,face,hw_out", [
    ("c2e", "rgb", torch.uint8, (20, 20), (32, 64)),
    ("c2e", "depth", torch.float32, (256, 256), (16, 32)),
    ("c2e", "semantic", torch.int32, (9, 9), (24, 48)),
    ("c2f", "rgb", torch.uint8, (13, 13), (40, 56)),
    ("c2f", "depth", torch.float32, (40, 56), (40, 56)),
    ("c2f", "semantic", torch.int32, (7, 7), (30, 30)),
    ("e2c", "rgb", torch.uint8, (32, 64), (12, 12)),
    ("e2c", "depth", torch.float32, (40, 80), (12, 16)),
    ("e2c", "semantic", torch.int32, (16, 32), (12, 12)),
])
def test_restatement_bit_identical_to_reference_forward(ot, ref_ot, kind, key, dtype, face, hw_out):
    n = 1 if kind == "e2c" else 6
    obs = _faces(key, n, 2, face, dtype, seed=len(key) * 10 + len(kind))
    ours, ref = _pair(kind, ot, ref_ot, list(obs), hw_out)
    want = ref({k: v.clone() for k, v in obs.items()})[f"{key}_0"]
    got = R.transform(ours, obs)[f"{key}_0"]
    assert _same_bits(got, want.contiguous())


@pytest.mark.parametrize("kind,key,dtype,face,hw_out", [
    ("c2e", "rgb", torch.uint8, (64, 64), (64, 128)),
    ("c2e", "depth", torch.float32, (256, 256), (32, 64)),
    ("c2f", "rgb", torch.uint8, (48, 48), (48, 64)),
    ("e2c", "depth", torch.float32, (64, 128), (16, 16)),
])
def test_restatement_within_float64_bar_and_perturbed_grid_misses(ot, kind, key, dtype, face, hw_out):
    n = 1 if kind == "e2c" else 6
    obs = _faces(key, n, 2, face, dtype, seed=7)
    t = {"c2e": lambda: ot.CubeMap2Equirect(list(obs), hw_out),
         "c2f": lambda: ot.CubeMap2Fisheye(list(obs), hw_out, *FISH),
         "e2c": lambda: ot.Equirect2CubeMap(list(obs), hw_out)}[kind]()
    _, uuids, is_depth = t.groups[0]
    faces = [obs[u] for u in uuids]
    got = R.stitch_float(t.stitch, faces, is_depth).double()
    want = R.bilinear64(t.stitch, faces, is_depth)
    bar = R.error_bar(t.stitch, faces, is_depth)
    err = float((got - want).abs().max())
    assert err <= bar, (err, bar)
    # a grid moved by a tenth of a face pixel breaks the bar
    bumped = t.stitch.grids.clone()
    bumped[bumped != 2] += 0.2 / max(face)
    saved, t.stitch.grids = t.stitch.grids, bumped
    try:
        err_b = float((R.stitch_float(t.stitch, faces, is_depth).double() - want).abs().max())
    finally:
        t.stitch.grids = saved
    assert err_b > 10 * bar, (err_b, bar)


def _golden_transformer(ot, name, obs):
    kind, hw_out, fish, _, _, _ = R.GOLDEN_CASES[name]
    return {"c2e": lambda: ot.CubeMap2Equirect(list(obs), hw_out),
            "c2f": lambda: ot.CubeMap2Fisheye(list(obs), hw_out, *fish),
            "e2c": lambda: ot.Equirect2CubeMap(list(obs), hw_out)}[kind]()


@pytest.mark.parametrize("name", list(R.GOLDEN_CASES))
def test_restatement_on_recorded_tables_matches_recorded_reference(name):
    """The recorded outputs (tests/golden/make_golden_projection.py) follow from the recorded tables and depth factors
    by the restatement's arithmetic, on any host: these are what the GPU kernel is held to."""
    rec = torch.load(GOLDEN)[name]
    _, _, _, key, _, _ = R.GOLDEN_CASES[name]
    obs = R.golden_faces(name)
    assert sum(float(v.double().sum()) for v in obs.values()) == rec["faces_sum"]
    faces = [obs[f"{key}_{i}"] for i in range(rec["n_in"])]
    assert _same_bits(R.stitch(R.recorded_stitch(rec), faces, key == "depth"), rec["out"])


@pytest.mark.parametrize("name", list(R.GOLDEN_CASES))
def test_tables_against_recorded_host(ot, name):
    """The tables' last bits follow torch.sqrt, which rounds differently on different CPUs (MKL picks its code path
    per CPU).  On a host whose torch.sqrt rounds the recorded probe the recording's way, the package rebuilds the
    recorded tables bit for bit; elsewhere every pixel keeps its input (up to 0.1 % of pixels at face boundaries) and
    moves by at most 2^-20 in normalised units, a few float32 ulps."""
    golden = torch.load(GOLDEN)
    rec = golden[name]
    t = _golden_transformer(ot, name, R.golden_faces(name))
    key = R.GOLDEN_CASES[name][3]
    table = t.stitch.table()
    zfs = [(None if z is None or key != "depth" else z[:, 0], rec[k])
           for z, k in ((t.stitch.in_zfactor, "in_zf"), (t.stitch.out_zfactor, "out_zf"))]
    if torch.equal(torch.sqrt(R.sqrt_probe_input()), golden["sqrt_probe"]):
        assert _same_bits(table, rec["table"])
        assert all(_same_bits(a, b) for a, b in zfs)
        return
    same = table[..., 2] == rec["table"][..., 2]
    assert int((~same).sum()) <= table[..., 2].numel() // 1000
    assert float((table[..., :2] - rec["table"][..., :2]).abs()[same].max()) <= 2.0 ** -20
    for a, b in zfs:
        assert (a is None) == (b is None)
        if a is not None:
            assert float(((a - b) / b).abs().max()) <= 2.0 ** -20


def test_config_defaults_and_from_config(ot, P):
    c = ot.Cube2EqConfig()
    assert (c.type, c.height, c.width, c.sensor_uuids) == ("CubeMap2Equirect", 256, 512, list(P.CUBE_FACES))
    f = ot.Cube2FishConfig()
    assert (f.type, f.height, f.width, f.fov, tuple(f.params)) == ("CubeMap2Fisheye", 256, 256, 180, (0.2, 0.2, 0.2))
    e = ot.Eq2CubeConfig()
    assert (e.type, e.height, e.width, e.sensor_uuids) == ("Equirect2CubeMap", 256, 256, list(P.CUBE_FACES))
    assert ot.Cube2EqConfig().sensor_uuids is not c.sensor_uuids
    t = ot.CubeMap2Equirect.from_config(c)
    assert t.img_shape == (256, 512) and t.target_uuids == ["BACK"] and not t.channels_last
    assert t.groups == [("BACK", list(P.CUBE_FACES), False)]
    t = ot.CubeMap2Fisheye.from_config(types.SimpleNamespace(**vars(f), target_uuids=["FRONT"]))
    assert t.target_uuids == ["FRONT"] and t.img_shape == (256, 256)
    twelve = [f"depth_{i}" for i in range(6)] + [f"rgb_{i}" for i in range(6)]
    t = ot.CubeMap2Equirect(twelve, (64, 128))
    assert t.target_uuids == ["depth_0", "rgb_0"]
    assert [(g[0], g[2]) for g in t.groups] == [("depth_0", True), ("rgb_0", False)]
    t = ot.Equirect2CubeMap.from_config(types.SimpleNamespace(**{**vars(e), "sensor_uuids": ["pano", "pano_depth"]}))
    assert t.target_uuids == ["pano"] and [g[2] for g in t.groups] == [False]   # sensor_uuids[::6]


def _config(**transforms):
    from habitat_lab_b200.rl.ppo_trainer import make_config

    return make_config(height=256, width=256, obs_transforms=transforms or None, cubemap="depth")


def test_active_transforms_and_observation_space(ot):
    from habitat_lab_b200.synthetic import cubemap_spaces

    uuids = [f"depth_{i}" for i in range(6)]
    active = ot.get_active_obs_transforms(_config(c=ot.Cube2EqConfig(height=256, width=256, sensor_uuids=uuids)))
    assert [type(t) for t in active] == [ot.CubeMap2Equirect]
    raw, _ = cubemap_spaces(256, "depth")
    space = ot.apply_obs_transforms_obs_space(raw, active)
    assert list(space.spaces) == list(raw.spaces)
    assert tuple(space["depth_0"].shape) == (256, 256, 1) and tuple(space["depth_1"].shape) == (256, 256, 1)
    fish = ot.get_active_obs_transforms(_config(c=ot.Cube2FishConfig(height=128, width=128, sensor_uuids=uuids)))
    assert tuple(ot.apply_obs_transforms_obs_space(cubemap_spaces(128, "depth")[0], fish)["depth_0"].shape) == \
        (128, 128, 1)
    plan = ot.ObsTransformPlan(active, raw)
    assert plan and plan.keys == {} and plan.projected == ("depth_0",)
    rgb, _ = cubemap_spaces(64, "rgb")
    assert tuple(ot.apply_obs_transforms_obs_space(rgb, [ot.CubeMap2Equirect(list(rgb.spaces)[:6], (32, 64))])
                 ["rgb_0"].shape) == (32, 64, 3)


def test_refusals(ot):
    from habitat_lab_b200 import Hb200Error
    from habitat_lab_b200.synthetic import cubemap_spaces

    uuids = [f"depth_{i}" for i in range(6)]
    for cls, args in ((ot.CubeMap2Equirect, ((64, 128),)), (ot.CubeMap2Fisheye, ((64, 64), *FISH)),
                      (ot.Equirect2CubeMap, ((64, 64),))):
        with pytest.raises(NotImplementedError, match="channels_last"):
            cls(uuids, *args, channels_last=True)
    with pytest.raises(ValueError, match="multiple of 6"):
        ot.CubeMap2Equirect(uuids[:5], (64, 128))
    with pytest.raises(ValueError, match="not one of its input"):
        ot.CubeMap2Equirect(uuids, (64, 128), target_uuids=["rgb"])
    # faces smaller than 3x3, before anything is launched
    rgb = {f"rgb_{i}": torch.zeros(1, 2, 2, 3, dtype=torch.uint8) for i in range(6)}
    with pytest.raises(Hb200Error, match="at least 3x3"):
        ot.CubeMap2Equirect(list(rgb), (8, 16))(rgb)
    # depth faces of another size than the stitch's cube cameras (256 for Cube2Equirect, the fisheye's size)
    with pytest.raises(Hb200Error, match="depth faces of 128x128"):
        ot.CubeMap2Equirect(uuids, (64, 128)).transform_observation_space(cubemap_spaces(128, "depth")[0])
    with pytest.raises(Hb200Error, match="depth faces of 128x128"):
        ot.CubeMap2Fisheye(uuids, (64, 64), *FISH)({u: torch.zeros(1, 128, 128, 1) for u in uuids})
    with pytest.raises(Hb200Error, match="depth faces"):
        ot.ObsTransformPlan([ot.CubeMap2Fisheye(uuids, (64, 64), *FISH)], cubemap_spaces(128, "depth")[0])
    # config nodes that carry no camera rig; AddVirtualKeys keeps its refusal
    for name in ("CubeMap2Equirect", "CubeMap2Fisheye", "Equirect2CubeMap"):
        with pytest.raises(NotImplementedError, match=f"{name}.*sensor_uuids"):
            ot.get_active_obs_transforms(_config(x=types.SimpleNamespace(type=name)))
    with pytest.raises(NotImplementedError, match="AddVirtualKeys"):
        ot.get_active_obs_transforms(_config(x=types.SimpleNamespace(type="AddVirtualKeys")))
    # the plan's combinations
    raw, _ = cubemap_spaces(256, "depth")
    c2e = ot.CubeMap2Equirect(uuids, (256, 256))
    with pytest.raises(NotImplementedError, match="Equirect2CubeMap"):
        ot.ObsTransformPlan([ot.Equirect2CubeMap(["depth_0"], (64, 64))], raw)
    with pytest.raises(NotImplementedError, match="at most one projection"):
        ot.ObsTransformPlan([c2e, ot.CubeMap2Fisheye(uuids, (256, 256), *FISH)], raw)
    with pytest.raises(NotImplementedError, match="depth_0.*resized or cropped"):
        ot.ObsTransformPlan([c2e, ot.CenterCropper(128, trans_keys=("depth_0",))], raw)
    with pytest.raises(NotImplementedError, match="depth_3.*resized or cropped"):
        ot.ObsTransformPlan([ot.ResizeShortestEdge(128, trans_keys=("depth_3",)), c2e], raw)
    # a projection next to a resize of keys it does not touch is accepted
    both = dict(raw.spaces)
    both["rgb"] = cubemap_spaces(64, "rgb")[0]["rgb_0"]
    from habitat_lab_b200.common import spaces

    plan = ot.ObsTransformPlan([c2e, ot.ResizeShortestEdge(32)], spaces.Dict(both))
    assert set(plan.keys) == {"rgb"} and plan.projected == ("depth_0",)
