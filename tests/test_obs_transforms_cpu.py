"""CPU: the observation-transform restatement (tests/obs_transform_reference.py) against the reference's
ResizeShortestEdge / CenterCropper, the observation-space shapes of this project's transformers against the
reference's, and the host-side plan and config handling (no GPU)."""
import logging
import sys
import types

import numpy as np
import pytest
import torch

import obs_transform_reference as R
from oracle import ref_shim


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


def _images(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return {
        "rgb": torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8),
        "depth": torch.rand((B, H, W, 1), generator=g),
        "semantic": torch.randint(0, 2 ** 30 + 1, (B, H, W, 1), generator=g, dtype=torch.int32),
        "rgba": torch.randint(0, 256, (B, H, W, 4), generator=g, dtype=torch.uint8),
        "feat": torch.rand((B, H, W, 4), generator=g) * 100 - 50,
        "pointgoal_with_gps_compass": torch.rand((B, 2), generator=g),
    }


def _bits(t):
    return t.contiguous().view(torch.uint8) if t.dtype != torch.uint8 else t.contiguous()


KEYS = ("rgb", "depth", "semantic", "rgba", "feat")


@pytest.mark.parametrize("H,W", [(480, 640), (640, 480), (256, 256), (512, 512), (128, 128), (392, 520),
                                 (257, 300), (300, 257)])
@pytest.mark.parametrize("size,crop", [(256, None), (None, (256, 256)), (256, (256, 256)), (128, (96, 120))])
def test_restatement_is_bit_identical_to_reference(ref_ot, H, W, size, crop):
    if crop is not None and size is None and (crop[0] > H or crop[1] > W):
        pytest.skip("crop larger than the image")
    obs = _images(2, H, W, seed=H * 7 + W)
    ref = dict(obs)
    if size is not None:
        ref = ref_ot.ResizeShortestEdge(size, True, KEYS, "semantic")(ref)
    if crop is not None:
        if size is not None and min(ref["rgb"].shape[1:3]) < max(crop):
            pytest.skip("crop larger than the resized image: the reference returns a degenerate slice")
        ref = ref_ot.CenterCropper(crop, True, KEYS)(ref)
    got = R.transform(obs, size, crop, KEYS)
    for k in obs:
        assert got[k].shape == ref[k].shape and got[k].dtype == ref[k].dtype, k
        assert torch.equal(_bits(got[k]), _bits(ref[k])), k
    # unbatched HWC input goes through the same ops
    one = R.transform({k: v[0] for k, v in obs.items()}, size, crop, KEYS)
    assert all(torch.equal(_bits(one[k]), _bits(got[k][0])) for k in KEYS)


def _space_pair(ref_ot, h, w):
    from habitat_lab_b200.common import spaces

    rs = ref_shim.ref().spaces
    mk = lambda S: S.Dict({  # noqa: E731
        "rgb": S.Box(0, 255, (h, w, 3), np.uint8),
        "depth": S.Box(0.0, 1.0, (h, w, 1), np.float32),
        "semantic": S.Box(0, 2 ** 30, (h, w, 1), np.int32),
        "pointgoal_with_gps_compass": S.Box(-1.0, 1.0, (2,), np.float32),
    })
    return mk(spaces), mk(rs)


def test_transform_observation_space_matches_reference(ref_ot, ot):
    n255 = 0
    for size in (128, 256):
        ours_r, ref_r = ot.ResizeShortestEdge(size), ref_ot.ResizeShortestEdge(size)
        ours_c, ref_c = ot.CenterCropper(size), ref_ot.CenterCropper(size)
        for short in range(1, 1025):
            for h, w in ((short, short + short // 3 + 1), (short + short // 2 + 1, short)):
                a, b = _space_pair(ref_ot, h, w)
                a, b = ours_r.transform_observation_space(a), ref_r.transform_observation_space(b)
                for k in b.spaces:
                    assert tuple(a[k].shape) == tuple(b[k].shape), (size, h, w, k)
                    assert a[k].dtype == b[k].dtype
                n255 += min(a["rgb"].shape[:2]) == size - 1
                a, b = ours_c.transform_observation_space(a), ref_c.transform_observation_space(b)
                assert all(tuple(a[k].shape) == tuple(b[k].shape) for k in b.spaces), (size, h, w)
    assert n255 > 0  # the "255 instead of 256" cases are in the sweep


def test_shortest_edge_rule_is_float64():
    assert R.resized_hw(392, 520, 256) == (255, 339)
    assert sum(R.resized_hw(s, s, 256)[0] == 255 for s in range(1, 4097)) == 505
    from habitat_lab_b200.common.obs_transformers import resized_hw

    assert all(resized_hw(s, s + 77, z) == R.resized_hw(s, s + 77, z) for s in range(1, 4097) for z in (128, 256))


def _config(**transforms):
    from habitat_lab_b200.rl.ppo_trainer import make_config

    return make_config(height=480, width=640, obs_transforms=transforms or None)


def test_plan_for_objectnav_pair(ot):
    from habitat_lab_b200 import ops
    from habitat_lab_b200.synthetic import objectnav_spaces

    cfg = _config(resize_shortest_edge=ot.ResizeShortestEdgeConfig(), center_cropper=ot.CenterCropperConfig())
    active = ot.get_active_obs_transforms(cfg)
    assert [type(t) for t in active] == [ot.ResizeShortestEdge, ot.CenterCropper]
    raw, _ = objectnav_spaces(480, 640)
    space = ot.apply_obs_transforms_obs_space(raw, active)
    assert [tuple(space[k].shape) for k in ("rgb", "depth", "semantic")] == [(256, 256, 3), (256, 256, 1),
                                                                             (256, 256, 1)]
    assert tuple(space["gps"].shape) == (2,) and tuple(raw["rgb"].shape) == (480, 640, 3)
    plan = ot.ObsTransformPlan(active, raw)
    # 480x640 -> 256x341, centre 256x256 window at column 341 // 2 - 128 = 42
    assert plan.keys == {"rgb": (ops.OBS_AREA, (256, 341), (0, 42), (256, 256)),
                         "depth": (ops.OBS_AREA, (256, 341), (0, 42), (256, 256)),
                         "semantic": (ops.OBS_NEAREST, (256, 341), (0, 42), (256, 256))}
    crop_only = ot.ObsTransformPlan([ot.CenterCropper((200, 300))], raw)
    assert crop_only.keys["semantic"] == (ops.OBS_COPY, (480, 640), (140, 170), (200, 300))
    assert not ot.ObsTransformPlan([], raw) and ot.get_active_obs_transforms(_config()) == []


def test_unsupported_configurations_raise(ot):
    from habitat_lab_b200 import Hb200Error
    from habitat_lab_b200.synthetic import pointnav_spaces

    raw, _ = pointnav_spaces(480, 640)
    with pytest.raises(NotImplementedError, match="CenterCropper.*ResizeShortestEdge"):
        ot.ObsTransformPlan([ot.CenterCropper(256), ot.ResizeShortestEdge(256)], raw)
    with pytest.raises(NotImplementedError, match="ResizeShortestEdge.*ResizeShortestEdge"):
        ot.ObsTransformPlan([ot.ResizeShortestEdge(256), ot.ResizeShortestEdge(128)], raw)
    with pytest.raises(NotImplementedError, match="channels_last"):
        ot.ResizeShortestEdge(256, channels_last=False)
    with pytest.raises(NotImplementedError, match="channels_last"):
        ot.CenterCropper(256, channels_last=False)
    for name in ("AddVirtualKeys", "CubeMap2Equirect", "CubeMap2Fisheye", "Equirect2CubeMap"):
        with pytest.raises(NotImplementedError, match=name):
            ot.get_active_obs_transforms(_config(x=types.SimpleNamespace(type=name)))
    with pytest.raises(ValueError):
        ot.get_active_obs_transforms(_config(x=types.SimpleNamespace(type="NoSuchTransform")))
    # a crop larger than the resized image (392x520 -> 255x339) is refused when the plan is built
    with pytest.raises(Hb200Error, match="larger"):
        ot.ObsTransformPlan([ot.ResizeShortestEdge(256), ot.CenterCropper(256)], pointnav_spaces(392, 520)[0])
    with pytest.raises(Hb200Error, match="larger"):
        ot.CenterCropper((256, 256))({"rgb": torch.zeros(1, 255, 339, 3, dtype=torch.uint8)})
    with pytest.raises(NotImplementedError, match="5-D"):
        ot.CenterCropper(8)({"rgb": torch.zeros(1, 2, 16, 16, 3, dtype=torch.uint8)})


def test_registry_lookup(ot):
    from habitat_lab_b200.common.baseline_registry import baseline_registry

    assert baseline_registry.get_obs_transformer("ResizeShortestEdge") is ot.ResizeShortestEdge
    assert baseline_registry.get_obs_transformer("CenterCropper") is ot.CenterCropper
    r = ot.ResizeShortestEdge.from_config(ot.ResizeShortestEdgeConfig(size=128, trans_keys=("rgb",)))
    assert (r._size, r.trans_keys, r.semantic_key) == (128, ("rgb",), "semantic")
    c = ot.CenterCropper.from_config(ot.CenterCropperConfig(height=100, width=120))
    assert c._size == (100, 120)
