"""CPU checks of the squeeze-excite backbones (se_resnet50 / se_resneXt50 / se_resneXt101): the engine builds for every
sensor set a user would train them on, routes every convolution through a layer the GPU parity table tests, and the
policy loads a reference-layout backbone state dict."""
import pytest

SE_BACKBONES = ["se_resnet50", "se_resneXt50", "se_resneXt101"]
SENSORS = ["rgb", "rgbd", "objectnav"]


def _policy(backbone, sensors):
    import habitat_lab_b200 as hb
    from habitat_lab_b200 import synthetic as syn

    spaces = {"rgbd": syn.pointnav_spaces(256, 256), "objectnav": syn.objectnav_spaces(256, 256, 6, 21)}
    if sensors == "rgb":
        obs, act = syn.pointnav_spaces(256, 256)
        obs.spaces.pop("depth")
        spaces["rgb"] = (obs, act)
    return hb.PointNavResNetPolicy(*spaces[sensors], hidden_size=512, num_recurrent_layers=1, rnn_type="GRU",
                                   resnet_baseplanes=32, backbone=backbone, normalize_visual_inputs=True)


@pytest.mark.parametrize("sensors", SENSORS)
@pytest.mark.parametrize("backbone", SE_BACKBONES)
def test_se_engine_builds_and_is_covered(backbone, sensors):
    from habitat_lab_b200.rl.resnet_policy import EncoderEngine, ResNetEncoder
    from test_gpu_deep_encoders import LAYER_TABLE
    from test_reduction_order import _family

    pol = _policy(backbone, sensors)
    n_blocks = 33 if backbone == "se_resneXt101" else 16
    rows = set()
    for enc in [m for m in pol.modules() if isinstance(m, ResNetEncoder)]:
        eng = EncoderEngine(enc, allow_s2d=False)   # the generic prep's routing (the stem as a gather conv)
        assert len(eng.se) == len(eng.blocks) == n_blocks and all(s is not None for s in eng.se)
        for (convs, _), ex in zip(eng.blocks, eng.se):
            assert ex[0].in_features == convs[-1].co and ex[0].out_features == convs[-1].co // 16
        for c in eng.convs:
            rows.add((c.ci_real, c.ci, c.co, c.k, c.stride, c.pad, c.in_hw[0], c.conv_groups, c.groups,
                      _family(eng, c)))
    missing = rows - set(LAYER_TABLE)
    assert not missing, f"{backbone} / {sensors} builds layers the GPU parity table does not test: {sorted(missing)}"


def test_se_resnext50_loads_a_reference_layout_state_dict():
    import torch

    from habitat_lab_b200.rl.backbones import make_backbone

    pol = _policy("se_resneXt50", "rgb")
    torch.manual_seed(3)
    ref = make_backbone("se_resneXt50", 3, 32, 16)
    sd = {k: torch.randn_like(v) if v.is_floating_point() else v for k, v in ref.state_dict().items()}
    bb = pol.net.visual_encoder.backbone
    assert set(bb.state_dict()) == set(sd)
    bb.load_state_dict(sd, strict=True)
    for k, v in bb.state_dict().items():
        assert torch.equal(v, sd[k]), k
