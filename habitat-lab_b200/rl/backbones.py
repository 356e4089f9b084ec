"""Parameter holders for every backbone of habitat-baselines/habitat_baselines/rl/ddppo/policy/resnet.py:284-340
(resnet18 / resnet50 / resneXt50 / se_resnet50 / se_resneXt50 / se_resneXt101) with the reference's module names, so
that `state_dict()` keys and shapes interchange with reference checkpoints.

Every backbone here runs on sm_90a kernels: rl/resnet_policy.py's EncoderEngine reads these holders' parameters and runs
the convolutions, GroupNorms and (for se_*) the squeeze-excite branch itself.  The holders perform no computation; they
pin the checkpoint contract (tests/test_host_api.py checks them against the layouts recorded from the real reference)."""
from __future__ import annotations

from typing import List

from torch import nn


def _conv3x3(cin, cout, stride=1, groups=1):
    return nn.Conv2d(cin, cout, 3, stride, 1, bias=False, groups=groups)


def _conv1x1(cin, cout, stride=1):
    return nn.Conv2d(cin, cout, 1, stride, bias=False)


class SE(nn.Module):
    """squeeze-excite gate: global average pool -> Linear(C, C/r) -> ReLU -> Linear(C/r, C) -> Sigmoid (resnet.py:92-110)"""

    def __init__(self, planes: int, r: int = 16):
        super().__init__()
        self.squeeze = nn.AdaptiveAvgPool2d(1)
        self.excite = nn.Sequential(nn.Linear(planes, int(planes / r)), nn.ReLU(True), nn.Linear(int(planes / r), planes),
                                    nn.Sigmoid())


class BasicBlock(nn.Module):
    expansion = 1
    resneXt = False

    def __init__(self, inplanes, planes, ngroups, stride=1, downsample=None, cardinality=1):
        super().__init__()
        self.convs = nn.Sequential(_conv3x3(inplanes, planes, stride, cardinality), nn.GroupNorm(ngroups, planes),
                                   nn.ReLU(True), _conv3x3(planes, planes, groups=cardinality),
                                   nn.GroupNorm(ngroups, planes))
        self.downsample = downsample
        self.stride = stride


class Bottleneck(nn.Module):
    """1x1 -> 3x3 (stride, groups = cardinality) -> 1x1 (x expansion), GroupNorm after each, ReLU after the first two
    (resnet.py:72-89, 113-151)"""
    expansion = 4
    resneXt = False
    has_se = False

    def __init__(self, inplanes, planes, ngroups, stride=1, downsample=None, cardinality=1):
        super().__init__()
        out = planes * self.expansion
        self.convs = nn.Sequential(_conv1x1(inplanes, planes), nn.GroupNorm(ngroups, planes), nn.ReLU(True),
                                   _conv3x3(planes, planes, stride, cardinality), nn.GroupNorm(ngroups, planes),
                                   nn.ReLU(True), _conv1x1(planes, out), nn.GroupNorm(ngroups, out))
        self.downsample = downsample
        self.stride = stride
        if self.has_se:
            self.se = SE(out)


class SEBottleneck(Bottleneck):
    has_se = True


class ResNeXtBottleneck(Bottleneck):
    expansion = 2
    resneXt = True


class SEResNeXtBottleneck(ResNeXtBottleneck):
    has_se = True


class ResNetBackbone(nn.Module):
    """stem (7x7 s2 conv + GroupNorm + ReLU, then a parameter-free 3x3 s2 max pool) and four stages; the ResNeXt
    variants double the base width of the stages (resnet.py:196-281)."""

    def __init__(self, in_channels: int, base_planes: int, ngroups: int, block, layers: List[int], cardinality: int = 1):
        super().__init__()
        self.conv1 = nn.Sequential(nn.Conv2d(in_channels, base_planes, 7, 2, 3, bias=False),
                                   nn.GroupNorm(ngroups, base_planes), nn.ReLU(True))
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        self.cardinality = cardinality
        inplanes = base_planes
        if block.resneXt:
            base_planes *= 2
        for li, (mult, n_blocks) in enumerate(zip((1, 2, 4, 8), layers), start=1):
            planes, stride = base_planes * mult, (1 if li == 1 else 2)
            blocks = []
            for b in range(n_blocks):
                s = stride if b == 0 else 1
                ds = None
                if b == 0 and (s != 1 or inplanes != planes * block.expansion):
                    ds = nn.Sequential(_conv1x1(inplanes, planes * block.expansion, s),
                                       nn.GroupNorm(ngroups, planes * block.expansion))
                # reference quirk (resnet.py:256-271): only the FIRST block of a stage receives the cardinality; the
                # remaining blocks of a ResNeXt stage are built with dense (groups = 1) 3x3 convolutions
                blocks.append(block(inplanes, planes, ngroups, s, ds, cardinality=cardinality if b == 0 else 1))
                inplanes = planes * block.expansion
            setattr(self, f"layer{li}", nn.Sequential(*blocks))
        self.final_channels = inplanes
        self.final_spatial_compress = 1.0 / 32


_SPECS = {
    "resnet18": (BasicBlock, [2, 2, 2, 2], False),
    "resnet50": (Bottleneck, [3, 4, 6, 3], False),
    "resneXt50": (ResNeXtBottleneck, [3, 4, 6, 3], True),
    "se_resnet50": (SEBottleneck, [3, 4, 6, 3], False),
    "se_resneXt50": (SEResNeXtBottleneck, [3, 4, 6, 3], True),
    "se_resneXt101": (SEResNeXtBottleneck, [3, 4, 23, 3], True),
}


def make_backbone(name: str, in_channels: int, base_planes: int, ngroups: int) -> ResNetBackbone:
    """`getattr(resnet, name)(in_channels, base_planes, ngroups)` of the reference (resnet_policy.py:110-121); the
    ResNeXt variants use cardinality = base_planes / 2 (resnet.py:308-339)."""
    if name not in _SPECS:
        raise ValueError(f"unknown backbone {name!r}; known: {sorted(_SPECS)}")
    block, layers, grouped = _SPECS[name]
    return ResNetBackbone(in_channels, base_planes, ngroups, block, layers,
                          cardinality=int(base_planes / 2) if grouped else 1)
