"""PointNavResNetPolicy on the hb200 kernels.

Mirrors the reference policy's interface and checkpoint layout
(habitat-baselines/habitat_baselines/rl/ddppo/policy/resnet_policy.py:50-162, 165-276, 394-767;
rl/ppo/policy.py:252-424): `from_config`, `act`, `get_value`, `evaluate_actions`, the properties the
trainer / agent-access-manager read, and a state_dict with the reference's exact key names and
shapes (the torch.nn modules below are parameter holders + initialisers only; their forward is
never called).  All arithmetic runs in libhb200.so:

  forward  : prep (u8/f32 rollout rows -> pooled, normalised bf16 NHWC) -> wgmma conv stack with
             GroupNorm statistics fused in the epilogue -> fp32 linears / masked LSTM -> heads
  backward : hand-written, layer by layer, into one flat fp32 gradient buffer (no autograd)

There is no CPU / PyTorch fallback: tensors must live on a CUDA device.
"""
from __future__ import annotations

import math
import os
from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch
from torch import nn

from .. import ops
from .._lib import Hb200Error
from ..common import spaces
from ..common.baseline_registry import baseline_registry
from .backbones import make_backbone

BF16 = torch.bfloat16   # gradients (g, dy, gz) and the dgrad weight images
F16 = torch.float16     # forward values: pooled input, conv outputs, activations, forward weight images
POINTGOAL_UUID = "pointgoal_with_gps_compass"  # IntegratedPointGoalGPSAndCompassSensor.cls_uuid
IMAGEGOAL_UUID = "imagegoal"
VISUAL_FEATURES_KEY = "visual_features"   # PointNavResNetNet.PRETRAINED_VISUAL_FEATURES_KEY: a frozen encoder's output


@dataclass
class PolicyActionData:
    """Subset of rl/ppo/policy.py:47-96 used by the trainer's rollout loop."""
    rnn_hidden_states: Optional[torch.Tensor] = None
    actions: Optional[torch.Tensor] = None
    values: Optional[torch.Tensor] = None
    action_log_probs: Optional[torch.Tensor] = None
    take_actions: Optional[torch.Tensor] = None
    policy_info: Optional[list] = None
    should_inserts: Optional[torch.Tensor] = None

    @property
    def env_actions(self):
        return self.actions if self.take_actions is None else self.take_actions


# ---------------------------------------------------------------------------------------------
# parameter holders (same module tree / names as the reference)
# ---------------------------------------------------------------------------------------------
class RunningMeanAndVar(nn.Module):
    def __init__(self, n_channels: int):
        super().__init__()
        self.register_buffer("_mean", torch.zeros(1, n_channels, 1, 1))
        self.register_buffer("_var", torch.zeros(1, n_channels, 1, 1))
        self.register_buffer("_count", torch.zeros(()))


class ResNetEncoder(nn.Module):
    """Parameter holder with the reference's constructor logic (resnet_policy.py:165-253): every 3-D observation
    except the image goal is a visual key, u8 keys are rescaled by 1 / high, channels are concatenated in
    observation-space order; the spatial / compression rule of :200-240 decides the output shape."""

    def __init__(self, observation_space, baseplanes=32, ngroups=16, normalize_visual_inputs=False,
                 backbone="resnet18"):
        super().__init__()
        self.visual_keys = [k for k, v in observation_space.spaces.items()
                            if len(v.shape) > 1 and k != IMAGEGOAL_UUID]
        self.key_needs_rescaling = {k: None for k in self.visual_keys}
        for k, v in observation_space.spaces.items():
            if v.dtype == np.uint8:
                self.key_needs_rescaling[k] = 1.0 / float(np.max(v.high))
        self._n_input_channels = sum(observation_space.spaces[k].shape[2] for k in self.visual_keys)
        self.key_channels = {k: observation_space.spaces[k].shape[2] for k in self.visual_keys}
        self.running_mean_and_var = (RunningMeanAndVar(self._n_input_channels)
                                     if normalize_visual_inputs else nn.Sequential())
        self.ngroups = ngroups
        if not self.is_blind:
            h, w = observation_space.spaces[self.visual_keys[0]].shape[:2]
            self.in_hw = (h, w)
            self.backbone = make_backbone(backbone, self._n_input_channels, baseplanes, ngroups)
            fh = int(np.ceil((h // 2) * self.backbone.final_spatial_compress))
            fw = int(np.ceil((w // 2) * self.backbone.final_spatial_compress))
            ncomp = int(round(2048 / (fh * fw)))
            self.compression = nn.Sequential(nn.Conv2d(self.backbone.final_channels, ncomp, 3, padding=1, bias=False),
                                             nn.GroupNorm(1, ncomp), nn.ReLU(True))
            self.output_shape = (ncomp, fh, fw)

    @property
    def is_blind(self):
        return self._n_input_channels == 0


class _LSTMStateEncoder(nn.Module):
    def __init__(self, input_size, hidden_size, num_layers):
        super().__init__()
        self.num_recurrent_layers = num_layers * 2
        self.rnn = nn.LSTM(input_size=input_size, hidden_size=hidden_size, num_layers=num_layers)
        for name, p in self.rnn.named_parameters():  # rnn_state_encoder.py:288-293
            if "weight" in name:
                nn.init.orthogonal_(p)
            elif "bias" in name:
                nn.init.constant_(p, 0)


class _GRUStateEncoder(nn.Module):
    def __init__(self, input_size, hidden_size, num_layers=1):
        super().__init__()
        self.num_recurrent_layers = num_layers
        self.rnn = nn.GRU(input_size=input_size, hidden_size=hidden_size, num_layers=num_layers)
        for name, p in self.rnn.named_parameters():  # rnn_state_encoder.py:288-293
            if "weight" in name:
                nn.init.orthogonal_(p)
            elif "bias" in name:
                nn.init.constant_(p, 0)


# sensor uuids (habitat/tasks/nav/nav.py:129-464, object_nav_task.py, instance_image_nav_task.py)
OBJECTGOAL_UUID, GPS_UUID, POINTGOAL_SENSOR_UUID = "objectgoal", "gps", "pointgoal"
HEADING_UUID, PROXIMITY_UUID, COMPASS_UUID = "heading", "proximity", "compass"
INSTANCE_IMAGEGOAL_UUID = "instance_imagegoal"
_GOAL_SENSOR_KEYS = {POINTGOAL_UUID, OBJECTGOAL_UUID, GPS_UUID, POINTGOAL_SENSOR_UUID, HEADING_UUID, PROXIMITY_UUID,
                     COMPASS_UUID, IMAGEGOAL_UUID, INSTANCE_IMAGEGOAL_UUID}


class PointNavResNetNet(nn.Module):
    """Parameter holder + input layout of the reference Net (resnet_policy.py:394-623): one module per sensor with
    the reference's attribute names (checkpoint keys), and `self.segments`: the column layout of the RNN input in the
    reference's concatenation order (:625-763)."""
    PRETRAINED_VISUAL_FEATURES_KEY = VISUAL_FEATURES_KEY

    def __init__(self, observation_space, action_space, hidden_size, num_recurrent_layers, rnn_type, backbone,
                 resnet_baseplanes, normalize_visual_inputs, fuse_keys=None, discrete_actions=True):
        super().__init__()
        if not discrete_actions:
            raise NotImplementedError("continuous prev-action input (gaussian policies) is a 'next' row (SURVEY 8f-4)")
        sp = observation_space.spaces
        self.prev_action_embedding = nn.Embedding(action_space.n + 1, 32)
        if fuse_keys is None:
            fuse_keys = [k for k in sp.keys() if k not in _GOAL_SENSOR_KEYS]
        self._fuse_keys_1d = [k for k in fuse_keys if len(sp[k].shape) == 1]
        segs = []   # (kind, obs key, width, module attr, transform)
        if self._fuse_keys_1d:
            for k in self._fuse_keys_1d:
                segs.append(("raw", k, sp[k].shape[0], None, ops.T_IDENTITY))
        if POINTGOAL_UUID in sp:
            n_goal = sp[POINTGOAL_UUID].shape[0]
            if n_goal not in (2, 3):
                raise AssertionError("Unsupported dimensionality")   # resnet_policy.py:675-677
            self.tgt_embeding = nn.Linear(n_goal + 1, 32)  # sic: the reference's spelling
            segs.append(("linear", POINTGOAL_UUID, 32, "tgt_embeding", ops.T_POLAR2 if n_goal == 2 else ops.T_POLAR3))
        if OBJECTGOAL_UUID in sp:
            self._n_object_categories = int(sp[OBJECTGOAL_UUID].high[0]) + 1
            self.obj_categories_embedding = nn.Embedding(self._n_object_categories, 32)
        if GPS_UUID in sp:
            self.gps_embedding = nn.Linear(sp[GPS_UUID].shape[0], 32)
        if POINTGOAL_SENSOR_UUID in sp:
            self.pointgoal_embedding = nn.Linear(sp[POINTGOAL_SENSOR_UUID].shape[0], 32)
            segs.append(("linear", POINTGOAL_SENSOR_UUID, 32, "pointgoal_embedding", ops.T_IDENTITY))
        if HEADING_UUID in sp:
            assert sp[HEADING_UUID].shape[0] + 1 == 2, "Expected heading with 2D rotation."
            self.heading_embedding = nn.Linear(2, 32)
        if PROXIMITY_UUID in sp:
            self.proximity_embedding = nn.Linear(sp[PROXIMITY_UUID].shape[0], 32)
            segs.append(("linear", PROXIMITY_UUID, 32, "proximity_embedding", ops.T_IDENTITY))
        if HEADING_UUID in sp:
            # the reference indexes the BATCH dimension here (`sensor_observations[0]`, :703-712), which only
            # type-checks for a single frame; per frame this is the same cos / sin feature
            segs.append(("linear", HEADING_UUID, 32, "heading_embedding", ops.T_COSSIN))
        if OBJECTGOAL_UUID in sp:
            segs.append(("embed", OBJECTGOAL_UUID, 32, "obj_categories_embedding", None))
        if COMPASS_UUID in sp:
            assert sp[COMPASS_UUID].shape[0] == 1, "Expected compass with 2D rotation."
            self.compass_embedding = nn.Linear(2, 32)
            segs.append(("linear", COMPASS_UUID, 32, "compass_embedding", ops.T_COSSIN))
        if GPS_UUID in sp:
            segs.append(("linear", GPS_UUID, 32, "gps_embedding", ops.T_IDENTITY))
        self._goal_encoder_uuids = []
        for uuid in (IMAGEGOAL_UUID, INSTANCE_IMAGEGOAL_UUID):
            if uuid in sp:
                genc = ResNetEncoder(spaces.Dict({"rgb": sp[uuid]}), baseplanes=resnet_baseplanes,
                                     ngroups=resnet_baseplanes // 2, normalize_visual_inputs=normalize_visual_inputs,
                                     backbone=backbone)
                setattr(self, f"{uuid}_encoder", genc)
                setattr(self, f"{uuid}_fc", nn.Sequential(nn.Flatten(), nn.Linear(int(np.prod(genc.output_shape)),
                                                                                  hidden_size), nn.ReLU(True)))
                self._goal_encoder_uuids.append(uuid)
                segs.append(("imagegoal", uuid, hidden_size, f"{uuid}_fc", None))
        segs.append(("prev_action", None, 32, "prev_action_embedding", None))
        self._hidden_size = hidden_size
        use_space = spaces.Dict(OrderedDict((k, sp[k]) for k in fuse_keys if len(sp[k].shape) == 3))
        self.visual_encoder = ResNetEncoder(use_space, baseplanes=resnet_baseplanes, ngroups=resnet_baseplanes // 2,
                                            normalize_visual_inputs=normalize_visual_inputs, backbone=backbone)
        if self.visual_encoder.is_blind:
            raise NotImplementedError("blind policies are not implemented")
        self.visual_fc = nn.Sequential(nn.Flatten(), nn.Linear(int(np.prod(self.visual_encoder.output_shape)),
                                                               hidden_size), nn.ReLU(True))
        # column layout of the RNN input: [visual_fc | segments in the reference's cat order]
        col = hidden_size
        self.segments = []
        for kind, key, width, attr, transform in segs:
            self.segments.append(dict(kind=kind, key=key, width=width, attr=attr, transform=transform, col=col))
            col += width
        self.rnn_input_size = col
        if rnn_type.lower() == "lstm":
            self.state_encoder = _LSTMStateEncoder(col, hidden_size, num_recurrent_layers)
        elif rnn_type.lower() == "gru":
            self.state_encoder = _GRUStateEncoder(col, hidden_size, num_recurrent_layers)
        else:
            raise RuntimeError(f"Did not recognize rnn type '{rnn_type}'")  # rnn_state_encoder.py:445
        self.train()

    @property
    def output_size(self):
        return self._hidden_size

    @property
    def is_blind(self):
        return False

    @property
    def num_recurrent_layers(self):
        return self.state_encoder.num_recurrent_layers

    @property
    def recurrent_hidden_size(self):
        return self._hidden_size

    @property
    def perception_embedding_size(self):
        return self._hidden_size


class CategoricalNet(nn.Module):
    def __init__(self, num_inputs, num_outputs):
        super().__init__()
        self.linear = nn.Linear(num_inputs, num_outputs)
        nn.init.orthogonal_(self.linear.weight, gain=0.01)
        nn.init.constant_(self.linear.bias, 0)


class CriticHead(nn.Module):
    def __init__(self, input_size):
        super().__init__()
        self.fc = nn.Linear(input_size, 1)
        nn.init.orthogonal_(self.fc.weight)
        nn.init.constant_(self.fc.bias, 0)


# ---------------------------------------------------------------------------------------------
# observation handle: lets the updater hand the policy the rollout buffers IN PLACE
# ---------------------------------------------------------------------------------------------
class RolloutObservations(dict):
    """dict of full rollout tensors [(T+1)*N, ...] plus `frame_rows` (int32 [B]): the buffer row
    of each minibatch frame.  Replaces the advanced-index gather copy of data_generator
    (common/rollout_storage.py:236-246), 1.9 GB per minibatch at config #2."""

    def __init__(self, tensors: Dict[str, torch.Tensor], frame_rows: torch.Tensor):
        super().__init__(tensors)
        self.frame_rows = frame_rows


def _as_rows(observations, device):
    if isinstance(observations, RolloutObservations):
        return observations, observations.frame_rows
    any_t = next(iter(observations.values()))
    rows = torch.arange(any_t.shape[0], dtype=torch.int32, device=device)
    return observations, rows


# ---------------------------------------------------------------------------------------------
# conv stack engine
# ---------------------------------------------------------------------------------------------
class _Conv:
    """One conv + GroupNorm unit of the encoder: geometry, packed weight images, the kernel family that serves it.
    A grouped conv (ResNeXt's 3x3 with groups = cardinality, resnet.py:72-89) runs as a dense conv over a
    block-diagonal weight: `dense_weight()` expands the [co, ci/g, k, k] parameter, `store_grad()` keeps the diagonal
    blocks of the dense gradient -- copies only, the arithmetic stays on the tensor cores."""

    def __init__(self, conv: nn.Conv2d, gn: nn.GroupNorm, in_hw, ci_pad=None):
        self.w, self.gamma, self.beta = conv.weight, gn.weight, gn.bias
        self.groups = gn.num_groups
        self.conv_groups = conv.groups
        self.co, _, self.k, _ = conv.weight.shape
        self.ci_real = conv.in_channels
        self.ci = ci_pad or self.ci_real
        self.stride, self.pad = conv.stride[0], conv.padding[0]
        self.in_hw = in_hw
        self.out_hw = tuple((d + 2 * self.pad - self.k) // self.stride + 1 for d in in_hw)
        self.wp = self.wt = self.dw_acc = None
        self.halo = False       # stride-1 3x3 layer served by the halo kernels (conv_halo.cu)
        self.halo_w = False     # weight gradient served by the (multi-image tile) halo wgrad kernel
        self.stem_s2d = False   # 7x7 s2 stem as a 4x4 s1 conv over the space-to-depth input
        self.s2_pair = None     # 3x3 stride-2 conv whose block's 1x1 stride-2 downsample conv shares its kernel (conv_s2.cu)
        self.s2_main = None     # ... and the downsample conv's pointer back
        self.dw_s2 = None
        self.wh = self.wht = None
        self._wd = self._gd = None

    def alloc_weights(self, dev, need_dgrad):
        if self.conv_groups > 1:
            self._wd = torch.zeros(self.co, self.ci_real, self.k, self.k, device=dev)
            self._gd = torch.empty_like(self._wd)
        if self.stem_s2d:
            self.wh = torch.empty(16 * 16 * self.co, dtype=F16, device=dev)
            self.dw_acc = torch.empty(16 * 16, self.co, device=dev)
            return
        if self.halo:
            self.wh = torch.empty(9 * self.ci * self.co, dtype=F16, device=dev)
            self.wht = torch.empty(9 * self.ci * self.co, dtype=BF16, device=dev)
            self.dw_acc = torch.empty(9 * self.ci, self.co, device=dev)
            return
        if self.s2_pair is not None:   # images of the concatenated filter [co + co_d, ci, 3, 3] (fwd fp16, dgrad bf16)
            ntot = self.co + self.s2_pair.co
            self.wh = torch.empty(9 * self.ci * ntot, dtype=F16, device=dev)
            self.wht = torch.empty(9 * self.ci * ntot, dtype=BF16, device=dev)
            self._wcat = torch.zeros(ntot, self.ci, 3, 3, device=dev)
            self.dw_s2 = (torch.empty(16 * self.ci, self.co, device=dev)
                          if ops.conv_s2_wgrad_supported(self.ci, self.co, self.in_hw[0], self.in_hw[1]) else None)
        self.wp = torch.empty(ops.packed_weight_elems(self.co, self.ci, self.k, self.k), dtype=F16, device=dev)
        self.wt = (torch.empty(ops.packed_weight_elems(self.ci, self.co, self.k, self.k), dtype=BF16, device=dev)
                   if need_dgrad else None)
        self.dw_acc = torch.empty(self.k * self.k * self.ci, self.co, device=dev)

    def _diag(self, dense):
        g = self.conv_groups
        return dense.view(g, self.co // g, g, self.ci_real // g, self.k, self.k).diagonal(dim1=0, dim2=2)

    def dense_weight(self):
        if self.conv_groups == 1:
            return self.w.data
        g = self.conv_groups
        self._diag(self._wd).copy_(self.w.data.view(g, self.co // g, self.ci_real // g, self.k, self.k).permute(1, 2, 3, 4, 0))
        return self._wd

    def grad_target(self):
        return self.w.grad if self.conv_groups == 1 else self._gd

    def store_grad(self):
        if self.conv_groups > 1:
            g = self.conv_groups
            self.w.grad.view(g, self.co // g, self.ci_real // g, self.k, self.k).copy_(self._diag(self._gd).permute(4, 0, 1, 2, 3))

    def shape(self, B):
        return ops.conv_shape(B, self.in_hw[0], self.in_hw[1], self.ci, self.co, self.k, self.k, self.stride, self.pad)


class SideStream:
    """Second CUDA stream for work nothing on the critical path consumes (weight gradients): the backward pass
    keeps the data-gradient chain on the main stream and lets the weight-gradient kernels of layer k overlap
    the GroupNorm-backward / dgrad kernels of layer k-1.  HB200_NO_SIDE_STREAM=1 runs everything in order."""

    def __init__(self):
        import os
        self.enabled = not os.environ.get("HB200_NO_SIDE_STREAM")
        self.stream = None

    class _Ctx:
        def __init__(self, side):
            self.side, self.cm = side, None

        def __enter__(self):
            sd = self.side
            if not sd.enabled:
                return self
            if sd.stream is None:
                sd.stream = torch.cuda.Stream()
            sd.stream.wait_stream(torch.cuda.current_stream())   # everything enqueued on main so far
            self.cm = torch.cuda.stream(sd.stream)
            self.cm.__enter__()
            return self

        def __exit__(self, *exc):
            if self.cm is not None:
                self.cm.__exit__(*exc)
            return False

    def after_main(self):
        return SideStream._Ctx(self)

    def mark(self):
        """event after the side work enqueued so far (None when disabled: program order already covers it)"""
        if not self.enabled or self.stream is None:
            return None
        ev = torch.cuda.Event()
        ev.record(self.stream)
        return ev

    @staticmethod
    def wait(ev):
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def join(self):
        if self.enabled and self.stream is not None:
            torch.cuda.current_stream().wait_stream(self.stream)


class EncoderEngine:
    """ResNet backbone (BasicBlock or Bottleneck / ResNeXt stages, resnet.py:37-151, 196-281) + compression, forward
    and backward on NHWC activations: forward values fp16 (+ a bf16 twin of every conv input for the weight-gradient
    MMAs), gradients bf16.  Any input size: layers whose shape the halo kernels cannot tile fall back to the gather
    kernels automatically."""

    def __init__(self, enc: ResNetEncoder, allow_s2d: bool = True):
        """allow_s2d: the input prep can write the space-to-depth form the halo stem kernel reads (only the vectorised
        rgb / depth prep does; the generic prep writes plain NHWC and the stem runs as a gather conv)."""
        self.enc = enc
        h, w = enc.in_hw
        self.hp, self.wp_ = h // 2, w // 2
        if enc._n_input_channels > 8:
            raise NotImplementedError(f"{enc._n_input_channels} visual input channels: the stem kernels take up to 8")
        bb = enc.backbone
        self.stem = _Conv(bb.conv1[0], bb.conv1[1], (self.hp, self.wp_), ci_pad=8)
        hw = tuple((d - 1) // 2 + 1 for d in self.stem.out_hw)  # MaxPool2d(3, 2, 1)
        self.pool_hw = hw
        self.blocks = []   # (main-branch convs, downsample conv or None)
        self.se = []       # per block: its SE module's excite Sequential (Linear, ReLU, Linear, Sigmoid), or None
        for li in (1, 2, 3, 4):
            for blk in getattr(bb, f"layer{li}"):
                self.se.append(blk.se.excite if hasattr(blk, "se") else None)
                seq = blk.convs
                pairs = [(i, i + 1) for i in range(0, len(seq), 3)]   # (conv, GroupNorm) positions: 0-1, 3-4 (, 6-7)
                convs, cur = [], hw
                for ci_, gi_ in pairs:
                    c = _Conv(seq[ci_], seq[gi_], cur)
                    convs.append(c)
                    cur = c.out_hw
                cd = _Conv(blk.downsample[0], blk.downsample[1], hw) if blk.downsample is not None else None
                self.blocks.append((convs, cd))
                hw = cur
        self.comp = _Conv(enc.compression[0], enc.compression[1], hw)
        assert self.comp.out_hw == tuple(enc.output_shape[1:]), (self.comp.out_hw, enc.output_shape)
        self.convs: List[_Conv] = ([self.stem] + [c for convs, cd in self.blocks for c in convs + ([cd] if cd else [])]
                                   + [self.comp])
        if not os.environ.get("HB200_NO_HALO"):
            for c in self.convs:
                if c is self.stem:
                    c.stem_s2d = (allow_s2d and c.k == 7 and c.stride == 2 and c.pad == 3 and c.ci_real <= 4 and
                                  self.hp % 2 == 0 and self.wp_ % 2 == 0 and
                                  ops.conv_halo_supported(16, c.co, 4, c.out_hw[0], c.out_hw[1]))
                elif c.k == 3 and c.stride == 1 and c.pad == 1:
                    c.halo = ops.conv_halo_supported(c.ci, c.co, 3, c.in_hw[0], c.in_hw[1])
                    c.halo_w = ops.conv_halo_wgrad_supported(c.ci, c.co, 3, c.in_hw[0], c.in_hw[1])
            if not os.environ.get("HB200_NO_CONV_S2"):
                for convs, cd in self.blocks:   # stride-2 block entry: 3x3 s2 conv + 1x1 s2 downsample in one kernel
                    c = convs[0]
                    if (cd is not None and c.k == 3 and c.stride == 2 and c.pad == 1 and cd.k == 1 and cd.stride == 2
                            and cd.pad == 0 and c.conv_groups == 1 and cd.conv_groups == 1 and c.ci == c.ci_real
                            and ops.conv_s2_supported(c.ci, c.co, cd.co, c.in_hw[0], c.in_hw[1])):
                        c.s2_pair, cd.s2_main = cd, c
        self._ws = {}
        self._dev = None
        self._packed_key = None
        self.side = SideStream()

    # ---- buffers -----------------------------------------------------------------------------
    def _act_names(self):
        names = ["x0", "x1"]
        for j, (convs, cd) in enumerate(self.blocks):
            names += [f"a{j}_{i}" for i in range(len(convs) - 1)] + [f"o{j}"]
        return names

    def _ensure(self, B, dev, train):
        if self._dev != dev:
            for c in self.convs:
                c.alloc_weights(dev, need_dgrad=c is not self.stem)
            # every weight-gradient accumulator in ONE arena: one memset per backward pass instead of one per conv
            accs = [(c, nm) for c in self.convs for nm in ("dw_acc", "dw_s2") if getattr(c, nm, None) is not None]
            self._dw_arena = torch.empty(sum(getattr(c, nm).numel() for c, nm in accs), device=dev)
            off = 0
            for c, nm in accs:
                t = getattr(c, nm)
                setattr(c, nm, self._dw_arena[off: off + t.numel()].view_as(t))
                off += t.numel()
            self._dev, self._ws, self._packed_key = dev, {}, None
        key = (B, train)
        if key in self._ws:
            return self._ws[key]
        e = lambda *s: torch.empty(*s, dtype=F16, device=dev)  # noqa: E731  (forward values)
        ws = {"x0": e(B, self.hp // 2, self.wp_ // 2, 16) if self.stem.stem_s2d else e(B, self.hp, self.wp_, 8)}
        # GroupNorm statistics of all convs live in one f64 arena (f64: reproducible atomics) zeroed by ONE memset
        tot = sum(B * c.groups * 2 for c in self.convs)
        ws["st_all"] = torch.empty(tot, device=dev, dtype=torch.float64)
        off = 0
        for i, c in enumerate(self.convs):
            ws[f"y{i}"] = e(B, *c.out_hw, c.co)
            ws[f"st{i}"] = ws["st_all"][off: off + B * c.groups * 2].view(B, c.groups, 2)
            off += B * c.groups * 2
        ws["x1"] = e(B, *self.pool_hw, self.stem.co)
        ws["argmax"] = torch.empty(B, *self.pool_hw, self.stem.co, dtype=torch.uint8, device=dev)
        for j, (convs, cd) in enumerate(self.blocks):
            for i, c in enumerate(convs[:-1]):
                ws[f"a{j}_{i}"] = e(B, *c.out_hw, c.co)
            ws[f"o{j}"] = e(B, *convs[-1].out_hw, convs[-1].co)
            if self.se[j] is not None:   # squeeze p, hidden h, scale s (forward); a, dh (backward): f32 per frame
                C, cr = convs[-1].co, self.se[j][0].out_features
                for nm, n in (("p", C), ("h", cr), ("s", C)) + ((("a", C), ("dh", cr)) if train else ()):
                    ws[f"se{nm}{j}"] = torch.empty(B, n, device=dev)
        ncomp, fh, fw = self.enc.output_shape
        ws["feat"] = torch.empty(B, ncomp * fh * fw, device=dev)
        if train:
            # bf16 twins of every conv INPUT: the weight-gradient MMAs need x in the gradients' format (bf16 x bf16);
            # the forward convs keep reading the fp16 originals.  Written by the same elementwise kernels.
            for nm in self._act_names():
                ws[nm + "_b"] = torch.empty_like(ws[nm], dtype=BF16)
            big = max(max(int(np.prod(c.out_hw)) * c.co, int(np.prod(c.in_hw)) * c.ci) for c in self.convs)
            for nm in ("g0", "g1", "dy", "dy2", "gz"):
                ws[nm] = torch.empty(B * big, dtype=BF16, device=dev)
        self._ws[key] = ws
        return ws

    def pack_weights(self):
        for c in self.convs:
            w = c.dense_weight()
            if c.stem_s2d:
                ops.pack_halo_weight(w, c.wh, 16, c.co, 4, 2)
            elif c.halo:
                ops.pack_halo_weight(w, c.wh, c.ci, c.co, 3, 0)
                ops.pack_halo_weight(w, c.wht, c.co, c.ci, 3, 1)
            elif c.s2_pair is not None:
                c._wcat[: c.co].copy_(w)
                c._wcat[c.co:, :, 1, 1].copy_(c.s2_pair.dense_weight()[:, :, 0, 0])
                ntot = c._wcat.shape[0]
                ops.pack_halo_weight(c._wcat, c.wh, c.ci, ntot, 3, 0)
                ops.pack_halo_weight(c._wcat, c.wht, ntot, c.ci, 3, 1)
            elif c.s2_main is not None:
                pass   # lives in the centre tap of its partner's images
            else:
                ops.pack_conv_weight_into(w, c.wp, c.wt, c.ci)

    def _dgrad(self, c, dy, dx, B, addend=None):
        if c.halo:
            ops.conv_halo(dy, c.wht, dx, B, c.in_hw[0], c.in_hw[1], c.co, c.ci, 3, 1, addend=addend)
        else:
            ops.conv_dgrad(dy, c.wt, dx, c.shape(B), addend=addend)

    # ---- forward -----------------------------------------------------------------------------
    def forward(self, x0_writer, B, dev, train, wkey=None, out=None):
        """x0_writer(x0, x0_bf16) fills the pooled / normalised input.  Returns feat f32 [B, C*h*w] in the
        reference's (c,h,w) flatten order, written into `out` (contiguous f32, B * C*h*w elements) when given.  `wkey`
        identifies the weight values: inference calls (act / get_value during a rollout) with an unchanged key reuse
        the packed weight images instead of re-packing every tensor per step; training forwards always re-pack."""
        ws = self._ensure(B, dev, train)
        packed = None
        if train:
            # ~40 tiny packing launches (launch-bound, 0.17 ms) ride on the side stream under the input prep, which
            # does not read the weights
            with self.side.after_main():
                self.pack_weights()
                packed = self.side.mark()
            self._packed_key = wkey
        elif wkey is None or wkey != self._packed_key:
            self.pack_weights()
            self._packed_key = wkey
        x0_writer(ws["x0"], ws.get("x0_b"))
        self.side.wait(packed)
        idx = {id(c): i for i, c in enumerate(self.convs)}
        ws["st_all"].zero_()

        def conv(c, x):
            i = idx[id(c)]
            if c.s2_main is not None:      # computed by its partner's launch
                return ws[f"y{i}"], ws[f"st{i}"]
            if c.s2_pair is not None:
                d, k = c.s2_pair, idx[id(c.s2_pair)]
                ops.conv_s2_fwd(x, c.wh, ws[f"y{i}"], ws[f"y{k}"], B, c.in_hw[0], c.in_hw[1], c.ci, c.co, d.co,
                                stats_a=ws[f"st{i}"], groups_a=c.groups, stats_b=ws[f"st{k}"], groups_b=d.groups)
                return ws[f"y{i}"], ws[f"st{i}"]
            if c.stem_s2d:
                ops.conv_halo(x, c.wh, ws[f"y{i}"], B, c.out_hw[0], c.out_hw[1], 16, c.co, 4, 0, gn_stats=ws[f"st{i}"],
                              gn_groups=c.groups)
            elif c.halo:
                ops.conv_halo(x, c.wh, ws[f"y{i}"], B, c.in_hw[0], c.in_hw[1], c.ci, c.co, 3, 0, gn_stats=ws[f"st{i}"],
                              gn_groups=c.groups)
            else:
                ops.conv_fwd(x, c.wp, ws[f"y{i}"], c.shape(B), ws[f"st{i}"], c.groups)
            return ws[f"y{i}"], ws[f"st{i}"]

        y, st = conv(self.stem, ws["x0"])
        sh, sw = self.stem.out_hw
        ops.gn_relu_maxpool(y, st, self.stem.gamma, self.stem.beta, ws["x1"], ws["argmax"], B, sh, sw,
                            self.stem.co, self.stem.groups, out_bf16=ws.get("x1_b"))
        x = ws["x1"]
        for j, (convs, cd) in enumerate(self.blocks):
            cur = x
            for i, c in enumerate(convs):
                yc, sc = conv(c, cur)
                hw = c.out_hw[0] * c.out_hw[1]
                if i < len(convs) - 1:     # conv -> GroupNorm -> ReLU
                    ops.gn_apply(yc, sc, c.gamma, c.beta, ws[f"a{j}_{i}"], B, hw, c.co, c.groups, relu=True,
                                 out_bf16=ws.get(f"a{j}_{i}_b"))
                    cur = ws[f"a{j}_{i}"]
                elif self.se[j] is not None:   # last conv: relu(SE(GN(y)) + r), r = x or GN_d(conv_d(x))
                    ex = self.se[j]
                    rkw = {}
                    if cd is not None:
                        yd, sd = conv(cd, x)
                        rkw = dict(res_stats=sd, res_gamma=cd.gamma, res_beta=cd.beta)
                    ops.gn_se_residual_relu(yc, sc, c.gamma, c.beta, yd if cd is not None else x, ex[0].weight,
                                            ex[0].bias, ex[2].weight, ex[2].bias, ws[f"sep{j}"], ws[f"seh{j}"],
                                            ws[f"ses{j}"], ws[f"o{j}"], B, hw, c.co, c.groups,
                                            out_bf16=ws.get(f"o{j}_b"), **rkw)
                elif cd is not None:       # last conv: relu(GN(y) + GN_d(conv_d(x)))
                    yd, sd = conv(cd, x)
                    ops.gn_residual_relu(yc, sc, c.gamma, c.beta, yd, ws[f"o{j}"], B, hw, c.co, c.groups, sd,
                                         cd.gamma, cd.beta, out_bf16=ws.get(f"o{j}_b"))
                else:                      # last conv: relu(GN(y) + x)
                    ops.gn_residual_relu(yc, sc, c.gamma, c.beta, x, ws[f"o{j}"], B, hw, c.co, c.groups,
                                         out_bf16=ws.get(f"o{j}_b"))
            x = ws[f"o{j}"]
        yc, sc = conv(self.comp, x)
        fhw = self.comp.out_hw[0] * self.comp.out_hw[1]
        feat = ws["feat"] if out is None else out
        ops.gn_apply(yc, sc, self.comp.gamma, self.comp.beta, feat, B, fhw, self.comp.co, self.comp.groups,
                     relu=True, chw_flat=True)
        return feat

    # ---- backward ----------------------------------------------------------------------------
    def backward(self, d_feat, B, dev):
        """d_feat f32 [B, C*h*w] (c,h,w order): gradient wrt the compression output (after ReLU).
        Writes every conv / GroupNorm parameter gradient into the parameters' .grad views."""
        ws = self._ws[(B, True)]
        idx = {id(c): i for i, c in enumerate(self.convs)}
        Y = lambda c: ws[f"y{idx[id(c)]}"]  # noqa: E731
        ST = lambda c: ws[f"st{idx[id(c)]}"]  # noqa: E731

        def view(buf, c_or_shape):
            shp = (B, *c_or_shape.out_hw, c_or_shape.co) if isinstance(c_or_shape, _Conv) else c_or_shape
            n = int(np.prod(shp))
            return buf[:n].view(*shp)

        # dy buffers alternate so that the weight-gradient kernel of layer k (side stream) can still read its dy
        # while GroupNorm backward of layer k-1 writes the other one; dy_busy[i] = side-stream event of the last reader
        side = self.side
        dy_bufs, dy_busy, dy_turn = [ws["dy"], ws["dy2"]], [None, None], [0]

        def gn_bwd(c, g, act, mode, want_gz):
            hw = c.out_hw[0] * c.out_hw[1]
            slot = dy_turn[0]
            dy_turn[0] ^= 1
            side.wait(dy_busy[slot])
            dy = view(dy_bufs[slot], c)
            gz = view(ws["gz"], c) if want_gz else None
            ops.gn_bwd(g, act, Y(c), ST(c), c.gamma, c.beta, c.gamma.grad, c.beta.grad, dy, gz, B, hw, c.co, c.groups, mode)
            return dy, gz

        def se_bwd(j, c, g):
            """gn_bwd(mode 2, want_gz) of an SE block's last conv, then its excitation weight gradients (side stream)"""
            hw = c.out_hw[0] * c.out_hw[1]
            slot = dy_turn[0]
            dy_turn[0] ^= 1
            side.wait(dy_busy[slot])
            dy, gz = view(dy_bufs[slot], c), view(ws["gz"], c)
            ex = self.se[j]
            ops.gn_se_bwd(g, ws[f"o{j}"], Y(c), ST(c), c.gamma, c.beta, ws[f"ses{j}"], ws[f"seh{j}"], ex[0].weight,
                          ex[2].weight, c.gamma.grad, c.beta.grad, dy, gz, ws[f"sea{j}"], ws[f"sedh{j}"], B, hw, c.co,
                          c.groups)
            with side.after_main():
                ops.se_excite_wgrad(ws[f"sea{j}"], ws[f"seh{j}"], ws[f"sep{j}"], ws[f"sedh{j}"], ex[0].weight.grad,
                                    ex[0].bias.grad, ex[2].weight.grad, ex[2].bias.grad)
            return dy, gz

        def wgrad(c, x, dy):
            with side.after_main():
                if c.stem_s2d:
                    ops.conv_halo_wgrad(x, dy, c.dw_acc, B, c.out_hw[0], c.out_hw[1], 16, c.co, 4)
                    ops.unpack_stem_wgrad(c.dw_acc, c.w.grad)
                elif c.s2_pair is not None and c.dw_s2 is not None:   # 3x3 stride-2 conv over the space-to-depth view
                    ops.conv_s2_wgrad(x, dy, c.dw_s2, B, c.in_hw[0], c.in_hw[1], c.ci, c.co)
                    ops.unpack_s2_wgrad(c.dw_s2, c.grad_target())
                else:
                    if c.halo or c.halo_w:
                        ops.conv_halo_wgrad(x, dy, c.dw_acc, B, c.in_hw[0], c.in_hw[1], c.ci, c.co, 3)
                    else:
                        ops.conv_wgrad(x, dy, c.dw_acc, c.shape(B))
                    ops.unpack_conv_wgrad(c.dw_acc, c.grad_target(), c.ci)
                    c.store_grad()
                ev = side.mark()
            for i in (0, 1):
                if dy.data_ptr() == dy_bufs[i].data_ptr():
                    dy_busy[i] = ev

        with side.after_main():
            self._dw_arena.zero_()   # all weight-gradient accumulators (split-K / per-tile red.add targets)
        g_bufs = [ws["g0"], ws["g1"]]
        cur = 0
        like = lambda buf, t: buf[: t.numel()].view_as(t)  # noqa: E731
        # compression: relu(GN(yc)) -> visual_fc
        comp = self.comp
        fhw = comp.out_hw[0] * comp.out_hw[1]
        g = view(g_bufs[cur], comp)
        ops.f32_chw_to_bf16_hwc(d_feat, g, B, fhw, comp.co)
        dy, _ = gn_bwd(comp, g, None, 1, False)
        last = len(self.blocks) - 1
        wgrad(comp, ws[f"o{last}_b"], dy)
        cur ^= 1
        g = like(g_bufs[cur], ws[f"o{last}"])
        self._dgrad(comp, dy, g, B)
        # residual blocks, last to first
        for j in reversed(range(len(self.blocks))):
            convs, cd = self.blocks[j]
            xin = ws[f"o{j - 1}"] if j > 0 else ws["x1"]
            xin_b = ws[f"o{j - 1}_b"] if j > 0 else ws["x1_b"]    # bf16 twin: the weight gradients' x operand
            n = len(convs)
            if self.se[j] is not None:
                dyl, gz = se_bwd(j, convs[-1], g)
            else:
                dyl, gz = gn_bwd(convs[-1], g, ws[f"o{j}"], 2, True)  # g: grad wrt the block output; gz = g * [o > 0]
            wgrad(convs[-1], ws[f"a{j}_{n - 2}_b"], dyl)
            cur ^= 1
            ga = like(g_bufs[cur], ws[f"a{j}_{n - 2}"])
            self._dgrad(convs[-1], dyl, ga, B)                    # grad wrt a = relu(GN(y)) of the previous conv
            for i in range(n - 2, 0, -1):
                dyi, _ = gn_bwd(convs[i], ga, None, 1, False)
                wgrad(convs[i], ws[f"a{j}_{i - 1}_b"], dyi)
                cur ^= 1
                ga = like(g_bufs[cur], ws[f"a{j}_{i - 1}"])
                self._dgrad(convs[i], dyi, ga, B)
            dy0, _ = gn_bwd(convs[0], ga, None, 1, False)
            wgrad(convs[0], xin_b, dy0)
            gx = like(g_bufs[cur], xin)                           # ga is consumed; reuse its buffer
            if cd is not None and convs[0].s2_pair is cd:
                c0 = convs[0]
                dyd, _ = gn_bwd(cd, gz, None, 0, False)
                wgrad(cd, xin_b, dyd)
                ops.conv_s2_dgrad(dy0, dyd, c0.wht, gx, B, c0.in_hw[0], c0.in_hw[1], c0.ci, c0.co, cd.co)
            elif cd is not None:
                self._dgrad(convs[0], dy0, gx, B)
                dyd, _ = gn_bwd(cd, gz, None, 0, False)           # ws["gz"] is only rewritten by the next block
                wgrad(cd, xin_b, dyd)
                self._dgrad(cd, dyd, gx, B, addend=gx)
            else:
                self._dgrad(convs[0], dy0, gx, B, addend=gz)
            g = gx
        # stem: maxpool -> relu(GN(y0)) -> conv1 (input needs no gradient)
        stem = self.stem
        sh, sw = stem.out_hw
        cur ^= 1
        if sh % 2 == 0 and sw % 2 == 0 and ops.gn_relu_maxpool_bwd_supported(sh, sw, stem.co, stem.groups):
            # pooled gradient -> dy of the stem conv in one pass (the 64x64 pooled gradient is never materialised)
            dy0 = like(g_bufs[cur], Y(stem))
            ops.gn_relu_maxpool_bwd(g, ws["argmax"], Y(stem), ST(stem), stem.gamma, stem.beta, stem.gamma.grad,
                                    stem.beta.grad, dy0, B, sh, sw, stem.co, stem.groups)
        else:
            gzs = like(g_bufs[cur], Y(stem))
            ops.maxpool_bwd(g, ws["argmax"], gzs, B, sh, sw, stem.co)
            dy0, _ = gn_bwd(stem, gzs, None, 1, False)
        wgrad(stem, ws["x0_b"], dy0)
        side.join()


# ---------------------------------------------------------------------------------------------
# generic policy machinery: flat parameters, recurrent encoder, heads, loss + backward
# ---------------------------------------------------------------------------------------------
class NativeNetPolicy(nn.Module):
    """NetPolicy (rl/ppo/policy.py:252-413) whose forward AND backward are libhb200 kernels.
    Subclasses provide the perception part through two hooks:
      _visual_forward(obs, rows, prev_actions, masks_u8, B, dev, train) -> (rnn_in f32 [B, D], saved)
      _visual_backward(d_rnn_in f32 [B, D], saved, B, dev)   (writes parameter gradients in place)
    """

    def __init__(self, net: nn.Module, action_space):
        super().__init__()
        self.action_distribution_type = "categorical"
        self._action_space = action_space
        self.net = net
        self.dim_actions = action_space.n
        self.action_distribution = CategoricalNet(self.net.output_size, self.dim_actions)
        self.critic = CriticHead(self.net.output_size)
        self.aux_loss_modules = nn.ModuleDict()
        self._flat = None
        self._buf = {}
        self._wver = 0   # bumped whenever parameter VALUES change through a path torch's tensor version cannot see
        self._side = SideStream()
        self.world_size = 1  # set by the distributed updater
        self.dist_group = None
        self.tail_grads_hook = None   # DDPPO: called (on the side stream) once the recurrent + head gradients are final

    # ---- reference API surface ----------------------------------------------------------------
    @property
    def should_load_agent_state(self):
        return True

    @property
    def num_recurrent_layers(self) -> int:
        return self.net.num_recurrent_layers

    @property
    def recurrent_hidden_size(self) -> int:
        return self.net.recurrent_hidden_size

    @property
    def hidden_state_shape(self):
        return (self.num_recurrent_layers, self.recurrent_hidden_size)

    @property
    def visual_encoder(self):
        return self.net.visual_encoder

    @property
    def policy_action_space(self):
        return self._action_space

    def _get_policy_components(self):
        return [self.net, self.critic, self.action_distribution]

    def policy_parameters(self):
        for c in self._get_policy_components():
            yield from c.parameters()

    def all_policy_tensors(self):
        yield from self.policy_parameters()
        for c in self._get_policy_components():
            yield from c.buffers()

    def aux_loss_parameters(self):
        return {}

    # ---- flat parameter / gradient storage ---------------------------------------------------------
    def flatten_parameters_(self):
        """Re-home every parameter in one flat fp32 buffer (and .grad in a second one) so the
        gradient all-reduce, the norm and Adam are single kernels.  Idempotent; re-run
        automatically after .to()/load_state_dict replaced the storage.

        Parameters with requires_grad=False (a frozen visual encoder, train_encoder=False) are placed after all the
        trainable ones and get no gradient: [0, n) of the parameter buffer and the whole gradient buffer hold exactly the
        trainable parameters, so the all-reduce, the norm and Adam never touch the frozen ones.  With every parameter
        trainable the layout is registration order, as before."""
        params = list(self.parameters())
        dev = params[0].device
        if dev.type != "cuda":
            raise Hb200Error("hb200 policy must live on a CUDA device (no CPU fallback)")
        train = [p for p in params if p.requires_grad]
        order = train + [p for p in params if not p.requires_grad]
        f = self._flat
        if f is not None and f["params"].device == dev and len(f["plist"]) == len(train) and all(
                p is q for p, q in zip(order, f["all"])) and all(
                p.data_ptr() == f["params"].data_ptr() + 4 * o and
                (p.grad is not None and p.grad.data_ptr() == f["grads"].data_ptr() + 4 * o if p.requires_grad
                 else p.grad is None) for p, o in zip(order, f["all_offsets"])):
            return f
        # every tensor starts on a 16-byte boundary (TF32 / vector kernels read rows as float4)
        offs, o, n = [], 0, 0
        for i, p in enumerate(order):
            offs.append(o)
            o += (p.numel() + 3) // 4 * 4
            if i + 1 == len(train):
                n = o
        flat_p = torch.zeros(o, device=dev)
        flat_g = torch.zeros(n, device=dev)
        for i, (p, off) in enumerate(zip(order, offs)):
            k = p.numel()
            flat_p[off:off + k].copy_(p.data.reshape(-1))
            p.data = flat_p[off:off + k].view(p.shape)
            p.grad = flat_g[off:off + k].view(p.shape) if i < len(train) else None
        self._flat = dict(params=flat_p, grads=flat_g, offsets=offs[: len(train)], n=n,
                          n_real=sum(p.numel() for p in train), plist=train, all=order, all_offsets=offs)
        self.mark_weights_changed()
        return self._flat

    def tail_offset(self) -> int:
        """First element of the flat buffers that belongs to the recurrent encoder / heads.  Their gradients are final
        as soon as the RNN backward is done, long before the conv stack's: the distributed updater reduces
        [tail_offset, n) while the encoder backward still runs (rl/ppo.py DDPPO)."""
        f = self.flatten_parameters_()
        names = {id(p): name for name, p in self.named_parameters()}
        for p, off in zip(f["plist"], f["offsets"]):
            if names[id(p)].startswith("net.state_encoder."):
                return off
        return f["n"]

    def mark_weights_changed(self) -> None:
        """Called by FusedAdam.step / load_state_dict / the DD-PPO broadcast: invalidates cached weight images."""
        self._wver += 1

    def weights_key(self):
        """(explicit counter, storage, torch version counters): in-place torch ops on a parameter (nn.init, copy_,
        optimizers) bump p._version; writes through p.data or raw pointers must call mark_weights_changed()."""
        f = self._flat
        if f is None:
            return None
        return (self._wver, f["params"].data_ptr(), f["params"]._version, sum(p._version for p in f["all"]))

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self.mark_weights_changed()
        return out

    def _tmp(self, name, shape, dev, dtype=torch.float32):
        key = (name, tuple(shape), dtype)
        t = self._buf.get(key)
        if t is None or t.device != dev:
            t = torch.empty(*shape, device=dev, dtype=dtype)
            self._buf[key] = t
        return t

    def _loss_ws(self, B, dev):
        key = ("loss_ws", B)
        if key not in self._buf or self._buf[key].device != dev:
            self._buf[key] = ops.ppo_loss_workspace(B, self.net.output_size, self.dim_actions, dev)
        return self._buf[key]

    # ---- recurrent state encoder -----------------------------------------------------------------------
    # ---- two stacked LSTM layers as a wavefront ----------------------------------------------------------------
    # A layer is T dependent steps of ~6 us (grid barrier + a 32 x 512 x 2048 mat-vec): latency, not throughput, and
    # the second layer only needs step t of the first.  The sequence is cut into time chunks; layer l runs chunk c on
    # its own stream as soon as layer l-1 has finished chunk c (forward; backward: top layer first, chunks last to
    # first), so the two persistent kernels are co-resident (128 CTAs each, two fit per SM) and the critical path is
    # (chunks + 1) / (2 * chunks) of the sequential one.  Arithmetic and its order are unchanged: bit-identical results.
    _RNN_CHUNKS = int(os.environ.get("HB200_RNN_CHUNKS", "4"))

    def _rnn_wavefront(self, lstm, H, L, T):
        return (lstm and H == 512 and L >= 2 and T >= 8 * self._RNN_CHUNKS and T % self._RNN_CHUNKS == 0
                and not os.environ.get("HB200_NO_RNN_WAVEFRONT"))

    def _rnn_streams(self, L):
        st = getattr(self, "_rnn_side_streams", None)
        if st is None or len(st) < L - 1:
            st = self._rnn_side_streams = [torch.cuda.Stream() for _ in range(L - 1)]
        return st

    def _rnn_forward(self, rnn_in, hid, mk, T, n, B, dev, train):
        rnn = self.net.state_encoder.rnn
        H, L = rnn.hidden_size, rnn.num_layers
        lstm = isinstance(rnn, nn.LSTM)
        if self._rnn_wavefront(lstm, H, L, T):
            return self._rnn_forward_wavefront(rnn_in, hid, mk, T, n, B, dev, train)
        ws = self._tmp("rnn_ws", (64,), dev, torch.uint8)
        layers, x = [], rnn_in
        for l in range(L):
            w_ih, w_hh = getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}")
            b_ih, b_hh = getattr(rnn, f"bias_ih_l{l}"), getattr(rnn, f"bias_hh_l{l}")
            G = 4 if lstm else 3
            xproj = self._tmp(f"xproj{l}", (B, G * H), dev)
            ops.linear_fwd(x, w_ih, b_ih, xproj, tf32=True)
            hs = self._tmp(f"hs{l}", (T, n, H), dev)
            if lstm:
                cs = self._tmp(f"cs{l}", (T, n, H), dev)
                gates = self._tmp(f"gates{l}", (T, n, 4 * H), dev) if train else None
                h0, c0 = hid[:, l], hid[:, L + l]
                ops.lstm_seq_fwd(xproj, w_hh, b_hh, mk, h0, c0, hs, cs, gates, T, n, H, ws)
                layers.append(dict(x=x, hs=hs, cs=cs, gates=gates, h0=h0, c0=c0))
            else:
                saved = self._tmp(f"gates{l}", (T, n, 4 * H), dev) if train else None
                h0 = hid[:, l]
                ops.gru_seq_fwd(xproj, w_hh, b_hh, mk, h0, hs, saved, T, n, H, ws)
                layers.append(dict(x=x, hs=hs, gates=saved, h0=h0))
            x = hs.view(B, H)
        parts = [ly["hs"][T - 1] for ly in layers] + ([ly["cs"][T - 1] for ly in layers] if lstm else [])
        return x, layers, torch.stack(parts, dim=1)

    def _rnn_forward_wavefront(self, rnn_in, hid, mk, T, n, B, dev, train):
        rnn = self.net.state_encoder.rnn
        H, L = rnn.hidden_size, rnn.num_layers
        C = self._RNN_CHUNKS
        Tc = T // C
        main = torch.cuda.current_stream()
        streams = [main] + self._rnn_streams(L)
        layers = []
        # every buffer is allocated (and the first layer's input projection runs for all frames) before the fork
        for l in range(L):
            layers.append(dict(
                x=rnn_in if l == 0 else layers[l - 1]["hs"].view(B, H),
                xproj=self._tmp(f"xproj{l}", (B, 4 * H), dev), hs=self._tmp(f"hs{l}", (T, n, H), dev),
                cs=self._tmp(f"cs{l}", (T, n, H), dev),
                gates=self._tmp(f"gates{l}", (T, n, 4 * H), dev) if train else None,
                h0=hid[:, l], c0=hid[:, L + l], ws=self._tmp(f"rnn_ws{l}", (64,), dev, torch.uint8)))
        ops.linear_fwd(rnn_in, rnn.weight_ih_l0, rnn.bias_ih_l0, layers[0]["xproj"], tf32=True)
        for s_ in streams[1:]:
            s_.wait_stream(main)
        done = [[None] * C for _ in range(L)]
        for c in range(C):
            t0, t1 = c * Tc, (c + 1) * Tc
            r0, r1 = t0 * n, t1 * n
            for l in range(L):
                ly = layers[l]
                w_ih, w_hh = getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}")
                b_ih, b_hh = getattr(rnn, f"bias_ih_l{l}"), getattr(rnn, f"bias_hh_l{l}")
                with torch.cuda.stream(streams[l]):
                    if l > 0:
                        streams[l].wait_event(done[l - 1][c])
                        ops.linear_fwd(ly["x"][r0:r1], w_ih, b_ih, ly["xproj"][r0:r1], tf32=True)
                    h0 = ly["h0"] if c == 0 else ly["hs"][t0 - 1]
                    c0 = ly["c0"] if c == 0 else ly["cs"][t0 - 1]
                    ops.lstm_seq_fwd(ly["xproj"][r0:r1], w_hh, b_hh, mk[r0:r1], h0, c0, ly["hs"][t0:t1], ly["cs"][t0:t1],
                                     ly["gates"][t0:t1] if train else None, Tc, n, H, ly["ws"])
                    if l + 1 < L:
                        done[l][c] = torch.cuda.Event()
                        done[l][c].record(streams[l])
        for s_ in streams[1:]:
            main.wait_stream(s_)
        out = [dict(x=ly["x"], hs=ly["hs"], cs=ly["cs"], gates=ly["gates"], h0=ly["h0"], c0=ly["c0"]) for ly in layers]
        parts = [ly["hs"][T - 1] for ly in out] + [ly["cs"][T - 1] for ly in out]
        return out[-1]["hs"].view(B, H), out, torch.stack(parts, dim=1)

    def _rnn_backward(self, d_out, layers, mk, T, n, B, dev):
        rnn = self.net.state_encoder.rnn
        H, L = rnn.hidden_size, rnn.num_layers
        lstm = isinstance(rnn, nn.LSTM)
        if self._rnn_wavefront(lstm, H, L, T):
            return self._rnn_backward_wavefront(d_out, layers, mk, T, n, B, dev)
        ws = self._tmp("rnn_ws", (64,), dev, torch.uint8)
        for l in reversed(range(L)):
            ly = layers[l]
            w_ih, w_hh = getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}")
            G = 4 if lstm else 3
            dgx = self._tmp(f"dgates{l}", (T, n, G * H), dev)
            if lstm:
                ops.lstm_seq_bwd(d_out.view(T, n, H), ly["gates"], ly["cs"], ly["c0"], w_hh, mk, dgx, T, n, H, ws)
                dgh = dgx
            else:
                dgh = self._tmp(f"dgh{l}", (T, n, G * H), dev)
                ops.gru_seq_bwd(d_out.view(T, n, H), ly["gates"], ly["hs"], ly["h0"], w_hh, mk, dgx, dgh, T, n, H, ws)
            self._rnn_weight_grads(l, ly, dgx, dgh, mk, T, n, B, dev, lstm)
            x = ly["x"]
            dx = self._tmp(f"dx{l}", (B, x.stride(0)), dev)[:, : x.shape[1]]   # same (16-byte) row pitch as x
            ops.linear_bwd_input(dgx.view(B, G * H), w_ih, dx, tf32=True)
            d_out = dx
        return d_out

    def _rnn_weight_grads(self, l, ly, dgx, dgh, mk, T, n, B, dev, lstm):
        rnn = self.net.state_encoder.rnn
        H = rnn.hidden_size
        G = 4 if lstm else 3
        w_ih, w_hh = getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}")
        b_ih, b_hh = getattr(rnn, f"bias_ih_l{l}"), getattr(rnn, f"bias_hh_l{l}")
        dgxf, dghf = dgx.view(B, G * H), dgh.view(B, G * H)
        x = ly["x"]
        with self._side.after_main():   # weight gradients: off the critical path (SideStream)
            ops.linear_bwd_weight(dgxf, x, w_ih.grad, accumulate=True, tf32=True)  # grads pre-zeroed: split-K
            hin = self._tmp(f"hin{l}", (T, n, H), dev)
            ops.rnn_shift_mask(ly["hs"], ly["h0"], mk, hin, T, n, H)
            ops.linear_bwd_weight(dghf, hin.view(B, H), w_hh.grad, accumulate=True, tf32=True)
            ops.colsum(dgxf, b_ih.grad)
            if lstm:
                b_hh.grad.copy_(b_ih.grad)
            else:
                ops.colsum(dghf, b_hh.grad)

    def _rnn_backward_wavefront(self, d_out, layers, mk, T, n, B, dev):
        """Mirror of _rnn_forward_wavefront: the top layer walks the time chunks last to first on the main stream and
        hands each chunk's input gradient (one TF32 GEMM per chunk) to the layer below, which follows one chunk behind on
        its own stream.  Weight gradients need all T steps of a layer: side stream, after that layer's last chunk."""
        rnn = self.net.state_encoder.rnn
        H, L = rnn.hidden_size, rnn.num_layers
        C = self._RNN_CHUNKS
        Tc = T // C
        main = torch.cuda.current_stream()
        order = list(reversed(range(L)))                 # top layer first
        streams = {l: s_ for l, s_ in zip(order, [main] + self._rnn_streams(L))}
        dgx = {l: self._tmp(f"dgates{l}", (T, n, 4 * H), dev) for l in range(L)}
        carry = {l: self._tmp(f"rnn_carry{l}", (2, n, H), dev) for l in range(L)}
        wsb = {l: self._tmp(f"rnn_ws{l}", (64,), dev, torch.uint8) for l in range(L)}
        dxs = {}
        for l in range(L):
            x = layers[l]["x"]
            dxs[l] = self._tmp(f"dx{l}", (B, x.stride(0)), dev)[:, : x.shape[1]]
        for l in order[1:]:
            streams[l].wait_stream(main)
        d_in = {order[0]: d_out}
        for l in order[1:]:
            d_in[l] = dxs[l + 1]
        done = {l: [None] * C for l in range(L)}
        for c in reversed(range(C)):
            t0, t1 = c * Tc, (c + 1) * Tc
            r0, r1 = t0 * n, t1 * n
            for l in order:
                ly = layers[l]
                w_ih, w_hh = getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}")
                with torch.cuda.stream(streams[l]):
                    if l != order[0]:
                        streams[l].wait_event(done[l + 1][c])
                    c0 = ly["c0"] if c == 0 else ly["cs"][t0 - 1]
                    ops.lstm_seq_bwd_chunk(d_in[l][r0:r1].view(Tc, n, H), ly["gates"][t0:t1], ly["cs"][t0:t1], c0, w_hh,
                                           mk[r0:r1], dgx[l][t0:t1], Tc, n, H, wsb[l], carry[l], carry_in=c < C - 1,
                                           carry_out=c > 0)
                    if l > 0:   # the layer below consumes this chunk's input gradient
                        ops.linear_bwd_input(dgx[l][t0:t1].view(Tc * n, 4 * H), w_ih, dxs[l][r0:r1], tf32=True)
                        done[l][c] = torch.cuda.Event()
                        done[l][c].record(streams[l])
        for l in order[1:]:
            main.wait_stream(streams[l])
        for l in order:
            self._rnn_weight_grads(l, layers[l], dgx[l], dgx[l], mk, T, n, B, dev, True)
        ops.linear_bwd_input(dgx[0].view(B, 4 * H), rnn.weight_ih_l0, dxs[0], tf32=True)
        return dxs[0]

    # ---- shared forward ----------------------------------------------------------------------------------
    def _trunk(self, observations, rnn_hidden_states, prev_actions, masks, train: bool):
        obs, rows = _as_rows(observations, rnn_hidden_states.device)
        dev = rnn_hidden_states.device
        if dev.type != "cuda":
            raise Hb200Error("hb200 policy: inputs must be CUDA tensors (no CPU fallback)")
        self.flatten_parameters_()
        B = rows.numel()
        n = rnn_hidden_states.shape[0]
        T = B // n
        assert T * n == B, "frames must be (t, env)-ordered with T*n rows"
        pa = prev_actions.reshape(-1)
        mk = ops.as_u8(masks.reshape(-1))
        rnn_in, vsaved = self._visual_forward(obs, rows, pa, mk, B, dev, train)
        hid = rnn_hidden_states.contiguous()
        feats, layers, hidden_out = self._rnn_forward(rnn_in, hid, mk, T, n, B, dev, train)
        return dict(B=B, n=n, T=T, rows=rows, obs=obs, masks=mk, pa=pa, layers=layers, features=feats,
                    hidden_out=hidden_out, visual=vsaved)

    def _heads(self, feats, B, dev):
        logits = self._tmp("logits", (B, self.dim_actions), dev)
        values = self._tmp("values_act", (B,), dev)
        ad, cr = self.action_distribution.linear, self.critic.fc
        ops.heads_fwd(feats, ad.weight, ad.bias, cr.weight, cr.bias, logits, values)
        return logits, values

    @torch.no_grad()
    def act(self, observations, rnn_hidden_states, prev_actions, masks, deterministic=False):
        """Policy.act (rl/ppo/policy.py:300-359).  The heads, the log-softmax, the draw (inverse CDF at one torch.rand number
        per frame -- same distribution as Categorical.sample, not the same random stream) or the mode, and
        log_probs(action) are ONE kernel (ops.heads_act)."""
        s = self._trunk(observations, rnn_hidden_states, prev_actions, masks, train=False)
        B = s["B"]
        feats = s["features"]
        dev = feats.device
        logp = self._tmp("logits", (B, self.dim_actions), dev)
        action = torch.empty(B, 1, dtype=torch.int64, device=dev)
        alp = torch.empty(B, 1, dtype=torch.float32, device=dev)
        vout = torch.empty(B, 1, dtype=torch.float32, device=dev)
        u = None if deterministic else torch.rand(B, device=dev, dtype=torch.float32)
        ad, cr = self.action_distribution.linear, self.critic.fc
        ops.heads_act(feats, ad.weight, ad.bias, cr.weight, cr.bias, u, logp, vout, action, alp)
        return PolicyActionData(values=vout, actions=action, action_log_probs=alp, rnn_hidden_states=s["hidden_out"])

    @torch.no_grad()
    def get_value(self, observations, rnn_hidden_states, prev_actions, masks):
        s = self._trunk(observations, rnn_hidden_states, prev_actions, masks, train=False)
        _, values = self._heads(s["features"], s["B"], s["features"].device)
        return values.view(s["B"], 1).clone()

    def evaluate_actions(self, observations, rnn_hidden_states, prev_actions, masks, action,
                         rnn_build_seq_info=None):
        """Forward only (values, log-probs, entropy, hidden, aux) like the reference
        (rl/ppo/policy.py:361-402); `rnn_build_seq_info` is accepted and ignored: the masked
        recurrence needs only `masks`."""
        s = self._trunk(observations, rnn_hidden_states, prev_actions, masks, train=True)
        feats, B = s["features"], s["B"]
        dev = feats.device
        out = dict(values=self._tmp("ea_values", (B,), dev), log_probs=self._tmp("ea_lp", (B,), dev),
                   entropy=self._tmp("ea_ent", (B,), dev), metrics=self._tmp("ea_metrics", (ops.N_METRICS,), dev))
        ad, cr = self.action_distribution.linear, self.critic.fc
        zero = self._tmp("zeros_B", (B,), dev)
        zero.zero_()
        ops.ppo_loss(feats, ad.weight, ad.bias, cr.weight, cr.bias, action.reshape(-1), zero, zero, zero, zero, 0.2,
                     0.5, 0.0, False, False, out, self._loss_ws(B, dev))
        return (out["values"].view(B, 1), out["log_probs"].view(B, 1), out["entropy"].view(B, 1),
                s["hidden_out"], {})

    def loss_and_backward(self, batch, clip_param, value_loss_coef, entropy_coef, use_clipped_value_loss,
                          observations=None):
        """Fused replacement of evaluate_actions + the loss section of PPO._update_from_batch +
        total_loss.backward() (rl/ppo/ppo.py:180-254).  Leaves every parameter's gradient in the flat
        gradient buffer (p.grad views) and returns the 12 metrics as a device tensor."""
        obs = observations if observations is not None else batch["observations"]
        s = self._trunk(obs, batch["recurrent_hidden_states"], batch["prev_actions"], batch["masks"], train=True)
        feats, B, n, T = s["features"], s["B"], s["n"], s["T"]
        dev = feats.device
        H = self.net.output_size
        self._flat["grads"].zero_()
        ad, cr = self.action_distribution.linear, self.critic.fc
        out = dict(values=self._tmp("ea_values", (B,), dev), log_probs=self._tmp("ea_lp", (B,), dev),
                   entropy=self._tmp("ea_ent", (B,), dev), metrics=self._tmp("ea_metrics", (ops.N_METRICS,), dev),
                   d_features=self._tmp("d_features", (B, H), dev), d_w_act=ad.weight.grad, d_b_act=ad.bias.grad,
                   d_w_val=cr.weight.grad, d_b_val=cr.bias.grad)
        f32 = lambda t: t.reshape(-1).contiguous()  # noqa: E731
        ops.ppo_loss(feats, ad.weight, ad.bias, cr.weight, cr.bias, f32(batch["actions"]),
                     f32(batch["action_log_probs"]), f32(batch["advantages"]), f32(batch["value_preds"]),
                     f32(batch["returns"]), clip_param, value_loss_coef, entropy_coef, use_clipped_value_loss, True,
                     out, self._loss_ws(B, dev), is_coeffs=f32(batch["is_coeffs"]) if "is_coeffs" in batch else None)
        d_rnn_in = self._rnn_backward(out["d_features"], s["layers"], s["masks"], T, n, B, dev)
        if self.tail_grads_hook is not None:
            with self._side.after_main():   # after the head gradients (main) and the RNN weight gradients (side)
                self.tail_grads_hook()
        self._visual_backward(d_rnn_in, s, B, dev)
        self._side.join()
        self._last = dict(values=out["values"], log_probs=out["log_probs"], entropy=out["entropy"],
                          hidden_out=s["hidden_out"])
        return out["metrics"]


# ---------------------------------------------------------------------------------------------
# PointNavResNetPolicy
# ---------------------------------------------------------------------------------------------
@baseline_registry.register_policy
class PointNavResNetPolicy(NativeNetPolicy):
    def __init__(self, observation_space, action_space, hidden_size: int = 512, num_recurrent_layers: int = 1,
                 rnn_type: str = "GRU", resnet_baseplanes: int = 32, backbone: str = "resnet18",
                 normalize_visual_inputs: bool = False, force_blind_policy: bool = False, policy_config=None,
                 aux_loss_config=None, fuse_keys=None, **kwargs):
        if force_blind_policy:
            raise NotImplementedError("force_blind_policy is not implemented")
        if policy_config is not None and getattr(policy_config, "action_distribution_type", "categorical") != "categorical":
            raise NotImplementedError("only categorical action distributions are implemented")
        super().__init__(PointNavResNetNet(observation_space, action_space, hidden_size, num_recurrent_layers,
                                           rnn_type, backbone, resnet_baseplanes, normalize_visual_inputs,
                                           fuse_keys=fuse_keys),
                         action_space)
        self.observation_space = observation_space
        self._engines: Dict[str, EncoderEngine] = {}

    @classmethod
    def from_config(cls, config, observation_space, action_space, **kwargs):
        hb = config.habitat_baselines
        ignore = []
        try:
            ignore = [s.uuid for s in hb.eval.extra_sim_sensors.values()]
        except Exception:
            pass
        filtered = spaces.Dict(OrderedDict((k, v) for k, v in observation_space.spaces.items() if k not in ignore))
        agent_name = kwargs.get("agent_name")
        policy_cfg = None
        try:
            if agent_name is None:
                agent_name = config.habitat.simulator.agents_order[0]
            policy_cfg = hb.rl.policy[agent_name]
        except Exception:
            pass
        return cls(observation_space=filtered, action_space=action_space, hidden_size=hb.rl.ppo.hidden_size,
                   rnn_type=hb.rl.ddppo.rnn_type, num_recurrent_layers=hb.rl.ddppo.num_recurrent_layers,
                   backbone=hb.rl.ddppo.backbone, normalize_visual_inputs="rgb" in observation_space.spaces,
                   force_blind_policy=getattr(hb, "force_blind_policy", False), policy_config=policy_cfg)

    # ---- encoders -------------------------------------------------------------------------------------------------
    def _encoder(self, name):
        """name: 'visual' or an image-goal uuid -> (ResNetEncoder holder, its fc Sequential)"""
        if name == "visual":
            return self.net.visual_encoder, self.net.visual_fc
        return getattr(self.net, f"{name}_encoder"), getattr(self.net, f"{name}_fc")

    def _fast_prep(self, name) -> bool:
        """True when the vectorised rgb-u8 (x3) / depth-f32 (x1) prep kernels serve this encoder's sensor set"""
        enc, _ = self._encoder(name)
        sp = self.observation_space.spaces
        keys = list(enc.visual_keys)
        kinds = {"rgb": (np.uint8, 3), "depth": (np.float32, 1)}
        src = {k: sp[k] for k in keys} if name == "visual" else {"rgb": sp[name]}
        H, W = enc.in_hw
        return (keys in (["rgb", "depth"], ["rgb"], ["depth"]) and W % 8 == 0 and H % 2 == 0 and
                all(np.dtype(src[k].dtype) == np.dtype(kinds[k][0]) and src[k].shape[2] == kinds[k][1] for k in keys))

    def _engine_(self, name="visual"):
        if name not in self._engines:
            eng = EncoderEngine(self._encoder(name)[0], allow_s2d=self._fast_prep(name))
            eng.side = self._side   # one side stream for the whole backward pass
            self._engines[name] = eng
        return self._engines[name]

    def refresh_inference_weights(self) -> None:
        """Re-pack the weight images now (same buffers) and mark them current: used by GraphedActor, whose
        captured act() step does not contain the packing kernels."""
        self.flatten_parameters_()
        for name in ["visual"] + list(self.net._goal_encoder_uuids):
            eng = self._engine_(name)
            eng.pack_weights()
            eng._packed_key = self.weights_key()

    def _visual_prep(self, name, observations, rows, B, dev, update_stats):
        """Input prep of one encoder (ResNetEncoder.forward, resnet_policy.py:255-271): u8 / f32 / i32 HWC sensors ->
        [running mean/var statistics] -> pooled, normalised fp16 NHWC (+ bf16 twin).  The rgb-u8 + depth-f32 PointNav
        sensor set takes the vectorised kernels, anything else the generic ones."""
        enc, _ = self._encoder(name)
        eng = self._engine_(name)
        H, W = enc.in_hw
        if name == "visual":
            srcs = [(observations[k], enc.key_needs_rescaling[k] or 1.0) for k in enc.visual_keys]
        else:   # goal_visual_encoder({"rgb": goal_image}), resnet_policy.py:739-742
            srcs = [(observations[name], enc.key_needs_rescaling["rgb"] or 1.0)]
        keys = list(enc.visual_keys)
        fast = self._fast_prep(name)
        rgb = srcs[keys.index("rgb")][0] if fast and "rgb" in keys else None
        depth = srcs[keys.index("depth")][0] if fast and "depth" in keys else None
        rgb_scale = srcs[keys.index("rgb")][1] if rgb is not None else 1.0 / 255.0
        rmv = enc.running_mean_and_var
        scale_shift = None
        if isinstance(rmv, RunningMeanAndVar):
            C = enc._n_input_channels
            scale_shift = self._tmp(f"scale_shift/{name}", (16,), dev)
            stats = self._tmp(f"prep_stats/{name}", (17,), dev, torch.float64)
            if update_stats:
                if fast:
                    ops.prep_stats(rgb, depth, rows, H, W, stats, rgb_scale=rgb_scale)
                else:
                    ops.prep_generic(srcs, rows, H, W, stats_acc=stats)
                if self.world_size > 1:  # one packed collective instead of the reference's three
                    torch.distributed.all_reduce(stats, group=self.dist_group)
            ops.prep_finalize(stats, rmv._mean, rmv._var, rmv._count, scale_shift, C, (H // 2) * (W // 2),
                              update_stats)
        s2d = eng.stem.stem_s2d

        def write(x0, x0_bf16=None):
            if fast:
                ops.prep_apply(rgb, depth, rows, H, W, scale_shift, x0, rgb_scale=rgb_scale, s2d=s2d, out_bf16=x0_bf16)
            else:
                ops.prep_generic(srcs, rows, H, W, scale_shift=scale_shift, out=x0, out_bf16=x0_bf16)

        return write

    def _stored_features(self, obs, rows, B, dev):
        """The main encoder's output cached in the observations (VISUAL_FEATURES_KEY, a frozen encoder's rollout) as
        f32 [B, C*h*w]: the step's own rows as they are, a minibatch's rows gathered into one scratch matrix (the
        visual_fc GEMM reads dense rows)."""
        vf = obs[VISUAL_FEATURES_KEY]
        vf = vf.reshape(vf.shape[0], -1)
        if not isinstance(obs, RolloutObservations) and vf.is_contiguous():
            return vf
        feat = self._tmp("visual_features_rows", (B, vf.shape[1]), dev)
        ops.gather_rows(vf, rows, feat)
        return feat

    @torch.no_grad()
    def encode_visual_features(self, observations, out):
        """Run the main visual encoder alone on a batch of observations ([N, ...] tensors) and write its output into
        `out` (f32, N x C x h x w, contiguous): what the trainer stores under VISUAL_FEATURES_KEY after every
        environment step when the encoder is frozen (ppo_trainer.py:261-279, 467-471).  In training mode the
        RunningMeanAndVar statistics are updated first, as the reference's encoder call does."""
        obs, rows = _as_rows(observations, out.device)
        dev = out.device
        if dev.type != "cuda":
            raise Hb200Error("hb200 policy: inputs must be CUDA tensors (no CPU fallback)")
        B = rows.numel()
        self.flatten_parameters_()
        write_x0 = self._visual_prep("visual", obs, rows, B, dev, update_stats=self.training)
        return self._engine_("visual").forward(write_x0, B, dev, False, wkey=self.weights_key(), out=out.view(B, -1))

    def _encode(self, name, obs, rows, B, dev, train, rnn_in, col):
        """one encoder + its Linear/ReLU head into columns [col, col + hidden) of the RNN input"""
        enc, fcs = self._encoder(name)
        if name == "visual" and VISUAL_FEATURES_KEY in obs:
            feat = self._stored_features(obs, rows, B, dev)
        else:
            write_x0 = self._visual_prep(name, obs, rows, B, dev, update_stats=train and self.training)
            feat = self._engine_(name).forward(write_x0, B, dev, train, wkey=self.weights_key())
        fc = fcs[1]
        ops.linear_fwd(feat, fc.weight, fc.bias, rnn_in[:, col:], relu=True, ldc=rnn_in.stride(0), tf32=True)
        return feat

    def _visual_forward(self, obs, rows, pa, mk, B, dev, train):
        net = self.net
        H = net._hidden_size
        D = net.rnn_input_size
        Dp = (D + 3) // 4 * 4                       # row pitch padded to 16 bytes (TF32 GEMM operand rows)
        rnn_in = self._tmp("rnn_in", (B, Dp), dev)[:, :D]
        feats = {"visual": self._encode("visual", obs, rows, B, dev, train, rnn_in, 0)}
        segs = net.segments
        if [sg["kind"] for sg in segs] == ["linear", "prev_action"] and segs[0]["transform"] == ops.T_POLAR2:
            # PointNav sensor set: goal embedding + prev-action embedding in one launch
            ops.embed_fwd(obs[POINTGOAL_UUID].reshape(-1, 2), pa, mk, rows, net.tgt_embeding.weight,
                          net.tgt_embeding.bias, net.prev_action_embedding.weight, rnn_in, H)
        else:
            for sg in segs:
                kind, col = sg["kind"], sg["col"]
                if kind in ("linear", "raw"):
                    x = obs[sg["key"]]
                    x = x.reshape(-1, x.shape[-1])
                    if x.dtype != torch.float32:
                        raise Hb200Error(f"sensor {sg['key']!r}: expected float32 observations")
                    m = getattr(net, sg["attr"]) if kind == "linear" else None
                    ops.sensor_linear_fwd(x, rows, sg["transform"], m.weight if m is not None else None,
                                          m.bias if m is not None else None, rnn_in, col, sg["width"])
                elif kind == "embed":
                    idx = obs[sg["key"]].reshape(-1)
                    if idx.dtype != torch.int64:
                        idx = idx.long()
                    ops.index_embed_fwd(idx, rows, None, getattr(net, sg["attr"]).weight, rnn_in, col, B)
                elif kind == "prev_action":
                    ops.index_embed_fwd(pa, None, mk, net.prev_action_embedding.weight, rnn_in, col, B)
                elif kind == "imagegoal":
                    feats[sg["key"]] = self._encode(sg["key"], obs, rows, B, dev, train, rnn_in, col)
        return rnn_in, dict(feats=feats, rnn_in=rnn_in, stored=VISUAL_FEATURES_KEY in obs)

    def _visual_backward(self, d_rnn_in, s, B, dev):
        net = self.net
        H = net._hidden_size
        v = s["visual"]
        obs, rows, pa, mk = s["obs"], s["rows"], s["pa"], s["masks"]
        segs = net.segments
        if [sg["kind"] for sg in segs] == ["linear", "prev_action"] and segs[0]["transform"] == ops.T_POLAR2:
            tg, emb = net.tgt_embeding, net.prev_action_embedding
            ops.embed_bwd(obs[POINTGOAL_UUID].reshape(-1, 2), pa, mk, rows, d_rnn_in, H, tg.weight.grad, tg.bias.grad,
                          emb.weight.grad)
        else:
            for sg in segs:
                kind, col = sg["kind"], sg["col"]
                if kind == "linear":
                    x = obs[sg["key"]]
                    m = getattr(net, sg["attr"])
                    ops.sensor_linear_bwd(x.reshape(-1, x.shape[-1]), rows, sg["transform"], d_rnn_in, col, sg["width"],
                                          m.weight.grad, m.bias.grad)
                elif kind == "embed":
                    idx = obs[sg["key"]].reshape(-1)
                    ops.index_embed_bwd(idx if idx.dtype == torch.int64 else idx.long(), rows, None, d_rnn_in, col,
                                        getattr(net, sg["attr"]).weight.grad, B)
                elif kind == "prev_action":
                    ops.index_embed_bwd(pa, None, mk, d_rnn_in, col, net.prev_action_embedding.weight.grad, B)
        # encoders: visual_fc (+ image-goal fc) -> conv stacks
        cols = [("visual", 0)] + [(sg["key"], sg["col"]) for sg in segs if sg["kind"] == "imagegoal"]
        for name, col in cols:
            _, fcs = self._encoder(name)
            fc = fcs[1]
            feat = v["feats"][name]
            d_seg, y_seg = d_rnn_in[:, col:], v["rnn_in"][:, col:]
            ops.relu_bwd(d_seg, y_seg, H)
            dvis = d_seg[:, :H]
            with self._side.after_main():
                ops.linear_bwd_weight(dvis, feat, fc.weight.grad, accumulate=True, tf32=True)
                ops.colsum(dvis, fc.bias.grad, n_cols=H)
            if name == "visual" and v["stored"]:   # cached features are inputs: the gradient stops at visual_fc
                continue
            d_feat = self._tmp(f"d_feat/{name}", tuple(feat.shape), dev)
            ops.linear_bwd_input(dvis, fc.weight, d_feat, tf32=True)
            self._engine_(name).backward(d_feat, B, dev)
