"""PointNavBaselinePolicy (SimpleCNN + GRU): BASELINE config #1, on the hb200 kernels.

Mirrors habitat-baselines/habitat_baselines/rl/ppo/policy.py:427-589 (PointNavBaselinePolicy / PointNavBaselineNet)
and rl/models/simple_cnn.py:12-158: three biased convolutions (8x8 s4 -> ReLU -> 4x4 s2 -> ReLU -> 3x3 s1) ->
Flatten -> Linear -> ReLU, concatenated with the raw 2-D pointgoal, into a 1-layer GRU.  state_dict keys and
initialisers are the reference's (the torch.nn modules are parameter holders only)."""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from .. import ops
from ..common.baseline_registry import baseline_registry
from .resnet_policy import BF16, F16, POINTGOAL_UUID, NativeNetPolicy, _GRUStateEncoder


class SimpleCNN(nn.Module):
    def __init__(self, observation_space, output_size):
        super().__init__()
        sp = observation_space.spaces
        self._n_input_rgb = sp["rgb"].shape[2] if "rgb" in sp else 0
        self._n_input_depth = sp["depth"].shape[2] if "depth" in sp else 0
        self._kernels, self._strides = [8, 4, 3], [4, 2, 1]
        if self.is_blind:
            raise NotImplementedError("blind SimpleCNN is not implemented")
        hw = np.array((sp["rgb"] if self._n_input_rgb else sp["depth"]).shape[:2])
        self.in_hw = tuple(int(v) for v in hw)
        dims = [self.in_hw]
        for k, s in zip(self._kernels, self._strides):
            hw = (hw - k) // s + 1
            dims.append(tuple(int(v) for v in hw))
        self.dims = dims
        cin = self._n_input_rgb + self._n_input_depth
        self.cnn = nn.Sequential(
            nn.Conv2d(cin, 32, 8, 4), nn.ReLU(True), nn.Conv2d(32, 64, 4, 2), nn.ReLU(True), nn.Conv2d(64, 32, 3, 1),
            nn.Flatten(), nn.Linear(32 * dims[3][0] * dims[3][1], output_size), nn.ReLU(True))
        for layer in self.cnn:  # simple_cnn.py:125-133
            if isinstance(layer, (nn.Conv2d, nn.Linear)):
                nn.init.kaiming_normal_(layer.weight, nn.init.calculate_gain("relu"))
                nn.init.constant_(layer.bias, val=0)

    @property
    def is_blind(self):
        return self._n_input_rgb + self._n_input_depth == 0


class PointNavBaselineNet(nn.Module):
    def __init__(self, observation_space, hidden_size):
        super().__init__()
        if POINTGOAL_UUID not in observation_space.spaces:
            raise NotImplementedError("PointNavBaselineNet: only the pointgoal_with_gps_compass goal is implemented")
        self._n_input_goal = observation_space.spaces[POINTGOAL_UUID].shape[0]
        self._hidden_size = hidden_size
        self.visual_encoder = SimpleCNN(observation_space, hidden_size)
        self.state_encoder = _GRUStateEncoder(hidden_size + self._n_input_goal, hidden_size)
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


@baseline_registry.register_policy
class PointNavBaselinePolicy(NativeNetPolicy):
    def __init__(self, observation_space, action_space, hidden_size: int = 512, aux_loss_config=None,
                 policy_config=None, **kwargs):
        if getattr(policy_config, "action_distribution_type", "categorical") != "categorical":
            raise NotImplementedError("PointNavBaselinePolicy (SimpleCNN) implements the categorical action "
                                      "distribution only")
        super().__init__(PointNavBaselineNet(observation_space, hidden_size), action_space)
        self.observation_space = observation_space
        self._ws = {}
        self._wimgs = None

    @classmethod
    def from_config(cls, config, observation_space, action_space, **kwargs):
        hb = config.habitat_baselines
        agent_name = kwargs.get("agent_name")
        if agent_name is None:   # configs without a simulator section describe a single, categorical agent
            simulator = getattr(getattr(config, "habitat", None), "simulator", None)
            agent_name = getattr(simulator, "agents_order", [None])[0]
        policies = getattr(hb.rl, "policy", {})
        policy_cfg = policies[agent_name] if agent_name in policies else None
        return cls(observation_space=observation_space, action_space=action_space, hidden_size=hb.rl.ppo.hidden_size,
                   policy_config=policy_cfg)

    # ---- conv stack bookkeeping ------------------------------------------------------------------------
    def _layers(self):
        cnn = self.net.visual_encoder
        convs = [cnn.cnn[0], cnn.cnn[2], cnn.cnn[4]]
        return convs, cnn.cnn[6], cnn.dims

    def _workspace(self, B, dev, train):
        key = (B, train)
        if key in self._ws and self._ws[key]["x0"].device == dev:
            return self._ws[key]
        convs, fc, dims = self._layers()
        e = lambda *s: torch.empty(*s, dtype=BF16, device=dev)  # noqa: E731  (gradients)
        ea = lambda *s: torch.empty(*s, dtype=F16, device=dev)  # noqa: E731  (forward values)
        ws = {"x0": ea(B, *dims[0], 8)}
        for i, c in enumerate(convs):
            ws[f"a{i}"] = ea(B, *dims[i + 1], c.out_channels)
        ws["flat"] = torch.empty(B, fc.in_features, device=dev)
        if train:
            ws["x0_b"] = e(B, *dims[0], 8)                 # bf16 twins of the conv inputs (weight-gradient operand)
            for i, c in enumerate(convs[:-1]):
                ws[f"a{i}_b"] = e(B, *dims[i + 1], c.out_channels)
            for i, c in enumerate(convs):
                ws[f"g{i}"] = e(B, *dims[i + 1], c.out_channels)
                ws[f"dy{i}"] = e(B, *dims[i + 1], c.out_channels)
            ws["dflat"] = torch.empty(B, fc.in_features, device=dev)
        self._ws[key] = ws
        return ws

    def _pack(self, dev):
        convs, _, _ = self._layers()
        if self._wimgs is None or self._wimgs[0][0].device != dev:
            self._wimgs = []
            for i, c in enumerate(convs):
                co, ci, k, _ = c.weight.shape
                cip = 8 if i == 0 else ci
                wp = torch.empty(ops.packed_weight_elems(co, cip, k, k), dtype=F16, device=dev)
                wt = torch.empty(ops.packed_weight_elems(cip, co, k, k), dtype=BF16, device=dev) if i > 0 else None
                acc = torch.empty(k * k * cip, co, device=dev)
                self._wimgs.append((wp, wt, acc, cip))
        for c, (wp, wt, _, cip) in zip(convs, self._wimgs):
            ops.pack_conv_weight_into(c.weight.data, wp, wt, cip)

    def _shape(self, i, B):
        convs, _, dims = self._layers()
        c = convs[i]
        cip = self._wimgs[i][3]
        return ops.conv_shape(B, dims[i][0], dims[i][1], cip, c.out_channels, c.kernel_size[0], c.kernel_size[0],
                              c.stride[0], 0)

    # ---- hooks ----------------------------------------------------------------------------------------------
    def _visual_forward(self, obs, rows, pa, mk, B, dev, train):
        cnn = self.net.visual_encoder
        convs, fc, dims = self._layers()
        ws = self._workspace(B, dev, train)
        self._pack(dev)
        H, W = dims[0]
        ops.prep_plain(obs.get("rgb") if cnn._n_input_rgb else None, obs.get("depth") if cnn._n_input_depth else None,
                       rows, H, W, cnn._n_input_rgb, cnn._n_input_depth, ws["x0"])
        x = ws["x0"]
        if train:
            ops.f16_to_bf16(x, ws["x0_b"])
        for i, c in enumerate(convs):
            ops.conv_bias_act_fwd(x, self._wimgs[i][0], c.bias, ws[f"a{i}"], self._shape(i, B), relu=(i < 2))
            x = ws[f"a{i}"]
            if train and i < len(convs) - 1:
                ops.f16_to_bf16(x, ws[f"a{i}_b"])
        hw3 = dims[3][0] * dims[3][1]
        ops.bf16_hwc_to_f32_chw(x, ws["flat"], B, hw3, convs[2].out_channels)
        Hs = self.net._hidden_size
        D = Hs + self.net._n_input_goal
        Dp = (D + 3) // 4 * 4                      # row pitch padded to 16 bytes
        rnn_in_full = self._tmp("rnn_in_b", (B, Dp), dev)
        rnn_in = rnn_in_full[:, :D]
        ops.linear_fwd(ws["flat"], fc.weight, fc.bias, rnn_in_full, relu=True, ldc=Dp, tf32=True)
        goal = obs[POINTGOAL_UUID].reshape(-1, self.net._n_input_goal)
        rnn_in[:, Hs:] = goal[rows.long()]          # raw goal vector appended (policy.py:571-580); tiny gather
        return rnn_in, dict(ws=ws, rnn_in=rnn_in_full)

    def _visual_backward(self, d_rnn_in, s, B, dev):
        convs, fc, dims = self._layers()
        v = s["visual"]
        ws = v["ws"]
        Hs = self.net._hidden_size
        ops.relu_bwd(d_rnn_in, v["rnn_in"], Hs)
        dvis = d_rnn_in[:, :Hs]
        ops.linear_bwd_weight(dvis, ws["flat"], fc.weight.grad, accumulate=True, tf32=True)
        ops.colsum(dvis, fc.bias.grad, n_cols=Hs)
        ops.linear_bwd_input(dvis, fc.weight, ws["dflat"], tf32=True)
        hw3 = dims[3][0] * dims[3][1]
        ops.f32_chw_to_bf16_hwc(ws["dflat"], ws["g2"], B, hw3, convs[2].out_channels)
        g = ws["g2"]
        for i in (2, 1, 0):
            c = convs[i]
            npix = B * dims[i + 1][0] * dims[i + 1][1]
            if i == 2:   # no ReLU after the last conv: dy = g
                ops.relu_bias_bwd(g, None, None, c.bias.grad, npix, c.out_channels)
                dy = g
            else:
                ops.relu_bias_bwd(g, ws[f"a{i}"], ws[f"dy{i}"], c.bias.grad, npix, c.out_channels)
                dy = ws[f"dy{i}"]
            wp, wt, acc, cip = self._wimgs[i]
            x = ws[f"a{i - 1}_b"] if i > 0 else ws["x0_b"]
            acc.zero_()
            ops.conv_wgrad(x, dy, acc, self._shape(i, B))
            ops.unpack_conv_wgrad(acc, c.weight.grad, cip)
            if i > 0:
                ops.conv_dgrad(dy, wt, ws[f"g{i - 1}"], self._shape(i, B))
                g = ws[f"g{i - 1}"]
