"""Observation transformers with the reference's classes, config fields and helpers
(habitat-baselines/habitat_baselines/common/obs_transformers.py:47-232, 1201-1242; the image helpers
utils/common.py:481-581), run on the GPU by the fused resample-and-window kernel (ops.obs_resample).

ResizeShortestEdge and CenterCropper are supported for channels-last 3-D (HWC) and 4-D (NHWC) tensors.  Their
results are bit-identical to the reference's torch ops on the CPU.  The trainer does not call them one by one: it
compiles the active list into an ObsTransformPlan, which writes every transformed key straight into the rollout
storage in one launch.
"""
from __future__ import annotations

import copy
import numbers
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Tuple

import torch
from torch import nn

from .. import ops
from .._lib import Hb200Error
from .baseline_registry import baseline_registry

_DEFAULT_KEYS = ("rgb", "depth", "semantic")
# the reference's other registered transformers; none has a GPU implementation here
_UNSUPPORTED = ("CubeMap2Equirect", "CubeMap2Fisheye", "Equirect2CubeMap", "AddVirtualKeys")


# ---- config nodes (habitat_baselines/config/default_structured_configs.py: resize_shortest_edge_base,
#      center_cropper_base) ---------------------------------------------------------------------------------------
@dataclass
class ResizeShortestEdgeConfig:
    type: str = "ResizeShortestEdge"
    size: int = 256
    channels_last: bool = True
    trans_keys: Tuple[str, ...] = _DEFAULT_KEYS
    semantic_key: str = "semantic"


@dataclass
class CenterCropperConfig:
    type: str = "CenterCropper"
    height: int = 256
    width: int = 256
    channels_last: bool = True
    trans_keys: Tuple[str, ...] = _DEFAULT_KEYS


# ---- shape rules ------------------------------------------------------------------------------------------------
def resized_hw(h: int, w: int, size: int) -> Tuple[int, int]:
    """The reference's float64 expression: int(h * (size / min(h, w))).  It is not integer arithmetic: a short
    edge of 392 at size 256 gives 255 (392 x 520 -> 255 x 339)."""
    scale = size / min(h, w)
    return int(h * scale), int(w * scale)


def crop_origin(h: int, w: int, size: Tuple[int, int]) -> Tuple[int, int]:
    """(y0, x0) of the reference's center_crop; raises where its slice would start before the image or run past
    it (the reference then silently returns a tensor smaller than its own observation space)."""
    ch, cw = size
    if ch > h or cw > w:
        raise Hb200Error(f"CenterCropper: crop {ch}x{cw} is larger than the {h}x{w} image")
    return h // 2 - ch // 2, w // 2 - cw // 2


def _image_hw(shape, what) -> Tuple[int, int]:
    if len(shape) != 3:
        raise NotImplementedError(f"{what}: only channels-last HWC images are supported, got shape {tuple(shape)}")
    return int(shape[0]), int(shape[1])


def _overwrite_box_shape(box, hw):
    if tuple(box.shape[:2]) == tuple(hw):
        return box
    low = box.low if box.low.ndim == 0 else box.low.min()
    high = box.high if box.high.ndim == 0 else box.high.max()
    return type(box)(low=low, high=high, shape=(*hw, *box.shape[2:]), dtype=box.dtype)


def _batched(img: torch.Tensor, what: str) -> torch.Tensor:
    if img.dim() == 3:
        return img.unsqueeze(0)
    if img.dim() != 4:
        raise NotImplementedError(f"{what}: only HWC / NHWC tensors are supported, got {img.dim()}-D "
                                  f"{tuple(img.shape)}")
    return img


def _check_channels_last(channels_last: bool, what: str) -> None:
    if not channels_last:
        raise NotImplementedError(f"{what}: channels_last=False (NCHW) is not supported")


# ---- transformers -----------------------------------------------------------------------------------------------
class ObservationTransformer(nn.Module):
    """Base class: transform_observation_space + in-place forward on an observation dict."""

    def transform_observation_space(self, observation_space, **kwargs):
        return observation_space

    @classmethod
    def from_config(cls, config):
        raise NotImplementedError

    def forward(self, observations: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        return observations


@baseline_registry.register_obs_transformer()
class ResizeShortestEdge(ObservationTransformer):
    """Resizes the shortest edge of every `trans_keys` image to `size`, keeping the aspect ratio: area resampling,
    nearest for keys containing `semantic_key`."""

    def __init__(self, size: int, channels_last: bool = True, trans_keys: Tuple[str, ...] = _DEFAULT_KEYS,
                 semantic_key: str = "semantic"):
        super().__init__()
        _check_channels_last(channels_last, "ResizeShortestEdge")
        self._size = size
        self.channels_last = channels_last
        self.trans_keys = tuple(trans_keys)
        self.semantic_key = semantic_key

    def mode(self, key: str) -> int:
        return ops.OBS_NEAREST if self.semantic_key in key else ops.OBS_AREA

    def transform_observation_space(self, observation_space, **kwargs):
        observation_space = copy.deepcopy(observation_space)
        if self._size:
            for key in observation_space.spaces:
                if key in self.trans_keys:
                    h, w = _image_hw(observation_space.spaces[key].shape, "ResizeShortestEdge")
                    if self._size == min(h, w):
                        continue
                    observation_space.spaces[key] = _overwrite_box_shape(observation_space.spaces[key],
                                                                         resized_hw(h, w, self._size))
        return observation_space

    @torch.no_grad()
    def forward(self, observations: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self._size is not None:
            for key in self.trans_keys:
                if key in observations:
                    img = observations[key]
                    x = _batched(img, "ResizeShortestEdge")
                    hr, wr = resized_hw(x.shape[1], x.shape[2], self._size)
                    out = torch.empty((x.shape[0], hr, wr, x.shape[3]), dtype=x.dtype, device=x.device)
                    ops.obs_resample([(x, out, self.mode(key), (hr, wr), (0, 0))])
                    observations[key] = out if img.dim() == 4 else out[0]
        return observations

    @classmethod
    def from_config(cls, config):
        return cls(config.size, config.channels_last, config.trans_keys, config.semantic_key)


@baseline_registry.register_obs_transformer()
class CenterCropper(ObservationTransformer):
    """Center-crops every `trans_keys` image to `size` (an int or (h, w)); forward returns the reference's slice
    view."""

    def __init__(self, size, channels_last: bool = True, trans_keys: Tuple[str, ...] = _DEFAULT_KEYS):
        super().__init__()
        _check_channels_last(channels_last, "CenterCropper")
        if isinstance(size, numbers.Integral):
            size = (int(size), int(size))
        size = tuple(int(s) for s in size)
        assert len(size) == 2, "forced input size must be len of 2 (h, w)"
        self._size = size
        self.channels_last = channels_last
        self.trans_keys = tuple(trans_keys)

    def transform_observation_space(self, observation_space, **kwargs):
        observation_space = copy.deepcopy(observation_space)
        for key in observation_space.spaces:
            if key in self.trans_keys and tuple(observation_space.spaces[key].shape[-3:-1]) != self._size:
                _image_hw(observation_space.spaces[key].shape, "CenterCropper")
                observation_space.spaces[key] = _overwrite_box_shape(observation_space.spaces[key], self._size)
        return observation_space

    @torch.no_grad()
    def forward(self, observations: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        for key in self.trans_keys:
            if key in observations:
                img = observations[key]
                _batched(img, "CenterCropper")
                y0, x0 = crop_origin(img.shape[-3], img.shape[-2], self._size)
                observations[key] = img[..., y0:y0 + self._size[0], x0:x0 + self._size[1], :]
        return observations

    @classmethod
    def from_config(cls, config):
        return cls((config.height, config.width), config.channels_last, config.trans_keys)


# ---- the reference's helpers --------------------------------------------------------------------------------------
def get_active_obs_transforms(config, agent_name: Optional[str] = None) -> List[ObservationTransformer]:
    """The transformers configured under rl.policy.<first agent>.obs_transforms, in order (the reference also
    ignores `agent_name`: the observation space is shared among agents)."""
    policy = config.habitat_baselines.rl.policy
    agent_name = list(policy.keys())[0]
    active = []
    for cfg in (getattr(policy[agent_name], "obs_transforms", None) or {}).values():
        if cfg.type in _UNSUPPORTED:
            raise NotImplementedError(f"observation transformer {cfg.type} has no GPU implementation "
                                      "(ResizeShortestEdge and CenterCropper do)")
        cls = baseline_registry.get_obs_transformer(cfg.type)
        if cls is None:
            raise ValueError(f"Unknown ObservationTransform with name {cfg.type}.")
        active.append(cls.from_config(cfg))
    return active


def apply_obs_transforms_batch(batch: Dict[str, torch.Tensor],
                               obs_transforms: Iterable[ObservationTransformer]) -> Dict[str, torch.Tensor]:
    for t in obs_transforms:
        batch = t(batch)
    return batch


def apply_obs_transforms_obs_space(obs_space, obs_transforms: Iterable[ObservationTransformer]):
    for t in obs_transforms:
        obs_space = t.transform_observation_space(obs_space)
    return obs_space


# ---- the trainer's fused form -----------------------------------------------------------------------------------
class ObsTransformPlan:
    """An active list of at most one ResizeShortestEdge followed by at most one CenterCropper, compiled per key into
    one resample-and-window launch that writes the transformed observations into caller-owned tensors (the
    rollout storage's next slot) with the same bits the two transformers produce one after the other."""

    def __init__(self, obs_transforms: List[ObservationTransformer], raw_space):
        kinds = [type(t) for t in obs_transforms]
        if kinds not in ([], [ResizeShortestEdge], [CenterCropper], [ResizeShortestEdge, CenterCropper]):
            raise NotImplementedError("fused observation transforms support at most one ResizeShortestEdge followed "
                                      f"by at most one CenterCropper, got {[k.__name__ for k in kinds]}")
        resize = next((t for t in obs_transforms if isinstance(t, ResizeShortestEdge)), None)
        crop = next((t for t in obs_transforms if isinstance(t, CenterCropper)), None)
        self.keys: Dict[str, tuple] = {}   # key -> (mode, (Hr, Wr), (y0, x0), (h, w))
        for key, sp in raw_space.spaces.items():
            resized = resize is not None and resize._size is not None and key in resize.trans_keys
            cropped = crop is not None and key in crop.trans_keys
            if not (resized or cropped):
                continue
            h, w = _image_hw(sp.shape, "observation transforms")
            mode, hr, wr = ops.OBS_COPY, h, w
            if resized:
                mode = resize.mode(key)
                hr, wr = resized_hw(h, w, resize._size)
            y0, x0, oh, ow = 0, 0, hr, wr
            if cropped:
                (y0, x0), (oh, ow) = crop_origin(hr, wr, crop._size), crop._size
            self.keys[key] = (mode, (hr, wr), (y0, x0), (oh, ow))

    def __bool__(self):
        return bool(self.keys)

    def apply_(self, observations: Dict[str, torch.Tensor], out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """Writes every planned key of `observations` into out[key] ([N, h, w, C], contiguous) in one launch; returns
        the observations the plan does not touch."""
        jobs = []
        for key, (mode, hw_r, origin, hw) in self.keys.items():
            src, dst = observations[key], out[key]
            if tuple(dst.shape[1:3]) != hw:
                raise Hb200Error(f"observation transforms: {key} target {tuple(dst.shape)} is not {hw}")
            jobs.append((src, dst, mode, hw_r, origin))
        if jobs:
            ops.obs_resample(jobs)
        return {k: v for k, v in observations.items() if k not in self.keys}
