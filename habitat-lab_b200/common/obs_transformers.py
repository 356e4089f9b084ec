"""Observation transformers with the reference's classes, config fields and helpers
(habitat-baselines/habitat_baselines/common/obs_transformers.py:47-232, 864-1242; the image helpers
utils/common.py:481-581), run on the GPU by the fused resample-and-window kernel (ops.obs_resample) and the cube-map
projection kernel (ops.obs_project).

ResizeShortestEdge and CenterCropper are supported for channels-last 3-D (HWC) and 4-D (NHWC) tensors;
CubeMap2Equirect, CubeMap2Fisheye and Equirect2CubeMap for 4-D (NHWC) tensors.  Their results are bit-identical to
the reference's torch ops on the CPU.  The trainer does not call them one by one: it compiles the active list into an
ObsTransformPlan, which writes every transformed key straight into the rollout storage.
"""
from __future__ import annotations

import copy
import numbers
from dataclasses import dataclass, field
from typing import Dict, Iterable, List, Optional, Tuple

import torch
from torch import nn

from .. import ops
from .._lib import Hb200Error
from . import projection
from .baseline_registry import baseline_registry

_DEFAULT_KEYS = ("rgb", "depth", "semantic")
# the reference's other registered transformer; it has no GPU implementation here
_UNSUPPORTED = ("AddVirtualKeys",)


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


# (default_structured_configs.py: cube_2_eq_base, cube_2_fish_base, eq_2_cube_base)
def _cube_faces():
    return list(projection.CUBE_FACES)


@dataclass
class Cube2EqConfig:
    type: str = "CubeMap2Equirect"
    height: int = 256
    width: int = 512
    sensor_uuids: List[str] = field(default_factory=_cube_faces)


@dataclass
class Cube2FishConfig:
    type: str = "CubeMap2Fisheye"
    height: int = 256
    width: int = 256
    fov: int = 180
    params: Tuple[float, ...] = (0.2, 0.2, 0.2)
    sensor_uuids: List[str] = field(default_factory=_cube_faces)


@dataclass
class Eq2CubeConfig:
    type: str = "Equirect2CubeMap"
    height: int = 256
    width: int = 256
    sensor_uuids: List[str] = field(default_factory=_cube_faces)


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


class ProjectionTransformer(ObservationTransformer):
    """Stitches each group of `stitch`'s input count of sensors (six cube faces, or one panorama) into the group's
    target sensor (by default its first), in one ops.obs_project launch for all groups.  A group is depth when
    `depth_key` is a substring of one of its uuids; its z-depth faces are converted as the reference converts them.
    The other sensors of a group stay in the observations unchanged."""

    def __init__(self, stitch: projection.Stitch, sensor_uuids: List[str], image_shape: Tuple[int, int],
                 channels_last: bool = False, target_uuids: Optional[List[str]] = None, depth_key: str = "depth"):
        super().__init__()
        name = type(self).__name__
        if channels_last:
            # the reference then feeds NHWC tensors to grid_sample as if they were NCHW
            raise NotImplementedError(f"{name}: channels_last=True is not supported (the inputs are NHWC with "
                                      "channels_last=False, the reference's configured path)")
        n_in = len(stitch.inputs)
        sensor_uuids = list(sensor_uuids)
        if not sensor_uuids or len(sensor_uuids) % n_in:
            raise ValueError(f"{name}: {len(sensor_uuids)} sensors is not a multiple of {n_in}")
        if len(image_shape) != 2:
            raise ValueError(f"{name}: image_shape must be (height, width), got {image_shape}")
        self.stitch = stitch
        self.sensor_uuids = sensor_uuids
        self.img_shape = (int(image_shape[0]), int(image_shape[1]))
        self.channels_last = channels_last
        self.target_uuids = list(sensor_uuids[::6] if target_uuids is None else target_uuids)
        self.depth_key = depth_key
        self.groups = []   # (target uuid, input uuids, is_depth)
        for i, target in enumerate(self.target_uuids):
            uuids = sensor_uuids[i * n_in:(i + 1) * n_in]
            if target not in uuids:
                raise ValueError(f"{name}: target {target} is not one of its input sensors {uuids}")
            self.groups.append((target, uuids, any(depth_key in u for u in uuids)))
        self._tables: Dict[torch.device, tuple] = {}

    @property
    def n_out(self) -> int:
        return len(self.stitch.outputs)

    def check_faces(self, is_depth: bool, hw: Tuple[int, int]) -> None:
        """Refuses faces the reference cannot convert: smaller than 3x3 (unassigned inputs would not sample to an
        exact 0), or depth faces of another size than the stitch's fixed cameras (a broadcast error there)."""
        name = type(self).__name__
        if hw[0] < 3 or hw[1] < 3:
            raise Hb200Error(f"{name}: input faces of {hw[0]}x{hw[1]} (at least 3x3)")
        if is_depth and self.stitch.in_zfactor is not None and tuple(hw) != self.stitch.in_hw:
            raise Hb200Error(f"{name}: depth faces of {hw[0]}x{hw[1]}; its z-depth conversion is defined for "
                             f"{self.stitch.in_hw[0]}x{self.stitch.in_hw[1]} faces only")

    def device_tables(self, device: torch.device):
        """(table, in_zf, out_zf) on `device`, built once: the table is normalised, so one serves every face size."""
        if device not in self._tables:
            s = self.stitch
            self._tables[device] = (
                s.table().to(device),
                None if s.in_zfactor is None else s.in_zfactor[:, 0].contiguous().to(device),
                None if s.out_zfactor is None else s.out_zfactor[:, 0].contiguous().to(device))
        return self._tables[device]

    def jobs(self, observations: Dict[str, torch.Tensor], outs: Dict[str, torch.Tensor]) -> list:
        """One ops.obs_project job per group, writing outs[target]."""
        jobs = []
        for target, uuids, is_depth in self.groups:
            faces = [observations[u] for u in uuids]
            if faces[0].dim() != 4:
                raise NotImplementedError(f"{type(self).__name__}: only NHWC batches are supported, got "
                                          f"{tuple(faces[0].shape)} for {uuids[0]}")
            self.check_faces(is_depth, tuple(faces[0].shape[1:3]))
            table, in_zf, out_zf = self.device_tables(faces[0].device)
            jobs.append((faces, outs[target], table, in_zf if is_depth else None, out_zf if is_depth else None))
        return jobs

    def transform_observation_space(self, observation_space, **kwargs):
        observation_space = copy.deepcopy(observation_space)
        for target, uuids, is_depth in self.groups:
            if target not in observation_space.spaces:
                raise KeyError(f"{target} not found in observation space: {list(observation_space.spaces)}")
            shape = observation_space.spaces[target].shape
            self.check_faces(is_depth, _image_hw(shape, type(self).__name__))
            observation_space.spaces[target] = _overwrite_box_shape(observation_space.spaces[target], self.img_shape)
        return observation_space

    @torch.no_grad()
    def forward(self, observations: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        outs = {}
        for target, uuids, _ in self.groups:
            f = observations[uuids[0]]
            outs[target] = torch.empty((f.shape[0] * self.n_out, *self.img_shape, f.shape[-1]), dtype=f.dtype,
                                       device=f.device)
        jobs = self.jobs(observations, outs)
        for i in range(0, len(jobs), ops.OBS_PROJECT_MAX_TARGETS):
            ops.obs_project(jobs[i:i + ops.OBS_PROJECT_MAX_TARGETS])
        observations.update(outs)
        return observations


def _target_uuids(config):
    return getattr(config, "target_uuids", None)


@baseline_registry.register_obs_transformer()
class CubeMap2Equirect(ProjectionTransformer):
    """Stitches six 90 degree cameras (Back, Down, Front, Left, Right, Up) into an eq_shape equirectangular panorama.
    The cube cameras are fixed at 256 x 256: RGB faces of any size work, depth faces must be 256 x 256."""

    def __init__(self, sensor_uuids: List[str], eq_shape: Tuple[int, int], channels_last: bool = False,
                 target_uuids: Optional[List[str]] = None, depth_key: str = "depth"):
        super().__init__(projection.cube_to_equirect(*eq_shape), sensor_uuids, eq_shape, channels_last, target_uuids,
                         depth_key)

    @classmethod
    def from_config(cls, config):
        return cls(config.sensor_uuids, eq_shape=(config.height, config.width), target_uuids=_target_uuids(config))


@baseline_registry.register_obs_transformer()
class CubeMap2Fisheye(ProjectionTransformer):
    """Stitches six 90 degree cameras (Back, Down, Front, Left, Right, Up) into a double-sphere fisheye of fish_shape,
    fish_fov degrees and fish_params (f, xi, alpha).  The cube cameras have the fisheye's size: depth faces must
    too."""

    def __init__(self, sensor_uuids: List[str], fish_shape: Tuple[int, int], fish_fov: float,
                 fish_params: Tuple[float, float, float], channels_last: bool = False,
                 target_uuids: Optional[List[str]] = None, depth_key: str = "depth"):
        super().__init__(projection.cube_to_fisheye(fish_shape[0], fish_shape[1], fish_fov, fish_params),
                         sensor_uuids, fish_shape, channels_last, target_uuids, depth_key)

    @classmethod
    def from_config(cls, config):
        return cls(config.sensor_uuids, fish_shape=(config.height, config.width), fish_fov=config.fov,
                   fish_params=config.params, target_uuids=_target_uuids(config))


@baseline_registry.register_obs_transformer()
class Equirect2CubeMap(ProjectionTransformer):
    """Resamples a 256 x 512 equirectangular panorama into six img_shape cube faces (Back, Down, Front, Left, Right,
    Up), returned as the reference returns them: [6 * B, h, w, C], env-major, under the target uuid."""

    def __init__(self, sensor_uuids: List[str], img_shape: Tuple[int, int], channels_last: bool = False,
                 target_uuids: Optional[List[str]] = None, depth_key: str = "depth"):
        super().__init__(projection.equirect_to_cube(*img_shape), sensor_uuids, img_shape, channels_last,
                         target_uuids, depth_key)

    @classmethod
    def from_config(cls, config):
        return cls(config.sensor_uuids, img_shape=(config.height, config.width), target_uuids=_target_uuids(config))


_PROJECTION_FIELDS = {"CubeMap2Equirect": ("sensor_uuids", "height", "width"),
                      "CubeMap2Fisheye": ("sensor_uuids", "height", "width", "fov", "params"),
                      "Equirect2CubeMap": ("sensor_uuids", "height", "width")}


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
                                      "(ResizeShortestEdge, CenterCropper and the cube-map projections do)")
        missing = [f for f in _PROJECTION_FIELDS.get(cfg.type, ()) if not hasattr(cfg, f)]
        if missing:
            raise NotImplementedError(f"observation transformer {cfg.type}: the config node has no {missing}, so "
                                      "there is no camera rig to build (see Cube2EqConfig / Cube2FishConfig / "
                                      "Eq2CubeConfig)")
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
    rollout storage's next slot) with the same bits the two transformers produce one after the other.  The list may
    also hold one CubeMap2Equirect or CubeMap2Fisheye, which adds one projection launch for all its targets; it must
    not share a key with the resize / crop pair."""

    def __init__(self, obs_transforms: List[ObservationTransformer], raw_space):
        projections = [t for t in obs_transforms if isinstance(t, ProjectionTransformer)]
        if any(isinstance(t, Equirect2CubeMap) for t in projections):
            raise NotImplementedError("Equirect2CubeMap returns six images per environment ([6 * B, h, w, C]), which "
                                      "no rollout storage holds")
        if len(projections) > 1:
            raise NotImplementedError("fused observation transforms support at most one projection transform, got "
                                      f"{[type(t).__name__ for t in projections]}")
        self.projection: Optional[ProjectionTransformer] = projections[0] if projections else None
        obs_transforms = [t for t in obs_transforms if not isinstance(t, ProjectionTransformer)]
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
        self.projected: Tuple[str, ...] = ()   # the projection's targets
        if self.projection is not None:
            shared = sorted(set(self.projection.sensor_uuids) & set(self.keys))
            if shared:
                raise NotImplementedError(f"{type(self.projection).__name__} reads or writes {shared}, which are also "
                                          "resized or cropped: a key takes one of the two")
            if len(self.projection.groups) > ops.OBS_PROJECT_MAX_TARGETS:
                raise NotImplementedError(f"{len(self.projection.groups)} projection targets (at most "
                                          f"{ops.OBS_PROJECT_MAX_TARGETS} in one launch)")
            for _, uuids, is_depth in self.projection.groups:
                self.projection.check_faces(is_depth, _image_hw(raw_space.spaces[uuids[0]].shape,
                                                                type(self.projection).__name__))
            self.projected = tuple(t for t, _, _ in self.projection.groups)

    def __bool__(self):
        return bool(self.keys) or self.projection is not None

    def apply_(self, observations: Dict[str, torch.Tensor], out: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """Writes every planned key of `observations` into out[key] ([N, h, w, C], contiguous): one launch for the
        resized / cropped keys, one for the projection targets.  Returns the observations the plan does not write
        (a projection's other input faces among them)."""
        if self.projection is not None:
            ops.obs_project(self.projection.jobs(observations, out))
        jobs = []
        for key, (mode, hw_r, origin, hw) in self.keys.items():
            src, dst = observations[key], out[key]
            if tuple(dst.shape[1:3]) != hw:
                raise Hb200Error(f"observation transforms: {key} target {tuple(dst.shape)} is not {hw}")
            jobs.append((src, dst, mode, hw_r, origin))
        if jobs:
            ops.obs_resample(jobs)
        return {k: v for k, v in observations.items() if k not in self.keys and k not in self.projected}
