"""Synthetic PointNav RGB-D rollouts of the reference's shapes/dtypes (habitat-sim is stubbed out of
the learner loop): rgb u8 HxWx3 (habitat_simulator.py:116-127), depth f32 HxWx1 in [0,1] (:157-162),
pointgoal_with_gps_compass f32[2]."""
from __future__ import annotations

import math

import numpy as np
import torch

from .common import spaces


def pointnav_spaces(H=256, W=256, n_actions=4):
    obs = spaces.Dict({
        "rgb": spaces.Box(0, 255, (H, W, 3), np.uint8),
        "depth": spaces.Box(0.0, 1.0, (H, W, 1), np.float32),
        "pointgoal_with_gps_compass": spaces.Box(np.finfo(np.float32).min, np.finfo(np.float32).max, (2,), np.float32),
    })
    return obs, spaces.Discrete(n_actions)


def objectnav_spaces(H=256, W=256, n_actions=6, n_categories=21):
    """ObjectNav sensor set of BASELINE config #3 (ddppo_objectnav.yaml): rgb u8, depth f32, the int32 `semantic` channel
    (habitat_simulator.py:197-209), objectgoal category id (object_nav_task.py ObjectGoalSensor), compass, gps."""
    import collections
    od = collections.OrderedDict()
    od["rgb"] = spaces.Box(0, 255, (H, W, 3), np.uint8)
    od["depth"] = spaces.Box(0.0, 1.0, (H, W, 1), np.float32)
    od["semantic"] = spaces.Box(0, 2 ** 30, (H, W, 1), np.int32)
    od["objectgoal"] = spaces.Box(0, n_categories - 1, (1,), np.int64)
    od["compass"] = spaces.Box(-np.pi, np.pi, (1,), np.float32)
    od["gps"] = spaces.Box(np.finfo(np.float32).min, np.finfo(np.float32).max, (2,), np.float32)
    return spaces.Dict(od), spaces.Discrete(n_actions)


def imagenav_spaces(H=256, W=256, n_actions=4):
    """ImageNav sensor set of BASELINE config #4 (ddppo_imagenav_example.yaml): rgb + the goal image, compass, gps."""
    import collections
    od = collections.OrderedDict()
    od["rgb"] = spaces.Box(0, 255, (H, W, 3), np.uint8)
    od["imagegoal"] = spaces.Box(0, 255, (H, W, 3), np.uint8)
    od["compass"] = spaces.Box(-np.pi, np.pi, (1,), np.float32)
    od["gps"] = spaces.Box(np.finfo(np.float32).min, np.finfo(np.float32).max, (2,), np.float32)
    return spaces.Dict(od), spaces.Discrete(n_actions)


def cubemap_spaces(face=256, sensor="depth", n_actions=4):
    """A cube-map rig for CubeMap2Equirect / CubeMap2Fisheye: six face x face cameras `{sensor}_0` .. `{sensor}_5` in
    the order Back, Down, Front, Left, Right, Up ("rgb": u8 x3, "depth": f32 x1 in [0, 1]), plus the point goal."""
    if sensor not in ("rgb", "depth"):
        raise ValueError(f"cubemap_spaces: sensor {sensor!r} (rgb or depth)")
    box = spaces.Box(0, 255, (face, face, 3), np.uint8) if sensor == "rgb" else \
        spaces.Box(0.0, 1.0, (face, face, 1), np.float32)
    od = {f"{sensor}_{i}": box for i in range(6)}
    od["pointgoal_with_gps_compass"] = spaces.Box(np.finfo(np.float32).min, np.finfo(np.float32).max, (2,),
                                                  np.float32)
    return spaces.Dict(od), spaces.Discrete(n_actions)


def fill_image_(t, g, dev):
    """Synthetic image values by dtype: u8 uniform, int32 class ids 0..39, f32 uniform [0, 1)."""
    if t.dtype == torch.uint8:
        t.copy_(torch.randint(0, 256, t.shape, generator=g, device=dev, dtype=torch.uint8))
    elif t.dtype == torch.int32:
        t.copy_(torch.randint(0, 40, t.shape, generator=g, device=dev, dtype=torch.int32))
    else:
        t.copy_(torch.rand(t.shape, generator=g, device=dev))


def fill_observations_(obs, observation_space, g, dev, chunk_steps: int = 8):
    """Synthetic values for ANY sensor of `observation_space` by dtype / rank: images chunk by chunk (u8 uniform, f32
    uniform [0,1), int32 class ids 0..39), 1-D sensors by name (angles uniform in [-pi, pi), categories uniform over the
    space's range, everything else N(0, 3))."""
    for k, t in obs.items():
        sp = observation_space.spaces[k]
        T1 = t.shape[0]
        if len(sp.shape) == 3:
            for t0 in range(0, T1, chunk_steps):
                fill_image_(t[t0:min(T1, t0 + chunk_steps)], g, dev)
        elif t.dtype == torch.int64:
            t.copy_(torch.randint(0, int(sp.high.max()) + 1, t.shape, generator=g, device=dev))
        elif k == "pointgoal_with_gps_compass":
            goal = torch.rand(t.shape, generator=g, device=dev)
            goal[..., 0] *= 10.0
            goal[..., 1:] = goal[..., 1:] * 2 * math.pi - math.pi
            t.copy_(goal)
        elif k in ("compass", "heading"):
            t.copy_(torch.rand(t.shape, generator=g, device=dev) * 2 * math.pi - math.pi)
        else:
            t.copy_(torch.randn(t.shape, generator=g, device=dev) * 3.0)


def fill_rollout_(storage, seed: int, p_done: float = 1.0 / 250.0, device=None, chunk_steps: int = 8,
                  observation_space=None, n_actions: int = 4):
    """Fill every buffer of a RolloutStorage in place with synthetic data generated ON THE STORAGE'S
    DEVICE chunk by chunk (the full rgb+depth buffer of config #2 is 3.8 GB)."""
    b = storage.buffers
    dev = b["rewards"].device
    g = torch.Generator(device=dev).manual_seed(seed)
    T1, N = b["rewards"].shape[:2]
    obs = b["observations"]
    if observation_space is not None:   # any sensor set (configs #3 / #4)
        fill_observations_(obs, observation_space, g, dev, chunk_steps)
    else:                               # the PointNav RGB-D set of config #2 (generator order kept: seeds are stable)
        for t0 in range(0, T1, chunk_steps):
            t1 = min(T1, t0 + chunk_steps)
            if "rgb" in obs:
                obs["rgb"][t0:t1] = torch.randint(0, 256, obs["rgb"][t0:t1].shape, generator=g, device=dev,
                                                  dtype=torch.uint8)
            if "depth" in obs:
                obs["depth"][t0:t1] = torch.rand(obs["depth"][t0:t1].shape, generator=g, device=dev)
        goal = torch.rand(T1, N, 2, generator=g, device=dev)
        goal[..., 0] *= 10.0
        goal[..., 1] = goal[..., 1] * 2 * math.pi - math.pi
        obs["pointgoal_with_gps_compass"].copy_(goal)
    A = n_actions
    b["masks"].copy_(torch.rand(T1, N, 1, generator=g, device=dev) > p_done)
    b["rewards"].copy_(torch.randn(T1, N, 1, generator=g, device=dev) * 0.1 + 2.5 * (~b["masks"]).float())
    b["value_preds"].copy_(torch.randn(T1, N, 1, generator=g, device=dev) * 0.5)
    b["action_log_probs"].copy_(-math.log(A) + 0.05 * torch.randn(T1, N, 1, generator=g, device=dev))
    b["actions"].copy_(torch.randint(0, A, (T1, N, 1), generator=g, device=dev))
    b["prev_actions"].copy_(torch.randint(0, A, (T1, N, 1), generator=g, device=dev))
    b["recurrent_hidden_states"].copy_(torch.randn(b["recurrent_hidden_states"].shape, generator=g, device=dev) * 0.1)
    storage.current_rollout_step_idxs = [storage.num_steps for _ in storage.current_rollout_step_idxs]
    return torch.randn(N, 1, generator=g, device=dev) * 0.5  # next_value
