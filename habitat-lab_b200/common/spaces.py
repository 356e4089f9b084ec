"""Minimal observation/action space containers (gym is absent in this image).  Only the
attributes the hot path reads -- shape, dtype, low/high, n, .spaces -- are provided, with gym's
names so the real gym.spaces objects are accepted interchangeably."""
from __future__ import annotations

import collections

import numpy as np


class Space:
    def __init__(self, shape=None, dtype=None):
        self.shape = None if shape is None else tuple(shape)
        self.dtype = None if dtype is None else np.dtype(dtype)


class Box(Space):
    def __init__(self, low, high, shape=None, dtype=np.float32):
        if shape is None:
            shape = np.asarray(low).shape
        super().__init__(shape, dtype)
        self.low = np.full(self.shape, low, dtype=self.dtype)
        self.high = np.full(self.shape, high, dtype=self.dtype)


class Discrete(Space):
    def __init__(self, n):
        super().__init__((), np.int64)
        self.n = int(n)


class Dict(Space):
    def __init__(self, spaces=None, **kw):
        super().__init__(None, None)
        self.spaces = collections.OrderedDict(spaces or {})
        self.spaces.update(kw)

    def __getitem__(self, k):
        return self.spaces[k]

    def __iter__(self):
        return iter(self.spaces)

    def __contains__(self, k):
        return k in self.spaces

    def keys(self):
        return self.spaces.keys()

    def items(self):
        return self.spaces.items()

    def __len__(self):
        return len(self.spaces)


def continuous_action_dim(space):
    """Number of action dimensions of a 1-D Box action space (continuous control), None for a discrete one (any space
    with `.n`, as before).  Any other action space (MultiDiscrete, Dict, a Box of another rank) raises
    NotImplementedError."""
    if hasattr(space, "n"):
        return None
    kind = type(space).__name__
    if kind == "Box" and len(space.shape) == 1:
        return int(space.shape[0])
    raise NotImplementedError(f"action space {kind} {getattr(space, 'shape', None)}: only Discrete and 1-D Box action "
                              "spaces are implemented")
