"""Name -> class registry with the reference's slots and accessor names
(habitat-baselines/habitat_baselines/common/baseline_registry.py:28-193, backed by
habitat-lab/habitat/core/registry.py:43-69).  Registering under an existing name overwrites
the entry -- that is how these classes drop in under the unchanged YAML keys
(`trainer_name`, `updater_name`, `distrib_updater_name`, `rollout_storage_name`,
`rl.policy.<agent>.name`).  If the real habitat_baselines registry is importable, every
registration is mirrored into it."""
from __future__ import annotations

import collections
from typing import Optional


class BaselineRegistry:
    mapping = collections.defaultdict(dict)

    @classmethod
    def _register(cls, kind: str, to_register=None, *, name: Optional[str] = None):
        def wrap(c):
            cls.mapping[kind][c.__name__ if name is None else name] = c
            try:  # mirror into the reference's registry when it is installed
                from habitat_baselines.common.baseline_registry import baseline_registry as ref
                getattr(ref, f"register_{kind}")(c, name=name)
            except Exception:
                pass
            return c

        return wrap if to_register is None else wrap(to_register)

    @classmethod
    def register_trainer(cls, to_register=None, *, name=None):
        return cls._register("trainer", to_register, name=name)

    @classmethod
    def register_policy(cls, to_register=None, *, name=None):
        return cls._register("policy", to_register, name=name)

    @classmethod
    def register_updater(cls, to_register=None, *, name=None):
        return cls._register("updater", to_register, name=name)

    @classmethod
    def register_storage(cls, to_register=None, *, name=None):
        return cls._register("storage", to_register, name=name)

    @classmethod
    def register_obs_transformer(cls, to_register=None, *, name=None):
        return cls._register("obs_transformer", to_register, name=name)

    @classmethod
    def get_obs_transformer(cls, name):
        return cls.mapping["obs_transformer"].get(name)

    @classmethod
    def get_trainer(cls, name):
        return cls.mapping["trainer"].get(name)

    @classmethod
    def get_policy(cls, name):
        return cls.mapping["policy"].get(name)

    @classmethod
    def get_updater(cls, name):
        return cls.mapping["updater"].get(name)

    @classmethod
    def get_storage(cls, name):
        return cls.mapping["storage"].get(name)


baseline_registry = BaselineRegistry()
