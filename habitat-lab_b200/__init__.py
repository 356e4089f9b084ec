"""hb200 -- H100-native DD-PPO learner hot path behind habitat-baselines' registry API.

The compute path is libhb200.so (hand-written sm_90a CUDA, C ABI in include/hb200.h);
this package is the thin Python host side that mirrors the reference's
Policy / Updater / Storage interfaces.  There is no CPU or PyTorch fallback.
"""
from . import _lib  # noqa: F401
from ._lib import Hb200Error, load  # noqa: F401

__version__ = "0.1.0"

_LAZY = {
    "PointNavResNetPolicy": ("rl.resnet_policy", "PointNavResNetPolicy"),
    "PointNavBaselinePolicy": ("rl.policy", "PointNavBaselinePolicy"),
    "RolloutObservations": ("rl.resnet_policy", "RolloutObservations"),
    "PPO": ("rl.ppo", "PPO"),
    "DDPPO": ("rl.ppo", "DDPPO"),
    "FusedAdam": ("rl.ppo", "FusedAdam"),
    "RolloutStorage": ("common.rollout_storage", "RolloutStorage"),
    "PPOTrainer": ("rl.ppo_trainer", "PPOTrainer"),
    "SingleAgentAccessMgr": ("rl.single_agent_access_mgr", "SingleAgentAccessMgr"),
    "ddp_utils": ("rl.ddp_utils", None),
    "GraphedActor": ("rl.graphed_actor", "GraphedActor"),
    "batch_obs": ("utils.common", "batch_obs"),
    "build_rnn_state_encoder": ("rl.models.rnn_state_encoder", "build_rnn_state_encoder"),
    "RNNStateEncoder": ("rl.models.rnn_state_encoder", "RNNStateEncoder"),
    "TensorDict": ("common.tensor_dict", "TensorDict"),
    "baseline_registry": ("common.baseline_registry", "baseline_registry"),
    "spaces": ("common.spaces", None),
    "ops": ("ops", None),
}


def __getattr__(name):
    if name in _LAZY:
        import importlib

        mod, attr = _LAZY[name]
        m = importlib.import_module(f"{__name__}.{mod}")
        return m if attr is None else getattr(m, attr)
    raise AttributeError(name)


def smoke() -> None:
    from .smoke import run

    run()
