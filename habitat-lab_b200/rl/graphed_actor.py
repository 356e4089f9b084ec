"""CUDA-graph replay of the actor step (SURVEY 8f row 1).

`policy.act` at rollout batch sizes (N = 64 frames) is ~100 kernels of a few microseconds each: launch-bound.  All of its
workspaces are persistent and its kernels are plain launches on the current stream, so one act() call can be captured
into a CUDA graph and replayed once per environment step; only the inputs are copied into static buffers first.

    actor = GraphedActor(policy, obs_example, hidden, prev_actions, masks)
    out = actor(obs, hidden, prev_actions, masks)      # PolicyActionData; tensors are overwritten by the next call

The packed bf16 weight images the graph reads are refreshed (outside the graph, same buffers) whenever the policy's
weights_key() changes, i.e. after every optimizer step.

With a frozen visual encoder (train_encoder=False) the observations must carry the step's cached `visual_features`:
the captured step then starts at visual_fc, like the trainer's act() calls."""
from __future__ import annotations

from typing import Dict

import torch

from .._lib import Hb200Error
from .resnet_policy import VISUAL_FEATURES_KEY


class GraphedActor:
    def __init__(self, policy, observations: Dict[str, torch.Tensor], rnn_hidden_states, prev_actions, masks,
                 deterministic: bool = False, warmup: int = 2):
        if not rnn_hidden_states.is_cuda:
            raise Hb200Error("GraphedActor: inputs must be CUDA tensors (no CPU fallback)")
        net = getattr(policy, "net", None)
        frozen = net is not None and any(not p.requires_grad for p in net.visual_encoder.parameters())
        if frozen and VISUAL_FEATURES_KEY not in observations:
            # the captured step would run the encoder every replay although the rollout already holds its output
            raise Hb200Error(f"GraphedActor: the policy's visual encoder is frozen (train_encoder=False); pass the "
                             f"rollout step's {VISUAL_FEATURES_KEY!r} with the observations so the captured act() reads "
                             "them instead of re-running the encoder")
        self.policy = policy
        self.deterministic = deterministic
        self.obs = {k: v.clone() for k, v in observations.items()}
        self.hid, self.pa, self.mk = rnn_hidden_states.clone(), prev_actions.clone(), masks.clone()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side), torch.no_grad():   # allocations + weight packing happen here, not in the graph
            for _ in range(max(1, warmup)):
                policy.act(self.obs, self.hid, self.pa, self.mk, deterministic=deterministic)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        self._wkey = policy.weights_key()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph), torch.no_grad():
            self.out = policy.act(self.obs, self.hid, self.pa, self.mk, deterministic=deterministic)

    @torch.no_grad()
    def __call__(self, observations, rnn_hidden_states, prev_actions, masks):
        for k, v in self.obs.items():
            v.copy_(observations[k])
        self.hid.copy_(rnn_hidden_states)
        self.pa.copy_(prev_actions)
        self.mk.copy_(masks)
        key = self.policy.weights_key()
        if key != self._wkey:   # the graph reads the packed images: refresh them in place, outside the graph
            self.policy.refresh_inference_weights()
            self._wkey = self.policy.weights_key()
        self.graph.replay()
        return self.out
