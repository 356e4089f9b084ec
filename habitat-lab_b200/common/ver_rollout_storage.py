"""VERRolloutStorage: the rollout storage of Variable Experience Rollout (habitat-baselines/habitat_baselines/rl/ver/
ver_rollout_storage.py), with the reference's constructor, buffers, auxiliary state and methods.

With `variable_experience` the buffers are one flat [(T+1) * N, ...] array written at `ptr` in the order environments
finish their steps, so an environment may contribute any number of steps to a rollout.  Returns are computed over the
episodes ("sequences") found in it by one kernel (ops.ver_gae) instead of the reference's host loop, and the minibatches
are whole sequences, handed to the learner with their packing metadata (PackedSequenceInfo).

Building the packing metadata stays on the host (numpy, one device-to-host copy of the three id arrays per update); every
arithmetic step on rewards, values and returns runs on the device.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Iterator, List, Optional

import numpy as np
import torch

from .. import ops
from ..rl.resnet_policy import RolloutObservations
from .baseline_registry import baseline_registry
from .rollout_storage import RolloutStorage


def build_pack_info_from_episode_ids(episode_ids: np.ndarray, environment_ids: np.ndarray,
                                     step_ids: np.ndarray) -> dict:
    """Packing metadata of the frames given by their (episode, environment, step) ids, with the reference's meaning
    and order (habitat_baselines/rl/models/rnn_state_encoder.py build_pack_info_from_episode_ids):

    - a sequence is the frames of one (environment, episode), in step order;
    - sequences are ordered by length, longest first (np.argsort of the negated lengths, as the reference sorts, so
      equal lengths come out in the same order);
    - select_inds lists the frames step-major: all sequences' step 0, then every sequence still running at step 1, ...;
      num_seqs_at_step[t] sequences have a step t;
    - last_sequence_in_batch_mask / first_sequence_in_batch_mask mark each environment's last / first episode;
      first_step_for_env is the first frame of each environment's first episode, environments in increasing id order;
      rnn_state_batch_inds maps each sequence to that environment's position in first_step_for_env."""
    episode_ids = np.asarray(episode_ids, dtype=np.int64).reshape(-1)
    environment_ids = np.asarray(environment_ids, dtype=np.int64).reshape(-1)
    step_ids = np.asarray(step_ids, dtype=np.int64).reshape(-1)
    uid = episode_ids * (environment_ids.max() + 1) + environment_ids       # one id per (environment, episode)
    key = uid * (step_ids.max() + 1) + step_ids
    if np.unique(key).size != key.size:
        raise ValueError("build_pack_info_from_episode_ids: duplicate (environment, episode, step) ids")
    by_episode = np.argsort(key)
    seq_uid, lengths = np.unique(uid[by_episode], return_counts=True)
    starts = np.cumsum(lengths) - lengths                                     # of each sequence in by_episode
    order = np.argsort(-lengths)
    lengths, starts = lengths[order], starts[order]
    num_seqs_at_step = (lengths[None, :] > np.arange(int(lengths[0]))[:, None]).sum(1).astype(np.int64)
    step_offset = np.cumsum(num_seqs_at_step) - num_seqs_at_step
    packed = np.empty(uid.size, dtype=np.int64)
    for t, n in enumerate(num_seqs_at_step):
        packed[step_offset[t]: step_offset[t] + n] = starts[:n] + t
    select_inds = by_episode[packed]
    sequence_starts = select_inds[: num_seqs_at_step[0]]
    seq_env = environment_ids[sequence_starts]
    seq_ep = uid[sequence_starts]
    envs, rnn_state_batch_inds = np.unique(seq_env, return_inverse=True)
    last_mask = np.zeros(seq_env.size, dtype=bool)
    first_mask = np.zeros(seq_env.size, dtype=bool)
    first_step_for_env = []
    for e in envs:
        mine = seq_env == e
        last_mask[mine] = seq_ep[mine] == seq_ep[mine].max()
        first = seq_ep[mine] == seq_ep[mine].min()
        first_mask[mine] = first
        first_step_for_env.append(int(sequence_starts[mine][first][0]))
    return dict(select_inds=select_inds, num_seqs_at_step=num_seqs_at_step, sequence_starts=sequence_starts,
                sequence_lengths=lengths, rnn_state_batch_inds=rnn_state_batch_inds.astype(np.int64),
                last_sequence_in_batch_mask=last_mask, first_sequence_in_batch_mask=first_mask,
                last_sequence_in_batch_inds=np.nonzero(last_mask)[0],
                first_episode_in_batch_inds=np.nonzero(first_mask)[0],
                first_step_for_env=np.asarray(first_step_for_env, dtype=np.int64))


def partition_n_into_p(n: int, p: int) -> List[int]:
    return [n // p + (1 if i < n % p else 0) for i in range(p)]


def generate_ver_mini_batches(num_mini_batch, sequence_lengths, num_seqs_at_step, select_inds,
                              last_sequence_in_batch_mask) -> Iterator[np.ndarray]:
    """Frame indices of each minibatch (rl/ver/ver_rollout_storage.py generate_ver_mini_batches): the sequences in a
    random order (np.random.permutation), each environment's bootstrap step left out, cut into num_mini_batch
    near-equal parts that are yielded in a second random order.  The np.random calls are the reference's, so a seeded
    run selects the same frames."""
    lengths = np.array(sequence_lengths, copy=True)
    lengths[last_sequence_in_batch_mask] -= 1
    step_offset = np.cumsum(num_seqs_at_step, dtype=np.int64) - num_seqs_at_step
    seq_order = np.random.permutation(len(lengths))
    steps = [select_inds[s + step_offset[: lengths[s]]] for s in range(len(lengths))]
    frames = np.concatenate([steps[s] for s in seq_order])
    sizes = np.array(partition_n_into_p(int(lengths.sum()), num_mini_batch), dtype=np.int64)
    starts = np.cumsum(sizes, dtype=np.int64) - sizes
    for mb in np.random.permutation(num_mini_batch):
        yield frames[starts[mb]: starts[mb] + sizes[mb]]


@dataclass
class PackedSequenceInfo:
    """What the learner needs to run the recurrence of a VER minibatch over its S sequences (rnn_build_seq_info).

    Frame f of the minibatch is step t of sequence s.  The recurrence runs time-major over [T_max, S] with zero
    padding after each sequence's end: `tm_to_frame[t * S + s]` is f or -1 (padding), `frame_to_tm[f]` is t * S + s.
    Sequence s starts from the hidden state `first_hidden[rnn_state_batch_inds[s]]` times the mask of its first frame
    (the reference's build_rnn_inputs)."""
    num_seqs: int
    max_len: int
    sequence_lengths: torch.Tensor       # int64 [S] on the device
    tm_to_frame: torch.Tensor            # int32 [T_max * S]
    frame_to_tm: torch.Tensor            # int32 [B]
    rnn_state_batch_inds: torch.Tensor   # int64 [S]
    sequence_starts: torch.Tensor        # int64 [S]: minibatch frame of each sequence's step 0
    last_sequence_in_batch_inds: torch.Tensor   # int64 [n_envs], environments in increasing id order
    cpu: dict                            # the numpy metadata (build_pack_info_from_episode_ids)

    @classmethod
    def build(cls, info: dict, device) -> "PackedSequenceInfo":
        lengths = info["sequence_lengths"]
        S, T = len(lengths), int(lengths[0])
        step_offset = np.cumsum(info["num_seqs_at_step"]) - info["num_seqs_at_step"]
        tm = np.full((T, S), -1, dtype=np.int64)
        f2tm = np.empty(info["select_inds"].size, dtype=np.int64)
        for t, n in enumerate(info["num_seqs_at_step"]):
            frames = info["select_inds"][step_offset[t]: step_offset[t] + n]
            tm[t, :n] = frames
            f2tm[frames] = t * S + np.arange(n)
        # the hidden state each environment's last sequence ends in, environments in increasing id order
        last = info["last_sequence_in_batch_inds"]
        last = last[np.argsort(info["rnn_state_batch_inds"][last])]
        dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dt)  # noqa: E731
        return cls(num_seqs=S, max_len=T, sequence_lengths=dev(lengths, torch.int64),
                   tm_to_frame=dev(tm.reshape(-1), torch.int32), frame_to_tm=dev(f2tm, torch.int32),
                   rnn_state_batch_inds=dev(info["rnn_state_batch_inds"], torch.int64),
                   sequence_starts=dev(info["sequence_starts"], torch.int64),
                   last_sequence_in_batch_inds=dev(last, torch.int64), cpu=info)

    @property
    def padding_fraction(self) -> float:
        """Share of the [T_max, S] recurrence steps that are padding."""
        return 1.0 - float(self.cpu["select_inds"].size) / (self.max_len * self.num_seqs)


@baseline_registry.register_storage
class VERRolloutStorage(RolloutStorage):
    def __init__(self, numsteps, num_envs, observation_space, action_space, actor_critic, variable_experience: bool,
                 is_double_buffered: bool = False):
        super().__init__(numsteps, num_envs, observation_space, action_space, actor_critic, is_double_buffered)
        self.use_is_coeffs = bool(variable_experience)
        self.variable_experience = bool(variable_experience)
        b = self.buffers
        if self.use_is_coeffs:
            b["is_coeffs"] = torch.ones_like(b["returns"])
        for k in ("policy_version", "environment_ids", "episode_ids", "step_ids"):
            b[k] = torch.zeros_like(b["returns"], dtype=torch.int64)
        b["is_stale"] = torch.ones_like(b["returns"], dtype=torch.bool)
        self.buffer_size = (self.num_steps + 1) * self._num_envs
        # auxiliary state (the reference keeps it in shared memory for its worker processes; here it is plain)
        self.next_hidden_states = b["recurrent_hidden_states"][0].clone()
        self.next_prev_actions = b["prev_actions"][0].clone()
        self.current_policy_version = torch.ones((1, 1), dtype=torch.int64)
        self.cpu_current_policy_version = np.ones((1, 1), dtype=np.int64)
        self.num_steps_collected = np.zeros((1,), dtype=np.int64)
        self.rollout_done = np.zeros((1,), dtype=bool)
        self.current_steps = np.zeros((num_envs,), dtype=np.int64)
        self.actor_steps_collected = np.zeros((num_envs,), dtype=np.int64)
        self.ptr = np.zeros((1,), dtype=np.int64)
        self.prev_inds = np.full((num_envs,), -1, dtype=np.int64)
        self._first_rollout = np.ones((1,), dtype=bool)
        self.will_replay_step = np.zeros((num_envs,), dtype=bool)
        if self.variable_experience:
            self.buffers.map_in_place(lambda t: t.flatten(0, 1))
        self._pack = None
        self._seq_table = None

    @property
    def num_steps_to_collect(self) -> int:
        return self.buffer_size if self._first_rollout else self._num_envs * self.num_steps

    def insert_first_observations(self, batch):
        """No-op: VER writes every step at `ptr` when it is acted on, the environments' first observations included."""

    def to(self, device):
        super().to(device)
        self.next_hidden_states = self.next_hidden_states.to(device)
        self.next_prev_actions = self.next_prev_actions.to(device)
        self.current_policy_version = self.current_policy_version.to(device)

    def _leaves(self):
        out = []

        def walk(d):
            for v in d.values():
                walk(v) if isinstance(v, dict) else out.append(v)
        walk(self.buffers)
        return out

    def after_update(self):
        self.current_steps[:] = 1
        self.current_steps[self.will_replay_step] -= 1
        self.buffers["is_stale"].fill_(True)
        if not self.variable_experience:
            if not np.all(self.will_replay_step):
                raise RuntimeError("VERRolloutStorage.after_update: every environment must replay its last step "
                                   "without variable experience")
            self.next_hidden_states[:] = self.buffers["recurrent_hidden_states"][-1]
            self.next_prev_actions[:] = self.buffers["prev_actions"][-1]
        else:
            # steps whose action is still in flight keep their row (their reward arrives in the next rollout) at the
            # front, [0, k); the steps to replay with the new policy follow, so the next rollout overwrites them first
            in_flight = ~self.will_replay_step
            k = int(np.count_nonzero(in_flight))
            src = np.concatenate((self.prev_inds[in_flight], self.prev_inds[~in_flight]))
            dst = np.arange(len(src))
            # moving src -> dst as a set of swaps: whatever dst held goes where a src row left a hole
            dst_all = np.concatenate((dst, src[~np.isin(src, dst)]))
            src_all = np.concatenate((src, dst[~np.isin(dst, src)]))
            if len(np.unique(src)) != len(src):
                raise RuntimeError("VERRolloutStorage.after_update: two environments share a previous step")
            d_t = torch.from_numpy(dst_all).to(self.device)
            s_t = torch.from_numpy(src_all).to(self.device)
            for t in self._leaves():
                t[d_t] = t[s_t]
            self.prev_inds[:] = -1
            self.prev_inds[in_flight] = np.arange(k, dtype=np.int64)
            self.will_replay_step[:] = False
            self.ptr[:] = k
            # the rest is ordered so that the oldest policy version is overwritten first (stable: on equal versions
            # the earlier row comes first)
            n = self._num_envs
            diff = self.current_policy_version.view(-1) - self.buffers["policy_version"].view(-1)[n:]
            tie = torch.arange(diff.numel() - 1, -1, -1, dtype=diff.dtype, device=diff.device)
            _, ordering = torch.sort(diff * diff.numel() + tie, descending=True)
            for t in self._leaves():
                t[n:] = t[n:].index_select(0, ordering)
        self.num_steps_collected[:] = 0
        self.rollout_done[:] = False
        self._first_rollout[:] = False
        self._adv_valid = False

    def increment_policy_version(self):
        self.current_policy_version += 1
        self.cpu_current_policy_version += 1

    def after_rollout(self):
        b = self.buffers
        b["is_stale"][:] = b["policy_version"] < self.current_policy_version
        self.current_rollout_step_idxs[0] = self.num_steps + 1
        if self.use_is_coeffs:
            # importance weights against the biased sampling: (T + 1) / (steps the environment contributed)
            env = b["environment_ids"].view(-1)
            count = torch.bincount(env, minlength=self._num_envs).to(torch.float32)
            b["is_coeffs"].copy_(((self.num_steps + 1) / count)[env].view(-1, 1))

    def build_pack_info(self) -> dict:
        """Packing metadata of the whole buffer: one device-to-host copy of the episode / environment / step ids."""
        b = self.buffers
        ids = torch.stack([b["episode_ids"].view(-1), b["environment_ids"].view(-1), b["step_ids"].view(-1)]).cpu()
        self.episode_ids_cpu, self.environment_ids_cpu, self.step_ids_cpu = ids.numpy()
        self._pack = build_pack_info_from_episode_ids(self.episode_ids_cpu, self.environment_ids_cpu,
                                                      self.step_ids_cpu)
        return self._pack

    def compute_returns(self, use_gae, gamma, tau):
        """GAE over the buffer's sequences in one launch (ops.ver_gae), fused with the advantages and their finite-entry
        statistics that PPO.get_advantages reads through fused_advantages()."""
        if self.device.type != "cuda":
            raise ops._lib.Hb200Error("VERRolloutStorage.compute_returns: buffers must be on a CUDA device")
        p = self.build_pack_info()
        table = np.concatenate([p["select_inds"], np.cumsum(p["num_seqs_at_step"]) - p["num_seqs_at_step"],
                                p["sequence_lengths"], p["last_sequence_in_batch_mask"]]).astype(np.int32)
        self._seq_table = torch.from_numpy(table).to(self.device)
        b = self.buffers
        if self._adv is None:
            self._adv = torch.empty_like(b["returns"])
            self._adv_stats = torch.zeros(4, dtype=torch.float64, device=self.device)
        ops.ver_gae(b["rewards"], b["value_preds"], b["returns"], b["is_stale"], self._seq_table,
                    len(p["sequence_lengths"]), len(p["num_seqs_at_step"]), gamma, tau, use_gae, self._adv,
                    self._adv_stats, expected_finite=self.num_steps * self._num_envs)
        self._adv_valid = True
        self.current_rollout_step_idxs[0] = self.num_steps

    def data_generator(self, advantages: Optional[torch.Tensor], num_mini_batch: int) -> Iterator[dict]:
        if not self.variable_experience:
            yield from super().data_generator(advantages, num_mini_batch)
            return
        p = self._pack
        b = self.buffers
        flat_obs = dict(b["observations"].items())
        for mb in generate_ver_mini_batches(num_mini_batch, p["sequence_lengths"], p["num_seqs_at_step"],
                                            p["select_inds"], p["last_sequence_in_batch_mask"]):
            inds = torch.from_numpy(mb).to(self.device)
            batch = {k: b[k][inds] for k in ("rewards", "value_preds", "returns", "action_log_probs", "actions",
                                             "prev_actions", "masks", "is_coeffs", "is_stale", "policy_version")}
            if advantages is not None:
                batch["advantages"] = advantages[inds]
            info = build_pack_info_from_episode_ids(self.episode_ids_cpu[mb], self.environment_ids_cpu[mb],
                                                    self.step_ids_cpu[mb])
            seq = PackedSequenceInfo.build(info, self.device)
            first = torch.from_numpy(mb[info["first_step_for_env"]]).to(self.device)
            batch["recurrent_hidden_states"] = b["recurrent_hidden_states"][first]
            batch["observations"] = RolloutObservations(flat_obs, inds.int())
            batch["mb_inds"] = mb
            batch["rnn_build_seq_info"] = seq
            yield batch
